"""Host mirror of ``ratinabox.Agent`` -- batched over ``n_agents`` -- whose
``update()`` runs on the GPU through libriab_b200 (C ABI: include/riab_b200.h).

API parity with the reference (ratinabox/Agent.py):
  * ``Agent(Environment, params)``; same ``default_params`` keys (Agent.py:68-84) plus
    ``n_agents`` (batch size, default 1), ``seed``, ``id_offset`` (multi-GPU shard
    offset), ``history_bytes_limit``.
  * ``update(dt=None, drift_velocity=None, drift_to_random_strength_ratio=1, **kwargs)``
    with the reference's per-call kwargs (Agent.py:280-285, :353-355).
  * state attributes ``pos, velocity, rotational_velocity, measured_velocity,
    measured_rotational_velocity, head_direction, distance_travelled,
    distance_to_closest_wall, t, dt`` are readable AND writable between steps (the
    reference's tests poke them: tests/test_advanced.py:47-48).  With ``n_agents == 1``
    they have the reference's shapes ((2,) / scalar); otherwise a leading agent axis.
  * ``history`` / ``get_history_arrays()`` (Agent.py:111-120, :1093-1102), backed by a
    device ring buffer that is only materialised on access.
  * ``import_trajectory(times, positions, dataset)`` (Agent.py:543-659) and
    ``update(forced_next_position=...)`` (Agent.py:202-253): the imported / forced branches of
    Agent.update.  One trajectory for every agent, or one per agent over shared times; its
    not-a-knot spline is solved on the device (riab_trajectory_build) and ``run()`` follows it.

The launch is lazy: ``update()`` queues the motion step, and the first
``Neurons.update()`` that follows runs it fused with its firing rates in one
kernel (riab_step_fused).  Reading any state attribute, or a second ``update()``,
flushes a queued step through the stand-alone kernel (riab_agent_update), so the
observable behaviour is that of the reference's eager calls.

There is no CPU fallback: without a CUDA device or the built library this raises.
"""
import copy
import ctypes as C
import warnings

import numpy as np

from . import _lib

_STATE = ("pos", "velocity", "rotational_velocity", "measured_velocity", "measured_rotational_velocity",
          "head_direction", "distance_travelled", "distance_to_closest_wall")
_VEC = {"pos", "velocity", "measured_velocity", "head_direction"}


def _torch():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("ratinabox_b200 needs a CUDA device (there is no CPU fallback)")
    return torch


class _HistoryView:
    """dict-like view with the reference's keys; values are materialised lazily."""

    def __init__(self, owner):
        self._o = owner

    def keys(self):
        return self._o._history_keys()

    def __iter__(self):
        return iter(self.keys())

    def __contains__(self, k):
        return k in self.keys()

    def __getitem__(self, k):
        return self._o.get_history_arrays()[k]

    def items(self):
        a = self._o.get_history_arrays()
        return [(k, a[k]) for k in self.keys()]


class Agent:
    _VEC_NAMES = _VEC          # state arrays with a trailing axis of 2 (a subclass may keep more arrays in self._s)
    default_params = {                                              # ratinabox/Agent.py:68-84
        "name": None,
        "dt": 0.05,
        "speed_coherence_time": 0.7,
        "speed_mean": 0.08,
        "speed_std": 0.08,
        "rotational_velocity_coherence_time": 0.08,
        "rotational_velocity_std": (120 * (np.pi / 180)),
        "head_direction_smoothing_timescale": 0.15,
        "thigmotaxis": 0.5,
        "wall_repel_distance": 0.1,
        "wall_repel_strength": 1.0,
        "save_history": True,
        # ---- batch-engine additions
        "n_agents": 1,
        "seed": 0,
        "id_offset": 0,
        "history_bytes_limit": 2 << 30,
        # stepped API: True  = update() queues the motion step and the first Neurons.update() runs it fused with its rates
        #                      (riab_step_fused, one kernel per (motion, cell type));
        #              False = update() launches the motion kernel at once and Neurons.update() the rate kernel: the float64
        #                      motion chain then overlaps the host side of Neurons.update() instead of gating the rate warps
        #                      inside one kernel (measured faster end to end), and reading
        #                      positions only waits for the motion kernel.
        "fused_step": False,
    }

    def __init__(self, Environment, params={}):
        torch = _torch()
        self._lib = _lib.load()
        self.params = copy.deepcopy(__class__.default_params)
        self.params.update(params)
        unexpected = [k for k in params if k not in __class__.default_params]
        if unexpected:
            warnings.warn(f"Found {len(unexpected)} unexpected params key(s) while initializing Agent: {unexpected}")
        for k, v in self.params.items():
            setattr(self, k, v)
        self.Environment = Environment
        self.agent_idx = len(Environment.Agents)
        if self.name is None:
            self.name = f"agent_{self.agent_idx}"
        Environment.add_agent(agent=self)
        self.Neurons = []
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.n_agents = int(self.n_agents)
        A = self.n_agents

        self.prev_t = 0
        self.t = 0
        self.average_measured_speed = max(self.speed_mean, self.speed_std)
        self.use_imported_trajectory = False
        self._step = 0
        self._t_hist = []
        self._shadow = {}
        self._pinned = {}
        self._pending = None
        self._tape = None
        self._rec = None
        self._pos_mirror_current = False
        self._drift_keep = None
        self._env_key = None
        self._staging_only = False          # run(): update() only fills the structs
        self._drift_host_ptr = None         # pinned drift commands of the queued step (eager stepped API)
        self._pos_copy_inflight = False
        self._motion_event_valid = False
        self._traj = None                   # imported trajectory: device arrays + riab_trajectory
        self._src = _lib.MotionSource()     # motion source of the current step
        self._forced_dev = None
        self._forced_keep = None

        # ---- initial state (Agent.py:523-535, :136-141), sampled on the host like the reference
        pos = Environment.sample_positions(n=A, method="random")
        direction = np.random.uniform(0, 2 * np.pi, size=A)
        vel = self.speed_mean * np.stack((np.cos(direction), np.sin(direction)), axis=1)
        f64 = dict(dtype=torch.float64, device=self.device)
        self._s = {
            "pos": torch.as_tensor(pos, **f64).contiguous(),
            "velocity": torch.as_tensor(vel, **f64).contiguous(),
            "rotational_velocity": torch.zeros(A, **f64),
            "measured_velocity": torch.as_tensor(vel, **f64).contiguous().clone(),
            "measured_rotational_velocity": torch.zeros(A, **f64),
            "head_direction": torch.as_tensor(vel / np.linalg.norm(vel, axis=1, keepdims=True), **f64).contiguous(),
            "distance_travelled": torch.zeros(A, **f64),
            "distance_to_closest_wall": torch.full((A,), float("inf"), **f64),
        }
        self._agents_c = _lib.Agents()
        self._refresh_agents_struct()
        self._mp = _lib.MotionParams()
        self._io = _lib.StepIO()
        self._env_c = _lib.Env()
        self._drift_dev = None
        # ---- history ring (device)
        self._hist = None
        self._hist_cap = 0
        self._hist_rows = 0        # rows written since reset
        self._history_view = _HistoryView(self)
        self._last_history_array_cache_time = None
        self._history_arrays = {}

    # ------------------------------------------------------------------ plumbing
    def _refresh_agents_struct(self):
        a = self._agents_c
        a.n_agents = self.n_agents
        a.id_offset = int(self.id_offset)
        for k in _STATE:
            setattr(a, {"velocity": "velocity"}.get(k, k), self._s[k].data_ptr())

    def _env_struct(self):
        env = self.Environment
        key = (env._walls_signature(), env.boundary_conditions)
        if key == self._env_key:
            return self._env_c
        self._env_key = key
        walls = env.walls_device(self.device)
        e = self._env_c
        e.walls_dev = walls.data_ptr()
        e.n_walls = int(walls.shape[0])
        e.n_boundary_walls = int(env.n_boundary_walls)
        for i in range(4):
            e.extent[i] = float(env.extent[i])
        e.boundary_mode = 1 if env.boundary_conditions == "periodic" else (2 if env.is_polygonal else 0)
        e.n_hole_walls, e.hole_wall0 = env.n_hole_walls, env.hole_wall0
        e.scale = float(env.scale)
        self._walls_keepalive = walls
        return e

    def _stream(self):
        """The caller's current CUDA stream on this device (raw handle; torch's C accessor is ~20x cheaper than
        building a torch.cuda.Stream object on the per-step path)."""
        import torch
        raw = getattr(torch._C, "_cuda_getCurrentRawStream", None)
        if raw is not None:
            return C.c_void_p(raw(self.device.index))
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _sync_stream(self):
        _lib.check(self._lib.riab_stream_synchronize(self._stream()))

    def _squeeze(self, name, arr):
        if self.n_agents != 1:
            return arr
        return arr[0].copy() if name in self._VEC_NAMES else arr[0].item()

    _SHADOW_MAX = 4096      # above this many agents state reads are plain copies (no in-place write tracking)

    def _get_state(self, name, view=False):
        self._flush_pending()
        if name in self._shadow and not view:
            return self._shadow[name][0]
        import torch
        t = self._s[name]
        if self.n_agents > self._SHADOW_MAX or view:
            # large batches: one pinned staging buffer per state array, asynchronous D2H on the current
            # stream + one stream sync.  `Ag.pos` hands out a fresh COPY of it (reference-style code keeps
            # such arrays: `traj.append(Ag.pos)`); in-place edits of that copy are not tracked -- assign to
            # write (``Ag.pos = new_positions``).  state_view() returns the staging buffer itself.
            buf = self._pinned_buffer(name)
            if name == "pos" and self._pos_mirror_current and self._motion_event_valid:
                # the copy engine is bringing the positions into this buffer: wait for that copy only
                _lib.check(self._lib.riab_positions_wait())
            else:
                if not (name == "pos" and self._pos_mirror_current):
                    # (the motion kernels post the new positions straight into the pinned `pos` buffer:
                    # riab_step_io.pos_mirror -- no copy needed while that mirror is current)
                    buf.copy_(t, non_blocking=True)
                self._sync_stream()
            arr = buf.numpy()
            if view:
                arr = arr.view()
                arr.flags.writeable = False
                return arr
            return arr.copy()
        host = t.cpu().numpy()
        val = self._squeeze(name, host)
        if isinstance(val, np.ndarray):
            self._shadow[name] = (val, val.copy())
        return val

    def _pinned_buffer(self, name):
        """The page-locked host copy of a state array that large batches read through (the motion kernels post the
        positions straight into the "pos" one)."""
        buf = self._pinned.get(name)
        if buf is None:
            import torch
            t = self._s[name]
            buf = self._pinned[name] = torch.empty(t.shape, dtype=t.dtype).pin_memory()
        return buf

    def state_view(self, name="pos"):
        """Zero-copy, READ-ONLY view of a state array in page-locked host memory, shape (n_agents, ...) -- the opt-in
        fast path for per-step control loops (`Ag.pos` returns a private copy instead).  The view ALIASES a buffer the
        engine reuses: it is valid until the next ``update()`` / ``run()`` of this Agent (the next motion kernel posts
        the new positions into the same memory, asynchronously); copy what you need to keep."""
        if name not in _STATE:
            raise KeyError(name)
        return self._get_state(name, view=True)

    def _set_state(self, name, value):
        import torch
        self._flush_pending()
        self._shadow.pop(name, None)
        if name == "pos":
            self._pos_mirror_current = False
        if name == "pos":
            self._wait_pos_copy()
        arr = np.asarray(value, dtype=np.float64)
        if name in self._VEC_NAMES:
            arr = np.broadcast_to(arr.reshape(-1, 2) if arr.size == 2 * self.n_agents else arr, (self.n_agents, 2))
        else:
            arr = np.broadcast_to(arr.reshape(-1) if arr.size == self.n_agents else arr, (self.n_agents,))
        self._s[name].copy_(torch.as_tensor(np.array(arr, dtype=np.float64, order="C", copy=True)))

    def _sync_user_writes(self):
        """Upload state arrays the user mutated in place since they were read."""
        for name, (host, snap) in list(self._shadow.items()):
            if not np.array_equal(host, snap, equal_nan=True):
                self._shadow.pop(name)
                self._set_state(name, host)
        self._shadow.clear()

    # state attributes (properties are generated below the class body)

    # -------------------------------------------------------------------- update
    def import_trajectory(self, times=None, positions=None, dataset=None, interpolate=True):
        """Agent.import_trajectory (ratinabox/Agent.py:543-659) for every agent.  ``times`` (T,) are shared by all
        agents; ``positions`` is (T, 2), one trajectory for every agent, or (n_agents, T, 2), one per agent.  update()
        and run() then move the agents to ``pos_interp(t % max(t_interp))``, pos_interp the not-a-knot cubic spline of
        scipy's interp1d(kind="cubic"), solved on the device.  ``dataset`` names ``<ratinabox>/data/<dataset>.npz`` of
        an installed ratinabox package (or is a path to such a file)."""
        import os
        import torch
        if interpolate is not True:
            raise NotImplementedError("import_trajectory(interpolate=False) is not supported: the reference itself fails "
                                      "there (Agent.py:657 reads self.pos_interp, which only interpolate=True creates)")
        self._flush_pending()
        assert self.Environment.boundary_conditions == "solid", "Only solid boundary conditions are supported"
        if dataset is not None:
            if dataset == "sargolini":
                print(
                    """Attempting to import Sargolini locomotion dataset.
                    Please cite Sargolini et al. (2006) DOI:10.1126/science.1125572 if you use this in your work.
                    The full dataset (along with many more) can be found here https://www.ntnu.edu/kavli/research/grid-cell-data
                    The exact datafile being used is 8F6BE356-3277-475C-87B1-C7A977632DA7_1/11084-03020501_t2c1.mat"""
                )
            try:
                import ratinabox
                base = os.path.abspath(os.path.join(ratinabox.__file__, os.pardir))
            except ImportError:
                base = os.path.abspath(os.path.join(__file__, os.pardir))
            dataset = os.path.join(os.path.join(base, "data"), dataset + ".npz")
            try:
                data = np.load(dataset)
            except FileNotFoundError:
                print(f"IMPORT FAILED. No datafile found at {dataset}. Please try a different one. For now the default "
                      f"inbuilt random policy will be used.")
                return
            times = data["t"]
            positions = data["pos"]
            print(f"Successfully imported dataset from {dataset}")
        else:
            if (times is not None) and (positions is not None):
                times, positions = np.array(times), np.array(positions)
                print("Successfully imported dataset from arrays passed")
            else:
                print("No data passed, provided arguments 'times' and 'positions'")
        times = np.asarray(times, dtype=np.float64)
        positions = np.asarray(positions, dtype=np.float64)
        if times.ndim != 1:
            raise NotImplementedError("per-agent time bases are not supported: pass one (T,) array of times shared by "
                                      "every agent, with positions (T, 2) or (n_agents, T, 2)")
        per_agent = positions.ndim == 3
        if per_agent and positions.shape[0] != self.n_agents:
            raise ValueError(f"positions of shape {positions.shape}: expected (T, 2) or (n_agents={self.n_agents}, T, 2)")
        assert (positions.shape[1] if per_agent else len(positions)) == len(times), \
            "time and position arrays must have same length"
        times = times - min(times)
        print(f"Total of {times[-1]:.1f} s of data available")
        ex = self.Environment.extent
        positions = positions.reshape(self.n_agents, -1, 2) if per_agent else positions.reshape(-1, 2)
        px, py = positions[..., 0], positions[..., 1]
        if (px.max() > ex[1]) or (px.min() < ex[0]) or (py.max() > ex[3]) or (py.min() < ex[2]):
            print(
                f"""WARNING: the size of the trajectory is significantly larger than the environment you are using.
                    The Environment extent is [minx,maxx,miny,maxy]=[{ex[0]:.1f},{ex[1]:.1f},{ex[2]:.1f},{ex[3]:.1f}], whereas extreme coords are [{px.min():.1f},{px.max():.1f},{py.min():.1f},{py.max():.1f}].
                    Recommended to use larger environment."""
            )
        # interp1d's own checks of the sample times (at least 4 for kind="cubic", no duplicates) and its sort
        from scipy.interpolate import interp1d
        interp1d(times, np.zeros(len(times)), kind="cubic", fill_value="extrapolate")
        order = np.argsort(times, kind="mergesort")
        xs = np.ascontiguousarray(times[order])
        ys = positions[:, order, :].transpose(1, 0, 2) if per_agent else positions[order][:, None, :]
        T, n_traj = len(xs), ys.shape[1]
        need = 32 * T * n_traj + 8 * T
        free, _ = torch.cuda.mem_get_info(self.device)
        if need > free:
            raise MemoryError(f"import_trajectory: {n_traj} trajectories of {T} samples need {need / 2**30:.2f} GiB of "
                              f"device memory (positions and spline coefficients), {free / 2**30:.2f} GiB are free")
        f64 = dict(dtype=torch.float64, device=self.device)
        tr = {"times": torch.as_tensor(xs, **f64), "y": torch.as_tensor(np.ascontiguousarray(ys), **f64)}
        tr["M"] = torch.empty_like(tr["y"])
        c = _lib.Trajectory()
        c.times_dev, c.y_dev, c.M_dev = tr["times"].data_ptr(), tr["y"].data_ptr(), tr["M"].data_ptr()
        c.T, c.n_traj, c.t_max = T, n_traj, float(xs[-1])
        _lib.check(self._lib.riab_trajectory_build(C.byref(c), xs.ctypes.data_as(_lib.c_double_p), self._stream()))
        tr["c"] = c
        self._traj = tr
        self.interpolate = interpolate
        self.t_interp = times
        self.use_imported_trajectory = True
        # pos = prev_pos = pos_interp(0) (Agent.py:658-659): the first sample
        self.pos = np.ascontiguousarray(ys[0])

    def _stage_source(self, forced):
        """Fill self._src for this step: the imported trajectory (which wins over forced_next_position, Agent.py:220-
        229) or the forced positions.  Returns the motion kind."""
        import torch
        src = self._src
        if self.use_imported_trajectory:
            src.kind = _lib.MOTION_IMPORTED
            src.traj = self._traj["c"]
            src.t = float(self.t)
            return src.kind
        src.kind = _lib.MOTION_FORCED
        if isinstance(forced, torch.Tensor):
            f = forced
        else:
            assert isinstance(forced, np.ndarray), "forced_next_position must be an np.array"       # Agent.py:250
            f = torch.as_tensor(forced)
        assert tuple(f.shape) in ((2,), (self.n_agents, 2)), \
            "forced_next_position must be an np.array of shape Env.D"                                 # Agent.py:251
        if f.dtype != torch.float64:
            f = f.to(torch.float64)
        src.forced_broadcast = 1 if tuple(f.shape) == (2,) else 0
        if (f.is_cuda or f.is_pinned()) and f.is_contiguous():
            # device or page-locked host positions are read by the motion kernel itself; like a non_blocking copy, the
            # buffer must not change before the step has run
            self._forced_keep = f
            src.forced_dev = f.data_ptr()
        else:
            if self._forced_dev is None or tuple(self._forced_dev.shape) != tuple(f.shape):
                self._forced_dev = torch.empty(tuple(f.shape), dtype=torch.float64, device=self.device)
            self._forced_dev.copy_(f, non_blocking=True)
            src.forced_dev = self._forced_dev.data_ptr()
        return src.kind

    def update(self, dt=None, drift_velocity=None, drift_to_random_strength_ratio=1, **kwargs):
        """Agent.update (ratinabox/Agent.py:160-242) for every agent: the random-motion branch, or the imported /
        forced one (import_trajectory, forced_next_position), which ignore drift_velocity and the motion kwargs."""
        import torch
        self._flush_pending()
        forced = kwargs.get("forced_next_position", None)
        if self.use_imported_trajectory or forced is not None:
            return self._update_source(dt, forced, kwargs)
        self._sync_user_writes()
        self._fill_motion_params(dt or self.dt, kwargs, drift_to_random_strength_ratio)
        io = self._io
        io.drift_velocity = None
        self._drift_host_ptr = None
        if drift_velocity is not None:
            if self._drift_dev is None:
                self._drift_dev = torch.empty((self.n_agents, 2), dtype=torch.float64, device=self.device)
            if isinstance(drift_velocity, torch.Tensor):
                d = drift_velocity
            else:
                assert isinstance(drift_velocity, np.ndarray), "drift_velocity must be an np.array"   # Agent.py:333
                d = torch.as_tensor(drift_velocity)        # zero-copy view of the host array
            assert tuple(d.shape) in ((2,), (self.n_agents, 2)), "drift_velocity must have shape (Env.D,) or (n_agents, Env.D)"
            if d.dtype != torch.float64:
                d = d.to(torch.float64)
            if (not d.is_cuda) and d.is_pinned() and d.is_contiguous() and tuple(d.shape) == (self.n_agents, 2):
                self._drift_keep = d
                if self.fused_step or self._staging_only:
                    # page-locked host commands: the fused kernel reads them over the bus itself (unified addressing),
                    # no staging copy.  Like a non_blocking copy, the buffer must not change before the step has run.
                    io.drift_velocity = d.data_ptr()
                else:
                    # page-locked host commands: riab_agent_update_host uploads them with a copy engine on the library's side
                    # stream at once -- while the previous step's rate kernel still occupies the compute stream -- and the
                    # motion kernel waits for that copy only.  (Zero-copy loads inside the float64 motion chain would stall
                    # it on PCIe latency instead.)
                    self._drift_host_ptr = d.data_ptr()
            else:
                # host -> device on the current stream (asynchronous when the host buffer is pinned)
                self._drift_dev.copy_(d.expand(self.n_agents, 2), non_blocking=True)
                io.drift_velocity = self._drift_dev.data_ptr()
        io.xi = None
        self._tape = None
        xi = kwargs.get("_xi", None)          # parity tap: injected standard normals (oracle mode A)
        if xi is not None:
            self._tape = torch.as_tensor(np.ascontiguousarray(xi, dtype=np.float64).reshape(self.n_agents, 2),
                                         device=self.device)
            io.xi = self._tape.data_ptr()
        io.collision_mask = io.first_hit = io.n_iters = None
        self._rec = None
        if kwargs.get("_record_collisions", False):
            W = int(self.Environment.walls.shape[0])
            self._rec = dict(
                mask=torch.zeros((self.n_agents, _lib.MAX_REC_ITERS, W), dtype=torch.uint8, device=self.device),
                first_hit=torch.full((self.n_agents, _lib.MAX_REC_ITERS), -1, dtype=torch.int32, device=self.device),
                n_iters=torch.zeros(self.n_agents, dtype=torch.int32, device=self.device))
            io.collision_mask = self._rec["mask"].data_ptr()
            io.first_hit = self._rec["first_hit"].data_ptr()
            io.n_iters = self._rec["n_iters"].data_ptr()
        self._stage_step(dt)
        io.pos_mirror = None
        if self.n_agents > self._SHADOW_MAX and (self.fused_step or self._staging_only):
            # large batches: the motion step also posts the new positions into the pinned host buffer that
            # `Ag.pos` hands out, so reading them back after the step costs a stream sync and no copy
            io.pos_mirror = self._pinned_buffer("pos").data_ptr()
            self._pos_mirror_current = True
        self._pending = True
        if not self.fused_step and not self._staging_only:
            self._flush_pending()                      # launch the motion kernel now (asynchronous)

    def _fill_motion_params(self, dt, kwargs, drift_to_random_strength_ratio=1, mp=None):
        mp = self._mp if mp is None else mp
        mp.dt = float(dt)
        mp.speed_coherence_time_kw = float(kwargs.get("speed_coherence_time", self.speed_coherence_time))
        mp.speed_mean_kw = float(kwargs.get("speed_mean", self.speed_mean))
        mp.speed_mean = float(self.speed_mean)
        mp.speed_std = float(self.speed_std)
        mp.speed_coherence_time = float(self.speed_coherence_time)
        mp.rotational_velocity_coherence_time_kw = float(
            kwargs.get("rotational_velocity_coherence_time", self.rotational_velocity_coherence_time))
        mp.rotational_velocity_std_kw = float(kwargs.get("rotational_velocity_std", self.rotational_velocity_std))
        mp.rotational_velocity_drift_kw = float(kwargs.get("rotational_velocity_drift", 0))
        mp.head_direction_smoothing_timescale = float(self.head_direction_smoothing_timescale)
        mp.thigmotaxis_kw = float(kwargs.get("thigmotaxis", self.thigmotaxis))
        mp.wall_repel_distance_kw = float(kwargs.get("wall_repel_distance", self.wall_repel_distance))
        mp.wall_repel_strength_kw = float(kwargs.get("wall_repel_strength", self.wall_repel_strength))
        mp.drift_to_random_strength_ratio = float(drift_to_random_strength_ratio)

    def _stage_step(self, dt):
        """The clock (t += dt, like the reference's), the Philox key and the agent-history row of the step that
        update() stages."""
        dt = (dt or self.dt)
        self.dt = dt
        self.prev_t = self.t
        self.t += dt
        io = self._io
        io.seed = int(self.seed) & 0xFFFFFFFFFFFFFFFF
        io.step = self._step
        io.history_row = None
        if self.save_history:
            io.history_row = self._history_row_ptr()
            self._t_hist.append(self.t)
        self._step += 1
        return io

    def _update_source(self, dt, forced, kwargs):
        """The imported / forced branches of Agent.update (Agent.py:219-242).  The motion kernel is launched at once
        (with fused_step too: the rates then take the unfused path), except while run() stages its first step."""
        if not self.use_imported_trajectory:
            self._stage_source(forced)          # validates before the clock moves
        self._sync_user_writes()
        io = self._stage_step(dt)
        if self.use_imported_trajectory:
            self._stage_source(None)
        self._fill_motion_params(self.dt, kwargs)
        io.drift_velocity = io.xi = None
        io.collision_mask = io.first_hit = io.n_iters = None
        io.pos_mirror = None
        self._tape = self._rec = None
        self._drift_host_ptr = None
        self._pos_mirror_current = False
        self._motion_event_valid = False
        if self._staging_only:
            return
        self._wait_pos_copy()
        _lib.check(self._lib.riab_agent_update_src(C.byref(self._agents_c), C.byref(self._env_struct()), C.byref(self._mp),
                                                   C.byref(io), C.byref(self._src), self._stream()))

    def _wait_pos_copy(self):
        """Order the compute stream behind an in-flight D2H copy of the positions (it reads what comes next overwrites)."""
        if self._pos_copy_inflight:
            _lib.check(self._lib.riab_positions_fence(self._stream()))
            self._pos_copy_inflight = False

    def _flush_pending(self):
        """Run a queued motion step that no Neurons.update() fused with."""
        if self._pending:
            self._pending = None
            if self.fused_step:
                self._wait_pos_copy()
                _lib.check(self._lib.riab_agent_update(C.byref(self._agents_c), C.byref(self._env_struct()),
                                                       C.byref(self._mp), C.byref(self._io), self._stream()))
                return
            # eager stepped API: one C call = [copy-engine upload of pinned drift commands on the side stream] -> motion
            # kernel -> [copy-engine download of the new positions on the side stream, large batches]; readers of `pos`
            # then wait for that download only, not for the rate kernels queued behind the motion kernel
            pos_out = None
            if self.n_agents > self._SHADOW_MAX:
                pos_out = self._pinned_buffer("pos").data_ptr()
            stage = self._drift_dev.data_ptr() if self._drift_host_ptr is not None else None
            _lib.check(self._lib.riab_agent_update_host(C.byref(self._agents_c), C.byref(self._env_struct()), C.byref(self._mp),
                                                        C.byref(self._io), self._drift_host_ptr, stage, pos_out, self._stream()))
            if pos_out is not None:
                self._pos_copy_inflight = True
                self._motion_event_valid = True
                self._pos_mirror_current = True

    def _take_pending(self):
        """Called by Neurons.update(): hands over the queued step for fusion."""
        if self._pending:
            self._pending = None
            self._wait_pos_copy()
            self._motion_event_valid = False            # the fused kernel posts the positions: wait for the stream
            return True
        return False

    def run(self, n_steps, **kwargs):
        """``for _ in range(n_steps): self.update(**kwargs); [Ns.update() for Ns in self.Neurons]``
        (the reference's user loop, tests/test_advanced.py:21-23) executed by libriab_b200's
        riab_run without returning to Python between steps.  History rows land in the
        device rings exactly as the per-step calls would put them."""
        import torch
        n_steps = int(n_steps)
        if n_steps <= 0:
            return
        if "drift_velocity" in kwargs and kwargs["drift_velocity"] is not None:
            raise NotImplementedError("run() is the free-exploration loop; step with update(drift_velocity=...) for control")
        if kwargs.get("forced_next_position", None) is not None:
            raise NotImplementedError("run() cannot take forced_next_position: a forced position belongs to one step; "
                                      "step with update(forced_next_position=...)")
        for ns in self.Neurons:
            ns._check_run()
        # stage everything exactly like one update() would, then hand the loop to C
        self._staging_only = True
        try:
            self.update(**kwargs)
        finally:
            self._staging_only = False
        self._pending = None
        # a device-resident loop needs no per-step host mirror of the positions (1 MB of bus writes per step at
        # 65 536 agents); reads after the run copy once
        self._io.pos_mirror = None
        self._pos_mirror_current = False
        self._motion_event_valid = False
        self._wait_pos_copy()
        dt = self.dt
        first_step = self._step - 1
        A = self.n_agents
        # rings: make room for n_steps rows (the single update() above already reserved one)
        if self.save_history:
            self._hist_rows -= 1
            self._t_hist.pop()
            self._reserve_history(n_steps)
            hist = _lib.AgentHistory(self._hist.data_ptr(), self._hist_cap, self._hist_rows % self._hist_cap)
        else:
            hist = _lib.AgentHistory(None, 0, 0)
        pops = (_lib.Population * max(1, len(self.Neurons)))()
        for ns in self.Neurons:
            ns._reserve_history(n_steps)          # first: a FeedForwardLayer binds the other populations' ring rows
        for i, ns in enumerate(self.Neurons):
            cells = ns._cells_for_run()
            out, nz = ns._fill_out_structs(None, None)
            nz.step = ns._upd
            p = pops[i]
            p.kind, p.cells = ns._cells_kind, C.cast(C.pointer(cells), C.c_void_p)
            p.noise, p.out = nz, out
            p.rates_ring = ns._hist.data_ptr()
            p.spikes_ring = ns._spk.data_ptr() if (ns.save_history and ns.save_spikes) else None
            p.ring_rows, p.ring_next = ns._hist_cap, ns._hist_rows % ns._hist_cap
        self._io.step = first_step
        if self.use_imported_trajectory:
            # the first step's clock (the staging update() made its `t += dt`); the library advances it per step
            _lib.check(self._lib.riab_run_src(C.byref(self._agents_c), C.byref(self._env_struct()), C.byref(self._mp),
                                              C.byref(self._io), C.byref(self._src), pops, len(self.Neurons), C.byref(hist),
                                              n_steps, self._stream()))
        else:
            _lib.check(self._lib.riab_run(C.byref(self._agents_c), C.byref(self._env_struct()), C.byref(self._mp),
                                          C.byref(self._io), pops, len(self.Neurons), C.byref(hist), n_steps,
                                          self._stream()))
        # host-side bookkeeping of the n_steps that just ran: the clock advances by `t += dt` per step like update()
        # (the staging update() above already made the first), so the times equal the stepped loop's bit for bit
        ts = [self.t]
        for _ in range(n_steps - 1):
            ts.append(ts[-1] + dt)
        if n_steps > 1:
            self.prev_t = ts[-2]
        self.t = ts[-1]
        self._step = first_step + n_steps
        if self.save_history:
            self._hist_rows += n_steps
            self._t_hist.extend(ts)
        for ns in self.Neurons:
            last = (ns._hist_rows + n_steps - 1) % ns._hist_cap
            ns._hist_rows += n_steps
            ns._upd += n_steps
            ns._last_slot = last
            if ns.save_history:
                ns._t_hist.extend(ts)

    def _reserve_history(self, n_more):
        """Grow the ring (within history_bytes_limit) so that n_more further rows fit without wrapping."""
        import torch
        A = self.n_agents
        row_bytes = A * 8 * 4
        need = self._hist_rows + n_more
        if self._hist is None:
            cap = int(max(1, min(max(1024, need), self.history_bytes_limit // row_bytes)))
            self._hist = torch.empty((cap, A, 8), dtype=torch.float32, device=self.device)
            self._hist_cap = cap
        elif need > self._hist_cap and self._hist_rows <= self._hist_cap:
            cap = int(min(max(need, 2 * self._hist_cap), self.history_bytes_limit // row_bytes))
            if cap > self._hist_cap:
                new = torch.empty((cap, A, 8), dtype=torch.float32, device=self.device)
                new[: self._hist_cap].copy_(self._hist)
                self._hist, self._hist_cap = new, cap

    def last_collision_info(self):
        """Parity tap (needs update(_record_collisions=True)): per loop iteration
        ``wall_collisions`` masks (Environment.check_wall_collisions), first-hit wall
        indices (Agent.py:437) and the number of loop iterations."""
        self._flush_pending()
        if self._rec is None:
            raise RuntimeError("call update(_record_collisions=True) first")
        return {k: v.cpu().numpy() for k, v in self._rec.items()}

    # ------------------------------------------------------------------- history
    def _history_keys(self):
        return ["t", "pos", "distance_travelled", "vel", "rot_vel", "head_direction"]

    def _history_row_ptr(self):
        import torch
        A = self.n_agents
        row_bytes = A * 8 * 4
        if self._hist is None:
            cap = int(max(1, min(1024, self.history_bytes_limit // row_bytes)))
            self._hist = torch.empty((cap, A, 8), dtype=torch.float32, device=self.device)
            self._hist_cap = cap
        elif self._hist_rows == self._hist_cap and 2 * self._hist_cap * row_bytes <= self.history_bytes_limit:
            new = torch.empty((2 * self._hist_cap, A, 8), dtype=torch.float32, device=self.device)
            new[: self._hist_cap].copy_(self._hist)
            self._hist, self._hist_cap = new, 2 * self._hist_cap
        slot = self._hist_rows % self._hist_cap
        self._hist_rows += 1
        return self._hist.data_ptr() + slot * row_bytes

    @property
    def history(self):
        return self._history_view

    def get_history_arrays(self):
        """dict of arrays (Agent.py:1093-1102).  With n_agents > 1 the arrays carry an
        agent axis after the time axis.  If the ring wrapped, the most recent
        ``capacity`` steps are returned (``history_dropped`` counts the rest)."""
        self._flush_pending()
        if self._last_history_array_cache_time != (self.t, self._hist_rows):
            self._last_history_array_cache_time = (self.t, self._hist_rows)
            n = min(self._hist_rows, self._hist_cap)
            if n == 0:
                rows = np.zeros((0, self.n_agents, 8), dtype=np.float32)
            else:
                h = self._hist[: self._hist_cap]
                start = self._hist_rows % self._hist_cap if self._hist_rows > self._hist_cap else 0
                import torch
                idx = (torch.arange(n, device=self.device) + start) % self._hist_cap
                rows = h[idx].cpu().numpy()
            sq = (lambda x: x[:, 0]) if self.n_agents == 1 else (lambda x: x)
            self.history_dropped = self._hist_rows - n
            self._history_arrays = {
                "t": np.array(self._t_hist[len(self._t_hist) - n:]),
                "pos": sq(rows[:, :, 0:2]).astype(np.float64),
                "vel": sq(rows[:, :, 2:4]).astype(np.float64),
                "head_direction": sq(rows[:, :, 4:6]).astype(np.float64),
                "rot_vel": sq(rows[:, :, 6]).astype(np.float64),
                "distance_travelled": sq(rows[:, :, 7]).astype(np.float64),
            }
        return self._history_arrays

    def _history_maps(self, dx, neurons=None):
        """Occupancy counts (nx, ny) [and rate sums (nx*ny, ld)] of the history rings, binned on the device
        (riab_history_rate_maps); the last min(rows available) steps of both rings are used."""
        import torch
        self._flush_pending()
        env = self.Environment
        dx = env.dx * 5 if dx is None else dx
        ex = np.arange(env.extent[0], env.extent[1] + dx, dx)
        ey = np.arange(env.extent[2], env.extent[3] + dx, dx)
        n = min(self._hist_rows, self._hist_cap) if self._hist is not None else 0
        if neurons is not None:
            n = min(n, min(neurons._hist_rows, neurons._hist_cap) if neurons._hist is not None else 0)
        nx, ny = len(ex) - 1, len(ey) - 1
        count = torch.zeros(nx * ny, dtype=torch.int64, device=self.device)
        ssum = None
        if n > 0:
            h = _lib.HistoryView()
            h.agent_ring, h.agent_ring_rows = self._hist.data_ptr(), int(self._hist_cap)
            h.agent_row0 = int((self._hist_rows - n) % self._hist_cap)
            h.n_steps, h.n_agents = n, self.n_agents
            if neurons is not None:
                ssum = torch.zeros((nx * ny, neurons._ld()), dtype=torch.float64, device=self.device)
                h.rates_ring, h.rates_ring_rows = neurons._hist.data_ptr(), int(neurons._hist_cap)
                h.rates_row0 = int((neurons._hist_rows - n) % neurons._hist_cap)
                h.ld, h.n_cells = neurons._ld(), neurons.n
            exd = torch.as_tensor(ex, device=self.device)
            eyd = torch.as_tensor(ey, device=self.device)
            _lib.check(self._lib.riab_history_rate_maps(C.byref(h), exd.data_ptr(), len(ex), eyd.data_ptr(), len(ey),
                                                        ssum.data_ptr() if ssum is not None else None, count.data_ptr(),
                                                        self._stream()))
        count = count.cpu().numpy().astype(np.float64).reshape(nx, ny)          # exact: counts stay below 2^53
        if ssum is not None:
            ssum = ssum[:, : neurons.n].cpu().numpy().reshape(nx, ny, neurons.n)
        elif neurons is not None:
            ssum = np.zeros((nx, ny, neurons.n))
        return count, ssum

    def get_position_heatmap(self, dx=None):
        """The occupancy heat-map of Agent.plot_position_heatmap (Agent.py:950-957):
        ``utils.bin_data_for_histogramming(history positions, extent, dx)`` pooled over all agents, binned on the device.
        dx defaults to 5 x Environment.dx like the reference."""
        count, _ = self._history_maps(dx)
        return count.T[::-1, :]

    def reset_history(self):                                        # Agent.py:537-541
        self._flush_pending()
        self._hist_rows = 0
        self._t_hist = []
        self._last_history_array_cache_time = None

    def initialise_position_and_velocity(self):                     # Agent.py:523-535
        A = self.n_agents
        self.pos = self.Environment.sample_positions(n=A, method="random")
        direction = np.random.uniform(0, 2 * np.pi, size=A)
        self.velocity = self.speed_mean * np.stack((np.cos(direction), np.sin(direction)), axis=1)
        self.rotational_velocity = np.zeros(A)


def _make_prop(name):
    return property(lambda self: self._get_state(name), lambda self, v: self._set_state(name, v))


for _n in _STATE:
    setattr(Agent, _n, _make_prop(_n))

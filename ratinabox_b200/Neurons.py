"""Host mirror of ``ratinabox.Neurons``: PlaceCells, GridCells, the VectorCells (Boundary-, Object- and AgentVectorCells,
allocentric or egocentric, and their FieldOfView forms), RandomSpatialNeurons, HeadDirectionCells, VelocityCells,
SpeedCell and FeedForwardLayer.  ``update()`` and ``get_state()`` run on the GPU through libriab_b200 (C ABI:
include/riab_b200.h).

API parity (ratinabox/Neurons.py): ``Neurons(Agent, params)`` registers itself in
``Agent.Neurons`` (:111-112); ``update(**kwargs)`` (:145-171) refreshes
``firingrate`` (OU noise + ``get_state`` + optional spikes) and appends to
``history`` (``t``, ``firingrate``, ``spikes``; :681-687); ``get_state(evaluate_at=
"agent"|"all"|None, pos=...)`` returns ``(n_cells, n_pos)`` like the reference.
Parameter arrays (``place_cell_centres``, ``gridscales`` ...) are plain NumPy
attributes the user may overwrite or mutate between steps
(tests/test_advanced.py:59): they are re-packed when their bytes change.

With ``n_agents > 1`` ``firingrate`` is ``(n_agents, n)`` and history arrays are
``(steps, n_agents, n)``.  Rates are float32 on the device (history rows double as
the step's output: one write per rate).
"""
import copy
import ctypes as C
import warnings

import numpy as np

from . import _lib
from .Agent import _HistoryView


def _f64p(a):
    return a.ctypes.data_as(_lib.c_double_p)


class Neurons:
    default_params = {                                              # ratinabox/Neurons.py:90-99
        "n": 10,
        "name": "Neurons",
        "color": None,
        "noise_std": 0,
        "noise_coherence_time": 0.5,
        "min_fr": 0.0,
        "max_fr": 1.0,
        "save_history": True,
        # ---- batch-engine additions
        "save_spikes": True,          # the reference draws spikes whenever save_history is True (:681-684)
        "history_bytes_limit": 8 << 30,
    }
    _cells_kind = None

    def __init__(self, Agent, params={}):
        import torch
        self._lib = _lib.load()
        self.Agent = Agent
        self.Agent.Neurons.append(self)
        self._population_id = len(self.Agent.Neurons) - 1
        all_defaults = {}
        for cls in reversed(type(self).__mro__):                    # utils.collect_all_params, utils.py:821-874
            all_defaults.update(getattr(cls, "default_params", {}))
        unexpected = [k for k in params if k not in all_defaults]
        if unexpected:
            warnings.warn(f"Found {len(unexpected)} unexpected params key(s) while initializing "
                          f"{type(self).__name__}: {unexpected}")
        self.params = copy.deepcopy(all_defaults)
        self.params.update(params)
        for k, v in self.params.items():
            setattr(self, k, v)
        self.device = Agent.device
        self._torch = torch
        self._sig = None
        self._packed = None
        self._keep = []
        self._hist = None
        self._hist_cap = 0
        self._hist_rows = 0
        self._spk = None
        self._noise = None
        self._t_hist = []
        self._last_slot = None
        self._ring_min = 1         # 2 when a FeedForwardLayer reads this population one step late (its previous row)
        self._upd = 0             # updates of THIS population so far: keys its OU-noise / spike Philox streams
        self._history_view = _HistoryView(self)
        self._last_history_array_cache_time = None
        self._history_arrays = {}
        self._out = _lib.RatesOut()
        self._nz = _lib.NeuronNoise()
        self.colormap = "inferno"

    # ---------------------------------------------------------------- subclass API
    def _signature(self):
        raise NotImplementedError

    def _pack(self):
        """(re)build the device parameter block + C struct; returns the struct."""
        raise NotImplementedError

    def _cells(self):
        sig = self._signature()
        if sig != self._sig:
            self._cstruct = self._pack()
            self._sig = sig
        return self._cstruct

    def _cells_for_run(self):
        """The struct Agent.run hands to riab_run."""
        return self._cells()

    def _check_run(self):
        """Raise if riab_run cannot run this population (Agent.run calls it before it stages anything)."""

    def _rates_from_positions(self, pos_dev, n_pos, out):
        raise NotImplementedError

    # ------------------------------------------------------------------- helpers
    def _ld(self):
        return (self.n + 3) // 4 * 4

    def _upload(self, host):
        return self._torch.as_tensor(np.ascontiguousarray(host), device=self.device)

    def _row_buffers(self):
        """Next history row (rates [+ spikes]) on the device; grows / wraps like Agent's ring."""
        torch = self._torch
        A, ld = self.Agent.n_agents, self._ld()
        words = 4 * ((self.n + 127) // 128)           # 4 ballot words per 128 cells (riab_b200.h, riab_rates_out)
        row_bytes = A * ld * 4
        if self._hist is None:
            cap = int(max(1, min(256, self.history_bytes_limit // row_bytes))) if self.save_history else 1
            cap = max(cap, self._ring_min)
            self._hist = torch.empty((cap, A, ld), dtype=torch.float32, device=self.device)
            self._spk = torch.zeros((cap, A, words), dtype=torch.int32, device=self.device)
            self._hist_cap = cap
        elif self._hist_cap < self._ring_min:
            self._grow_ring(self._ring_min)
        elif self.save_history and self._hist_rows == self._hist_cap and 2 * self._hist_cap * row_bytes <= self.history_bytes_limit:
            cap = self._hist_cap
            new = torch.empty((2 * cap, A, ld), dtype=torch.float32, device=self.device)
            new[:cap].copy_(self._hist)
            spk = torch.zeros((2 * cap, A, words), dtype=torch.int32, device=self.device)
            spk[:cap].copy_(self._spk)
            self._hist, self._spk, self._hist_cap = new, spk, 2 * cap
        slot = self._hist_rows % self._hist_cap
        self._hist_rows += 1
        self._last_slot = slot
        # raw pointers of the slot (no tensor views on the per-step path)
        return (self._hist.data_ptr() + slot * row_bytes, self._spk.data_ptr() + slot * A * words * 4)

    def _reserve_history(self, n_more):
        """Grow the ring (within history_bytes_limit) so n_more further rows fit without wrapping if possible."""
        torch = self._torch
        A, ld = self.Agent.n_agents, self._ld()
        words = 4 * ((self.n + 127) // 128)           # 4 ballot words per 128 cells (riab_b200.h, riab_rates_out)
        row_bytes = A * ld * 4
        limit_rows = max(1, self.history_bytes_limit // row_bytes)
        need = self._hist_rows + n_more if self.save_history else 1
        if self._hist is None:
            cap = int(max(1, min(max(256, need), limit_rows))) if self.save_history else 1
            cap = max(cap, self._ring_min)
            self._hist = torch.empty((cap, A, ld), dtype=torch.float32, device=self.device)
            self._spk = torch.zeros((cap, A, words), dtype=torch.int32, device=self.device)
            self._hist_cap = cap
        elif self._hist_cap < self._ring_min:
            self._grow_ring(self._ring_min)
        elif need > self._hist_cap and self._hist_rows <= self._hist_cap:
            cap = int(min(max(need, 2 * self._hist_cap), limit_rows))
            if cap > self._hist_cap:
                new = torch.empty((cap, A, ld), dtype=torch.float32, device=self.device)
                new[: self._hist_cap].copy_(self._hist)
                spk = torch.zeros((cap, A, words), dtype=torch.int32, device=self.device)
                spk[: self._hist_cap].copy_(self._spk)
                self._hist, self._spk, self._hist_cap = new, spk, cap

    def _grow_ring(self, cap):
        """Re-allocate the rings with `cap` rows; rows keep their slot index."""
        torch = self._torch
        new = torch.empty((cap,) + tuple(self._hist.shape[1:]), dtype=torch.float32, device=self.device)
        new[: self._hist_cap].copy_(self._hist)
        spk = torch.zeros((cap,) + tuple(self._spk.shape[1:]), dtype=torch.int32, device=self.device)
        spk[: self._hist_cap].copy_(self._spk)
        self._hist, self._spk, self._hist_cap = new, spk, cap

    # -------------------------------------------------------------------- update
    def _fill_out_structs(self, row, spk):
        ag = self.Agent
        out, nz = self._out, self._nz
        out.rates_row = row
        out.ld = self._ld()
        want_spikes = bool(self.save_history and self.save_spikes)
        out.spikes_row = spk if (want_spikes and spk is not None) else None
        out.noise_state = None
        if self.noise_std != 0:
            if self._noise is None:
                self._noise = self._torch.zeros((ag.n_agents, self._ld()), dtype=self._torch.float32, device=self.device)
            out.noise_state = self._noise.data_ptr()
        out.bvc_scratch = self._scratch_ptr(ag.n_agents)
        nz.noise_std = float(self.noise_std)
        nz.noise_coherence_time = float(self.noise_coherence_time)
        nz.dt = float(ag.dt)
        nz.seed = int(ag.seed) & 0xFFFFFFFFFFFFFFFF
        nz.step = self._upd
        nz.id_offset = int(ag.id_offset)
        nz.population_id = self._population_id
        return out, nz

    def update(self, **kwargs):
        """Neurons.update (ratinabox/Neurons.py:145-171)."""
        ag = self.Agent
        cells = self._cells()
        ag._sync_user_writes()                 # in-place edits of Ag.pos etc. since they were read
        saved = (self._hist_rows, self._last_slot)
        row, spk = self._row_buffers()
        out, nz = self._fill_out_structs(row, spk)
        fused = ag._take_pending()
        try:
            if fused:
                _lib.check(self._lib.riab_step_fused(C.byref(ag._agents_c), C.byref(ag._env_struct()), C.byref(ag._mp),
                                                     C.byref(ag._io), self._cells_kind, C.byref(cells), C.byref(nz),
                                                     C.byref(out), ag._stream()))
            else:
                self._update_unfused(cells, out, nz)
        except Exception:
            # the library refused the call (validation): nothing ran -- keep the queued motion step and the ring as they were
            self._hist_rows, self._last_slot = saved
            if fused:
                ag._pending = True
            raise
        self._upd += 1
        if self.save_history:
            self._t_hist.append(ag.t)

    def _update_unfused(self, cells, out, nz):
        """Rates for the agents' current positions (no queued motion step to fuse with)."""
        ag = self.Agent
        _lib.check(self._lib.riab_neurons_update(C.byref(ag._agents_c), C.byref(ag._env_struct()), self._cells_kind,
                                                 C.byref(cells), C.byref(nz), C.byref(out), ag._stream()))

    def _scratch_ptr(self, n):
        return None

    # ----------------------------------------------------------------- get_state
    _zeroed_state = False         # get_state's rates start as zeros (for populations whose kernel may not run)

    def get_state(self, evaluate_at="agent", **kwargs):
        """(n_cells, n_pos) firing rates, float64 NumPy (pass ``return_tensor=True``
        for the (n_pos, n_cells) float32 device tensor)."""
        torch = self._torch
        self._cells()
        pos_dev = self._positions(evaluate_at, kwargs)
        n_pos = int(pos_dev.shape[0])
        inputs = self._kernel_inputs(evaluate_at, n_pos, kwargs)
        out = (torch.zeros if self._zeroed_state else torch.empty)((n_pos, self._ld()), dtype=torch.float32,
                                                                   device=self.device)
        if n_pos:
            self._rates_from_positions(pos_dev, n_pos, out, **inputs)
        return self._result(out, kwargs.get("return_tensor", False))

    def _agent_state(self):
        """The Agent's device state as it stands now: its queued motion step run, the user's in-place edits of its
        arrays (``Ag.pos``, ``Ag.head_direction`` ...) uploaded."""
        self.Agent._flush_pending()
        self.Agent._sync_user_writes()
        return self.Agent._s

    def _positions(self, evaluate_at, kwargs):
        """get_state's points as a (n_pos, 2) float64 device tensor: the agents' positions at "agent", the discretised
        environment at "all", else the ``pos`` kwarg."""
        if evaluate_at == "agent":
            return self._agent_state()["pos"]
        return self._rows(self.Agent.Environment.flattened_discrete_coords if evaluate_at == "all" else kwargs["pos"])

    def _n_pos(self, evaluate_at, kwargs, default):
        """How many points get_state evaluates away from the agents, for populations that need only the count: the
        discretised environment's for "all", the ``pos`` kwarg's rows, else ``default``."""
        if evaluate_at == "all":
            return self.Agent.Environment.flattened_discrete_coords.shape[0]
        if "pos" in kwargs:
            pos = kwargs["pos"]
            return int((pos if isinstance(pos, self._torch.Tensor) else np.asarray(pos)).reshape(-1, 2).shape[0])
        return default

    def _rows(self, x, n=None):
        """``x`` (NumPy, a list, or a torch tensor on any device) as a C-contiguous (k, 2) float64 device tensor; with
        ``n``, broadcast to (n, 2)."""
        torch = self._torch
        if isinstance(x, torch.Tensor):
            x = x.to(device=self.device, dtype=torch.float64).reshape(-1, 2)
            return (x if n is None else x.expand(n, 2)).contiguous()
        x = np.asarray(x, dtype=np.float64).reshape(-1, 2)
        if n is not None:
            x = np.array(np.broadcast_to(x, (n, 2)), order="C")          # own, writable copy
        return torch.as_tensor(np.ascontiguousarray(x), device=self.device)

    def _kernel_inputs(self, evaluate_at, n_pos, kwargs):
        """Keyword arguments of ``_rates_from_positions`` besides the positions (head directions, partner positions)."""
        return {}

    def _result(self, out, return_tensor):
        """get_state's value from its (n_pos, ld) float32 rates: the (n_pos, n) device view with ``return_tensor``, else
        the (n, n_pos) float64 NumPy array."""
        if return_tensor:
            return out[:, : self.n]
        return out[:, : self.n].T.contiguous().cpu().numpy().astype(np.float64)

    def get_head_direction_averaged_state(self, evaluate_at="agent", angular_resolution_degrees=10, **kwargs):
        """Neurons.get_head_direction_averaged_state (ratinabox/Neurons.py:176-192): the mean of ``get_state`` over the
        head directions at ``np.linspace(0, 2 pi, int(360 / angular_resolution_degrees))`` (0 and 2 pi both count), for
        head-direction-tuned populations (HeadDirectionCells, egocentric vector cells); the others ignore the head
        direction.  The rates are summed on the device in float64.  Returns (n, n_pos) float64."""
        kwargs.pop("return_tensor", None)
        n_angles = int(360 / angular_resolution_degrees)
        acc = None
        for ang in np.linspace(0, 2 * np.pi, n_angles):
            r = self.get_state(evaluate_at=evaluate_at, head_direction=np.array([np.cos(ang), np.sin(ang)]),
                               return_tensor=True, **kwargs)
            acc = r.to(self._torch.float64) if acc is None else acc.add_(r)
        return (acc / n_angles).T.contiguous().cpu().numpy()

    # ------------------------------------------------------------------ firingrate
    @property
    def firingrate(self):
        if self._last_slot is None:
            return np.zeros(self.n)
        r = self._hist[self._last_slot][:, : self.n].cpu().numpy().astype(np.float64)
        return r[0] if self.Agent.n_agents == 1 else r

    # --------------------------------------------------------------------- history
    def _history_keys(self):
        return ["t", "firingrate", "spikes"]

    @property
    def history(self):
        return self._history_view

    def get_history_arrays(self):                                   # Neurons.py:812-821
        key = (self.Agent.t, self._hist_rows)
        if self._last_history_array_cache_time != key:
            self._last_history_array_cache_time = key
            torch = self._torch
            n = min(self._hist_rows, self._hist_cap) if self.save_history else 0
            A = self.Agent.n_agents
            if n == 0:
                fr = np.zeros((0, A, self.n))
                sp = np.zeros((0, A, self.n), dtype=bool)
            else:
                start = self._hist_rows % self._hist_cap if self._hist_rows > self._hist_cap else 0
                idx = (torch.arange(n, device=self.device) + start) % self._hist_cap
                fr = self._hist[idx][:, :, : self.n].cpu().numpy().astype(np.float64)
                words = self._spk[idx].cpu().numpy().view(np.uint32)
                # bit L of word 4B+i = cell 128B + 4L + i  (one warp ballot per cell slot i)
                bits = np.unpackbits(words.view(np.uint8), axis=-1, bitorder="little")
                bits = bits.reshape(n, A, -1, 4, 32).transpose(0, 1, 2, 4, 3).reshape(n, A, -1)
                sp = bits[:, :, : self.n].astype(bool)
            if A == 1:
                fr, sp = fr[:, 0], sp[:, 0]
            self.history_dropped = self._hist_rows - n
            self._history_arrays = {"t": np.array(self._t_hist[len(self._t_hist) - n:]), "firingrate": fr, "spikes": sp}
        return self._history_arrays

    def get_history_rate_maps(self, dx=None, return_zero_bins=False):
        """Rate maps from the history, the data of ``plot_rate_map(method="history")`` (Neurons.py:470-490): for every
        cell ``utils.bin_data_for_histogramming(pos, extent, dx, weights=rate, norm_by_bincount=True)`` over the history of
        ALL agents, binned on the device (riab_history_rate_maps).  Returns (n_cells, ny, nx) [and the empty-bin mask]."""
        count, ssum = self.Agent._history_maps(dx, neurons=self)
        zero = (count == 0)
        c = count.copy()
        c[zero] = 1
        maps = (ssum / c[:, :, None]).transpose(2, 1, 0)[:, ::-1, :]            # per cell: heatmap.T[::-1, :]
        if return_zero_bins:
            return maps, zero.T[::-1, :]
        return maps

    def reset_history(self):                                        # Neurons.py:689-692
        self._hist_rows = 0
        self._t_hist = []
        self._last_history_array_cache_time = None


# =============================================================================
class PlaceCells(Neurons):
    default_params = {                                              # ratinabox/Neurons.py:857-867
        "n": 10,
        "name": "PlaceCells",
        "description": "gaussian",
        "widths": 0.20,
        "place_cell_centres": None,
        "wall_geometry": "geodesic",
        "min_fr": 0,
        "max_fr": 1,
    }
    _cells_kind = _lib.CELLS_PLACE

    def __init__(self, Agent, params={}):
        params = dict(params)
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        env = Agent.Environment
        if p["place_cell_centres"] is None:                         # Neurons.py:881-901
            p["place_cell_centres"] = env.sample_positions(n=p["n"], method="uniform_jitter")
        elif type(p["place_cell_centres"]) is str:
            if p["place_cell_centres"] in ["random", "uniform", "uniform_jitter"]:
                p["place_cell_centres"] = env.sample_positions(n=p["n"], method=p["place_cell_centres"])
            else:
                raise ValueError("self.params['place_cell_centres'] must be None, an array of locations or one of "
                                 "the instructions ['random', 'uniform', 'uniform_jitter']")
        else:
            p["place_cell_centres"] = np.array(p["place_cell_centres"], dtype=float)
            p["n"] = p["place_cell_centres"].shape[0]
        params["place_cell_centres"], params["n"] = p["place_cell_centres"], p["n"]
        super().__init__(Agent, params)
        self.place_cell_widths = self.widths * np.ones(self.n)
        if self.description not in _lib.PC_DESCRIPTIONS:
            raise ValueError(f"unknown PlaceCells description {self.description!r}")
        if self.wall_geometry in ("line_of_sight", "geodesic") and env.boundary_conditions == "periodic":   # Neurons.py:907-921
            print(f"{self.wall_geometry} wall geometry only possible in 2D when the boundary conditions are solid. "
                  "Using 'euclidean' instead.")
            self.wall_geometry = "euclidean"
        if (self.wall_geometry == "geodesic") and (len(env.walls) > 5):   # Neurons.py:922-928
            print("'geodesic' wall geometry only supported for enivironments with 1 additional wall "
                  "(4 bounding walls + 1 additional). Sorry. Using 'line_of_sight' instead.")
            self.wall_geometry = "line_of_sight"

    def _effective_geometry(self):
        n_inner = len(self.Agent.Environment.walls) - self.Agent.Environment.los_skip
        if self.wall_geometry not in _lib.WALL_GEOMETRIES:
            raise ValueError(f"unknown wall_geometry {self.wall_geometry!r}")
        if self.wall_geometry == "geodesic":
            if self.Agent.Environment.is_polygonal:
                raise NotImplementedError("geodesic distances in polygon / holed environments are outside the CUDA hot path")
            assert n_inner <= 1, ("unfortunately geodesic geometry is only defined in closed rooms with one "
                                  "additional wall (Environment.py:736-739)")
        if n_inner == 0:
            return "euclidean"          # line_of_sight / geodesic without inner walls are plain distances
        return self.wall_geometry

    def _signature(self):
        env = self.Agent.Environment
        return (np.ascontiguousarray(self.place_cell_centres, dtype=np.float64).tobytes(),
                np.ascontiguousarray(self.place_cell_widths, dtype=np.float64).tobytes(),
                env._walls_signature(), self.description, self.wall_geometry, float(self.min_fr), float(self.max_fr),
                float(self.widths) if np.isscalar(self.widths) else None, self.n)

    def _pack(self):
        env = self.Agent.Environment
        centres = np.ascontiguousarray(self.place_cell_centres, dtype=np.float64).reshape(-1, 2)
        widths = np.ascontiguousarray(self.place_cell_widths, dtype=np.float64).reshape(-1)
        self.n = centres.shape[0]
        assert widths.shape[0] == self.n
        geom = _lib.WALL_GEOMETRIES[self._effective_geometry()]
        walls = np.ascontiguousarray(env.walls, dtype=np.float64)
        n_inner = 0 if geom == 0 else walls.shape[0] - env.los_skip
        c = _lib.PlaceCells()
        nfl = self._lib.riab_place_pack_floats(self.n, n_inner)
        host = np.zeros(nfl, dtype=np.float32)
        ext = np.ascontiguousarray(env.extent, dtype=np.float64)
        _lib.check(self._lib.riab_place_pack(_f64p(centres), _f64p(widths), self.n, _f64p(walls), walls.shape[0],
                                             env.los_skip, _f64p(ext), geom, C.byref(c),
                                             host.ctypes.data_as(_lib.c_float_p)))
        if geom == _lib.WALL_GEOMETRIES["geodesic"] and n_inner == 1 and c.ep_valid == 0:
            # the reference reduces the detours via the wall's ends inside the box with np.amin, which raises on an
            # empty list at every rate evaluation (Environment.py:769-773)
            raise ValueError("zero-size array to reduction operation minimum which has no identity: geodesic distances "
                             "need an end of the additional wall strictly inside the environment")
        self._packed = self._upload(host)
        self._centres_dev = self._upload(centres)
        c.n_cells, c.description, c.wall_geometry = self.n, _lib.PC_DESCRIPTIONS[self.description], geom
        c.min_fr, c.max_fr = float(self.min_fr), float(self.max_fr)
        c.top_hat_width = float(self.widths) if np.isscalar(self.widths) else float(np.asarray(self.widths).reshape(-1)[0])
        c.packed_dev, c.centres_dev = self._packed.data_ptr(), self._centres_dev.data_ptr()
        return c

    def _check_run(self):
        self._cells()                   # _pack's geodesic check raises before Agent.run stages anything

    def _rates_from_positions(self, pos_dev, n_pos, out):
        ag = self.Agent
        _lib.check(self._lib.riab_place_rates(pos_dev.data_ptr(), n_pos, C.byref(ag._env_struct()),
                                              C.byref(self._cells()), out.data_ptr(), out.stride(0), ag._stream()))


# =============================================================================
class GridCells(Neurons):
    default_params = {                                              # ratinabox/Neurons.py:1055-1068
        "n": 30,
        "gridscale_distribution": "modules",
        "gridscale": (0.3, 0.5, 0.8),
        "orientation_distribution": "modules",
        "orientation": (0, 0.1, 0.2),
        "phase_offset_distribution": "uniform",
        "phase_offset": (0, 2 * np.pi),
        "description": "rectified_cosines",
        "width_ratio": 4 / (3 * np.sqrt(3)),
        "min_fr": 0,
        "max_fr": 1,
        "name": "GridCells",
    }
    _cells_kind = _lib.CELLS_GRID

    def __init__(self, Agent, params={}):
        from .utils import distribution_sampler, rotate
        params = dict(params)
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        if p["description"] in ("three_rectified_cosines", "three_shifted_cosines"):   # Neurons.py:1091-1095
            p["description"] = p["description"][6:]
            params["description"] = p["description"]
        if type(p["gridscale"]) in (list, np.ndarray):              # Neurons.py:1098-1113
            gridscales = np.array(p["gridscale"], dtype=float)
            p["n"] = len(gridscales)
        else:
            gridscales = distribution_sampler(p["gridscale_distribution"], p["gridscale"], (p["n"],))
        params["n"] = p["n"]
        super().__init__(Agent, params)
        self.gridscales = gridscales
        if type(self.params["phase_offset"]) in (list, np.ndarray) and np.array(self.params["phase_offset"]).ndim == 2:
            self.phase_offsets = np.array(self.params["phase_offset"], dtype=float)
            assert len(self.phase_offsets) == self.n, "number of phase offsets supplied incompatible with number of neurons"
        else:
            if self.params["phase_offset_distribution"] == "grid":
                raise NotImplementedError("phase_offset_distribution='grid' is host set-up outside the hot path")
            self.phase_offsets = distribution_sampler(self.params["phase_offset_distribution"],
                                                      self.params["phase_offset"], (self.n, 2))
        if type(self.params["orientation"]) in (list, np.ndarray):
            self.orientations = np.array(self.params["orientation"], dtype=float)
            assert len(self.orientations) == self.n, "number of orientations supplied incompatible with number of neurons"
        else:
            self.orientations = distribution_sampler(self.params["orientation_distribution"],
                                                     self.params["orientation"], (self.n,))
        w = []
        for i in range(self.n):                                     # Neurons.py:1154-1161
            w1 = rotate(np.array([1, 0]), self.orientations[i])
            w.append(np.array([w1, rotate(w1, np.pi / 3), rotate(w1, 2 * np.pi / 3)]))
        self.w = np.array(w)
        if self.description == "rectified_cosines":
            assert self.width_ratio > 0 and self.width_ratio <= 1, "width_ratio must be between 0 and 1"
        if self.description not in _lib.GC_DESCRIPTIONS:
            raise ValueError(f"unknown GridCells description {self.description!r}")

    def _signature(self):
        return (np.ascontiguousarray(self.gridscales, dtype=np.float64).tobytes(),
                np.ascontiguousarray(self.phase_offsets, dtype=np.float64).tobytes(),
                np.ascontiguousarray(self.w, dtype=np.float64).tobytes(),
                self.description, float(self.width_ratio), float(self.min_fr), float(self.max_fr))

    def _pack(self):
        env = self.Agent.Environment
        gs = np.ascontiguousarray(self.gridscales, dtype=np.float64).reshape(-1)
        ph = np.ascontiguousarray(self.phase_offsets, dtype=np.float64).reshape(-1, 2)
        w = np.ascontiguousarray(self.w, dtype=np.float64).reshape(-1, 3, 2)
        self.n = gs.shape[0]
        c = _lib.GridCells()
        host = np.zeros(self._lib.riab_grid_pack_floats(self.n), dtype=np.float32)
        ext = np.ascontiguousarray(env.extent, dtype=np.float64)
        _lib.check(self._lib.riab_grid_pack(_f64p(gs), _f64p(ph), _f64p(w), self.n, _f64p(ext), C.byref(c),
                                            host.ctypes.data_as(_lib.c_float_p)))
        self._packed = self._upload(host)
        c.n_cells, c.description = self.n, _lib.GC_DESCRIPTIONS[self.description]
        c.width_ratio, c.min_fr, c.max_fr = float(self.width_ratio), float(self.min_fr), float(self.max_fr)
        c.packed_dev = self._packed.data_ptr()
        return c

    def _rates_from_positions(self, pos_dev, n_pos, out):
        ag = self.Agent
        _lib.check(self._lib.riab_grid_rates(pos_dev.data_ptr(), n_pos, C.byref(ag._env_struct()),
                                             C.byref(self._cells()), out.data_ptr(), out.stride(0), ag._stream()))


# =============================================================================
class VectorCells(Neurons):
    """ratinabox.VectorCells (Neurons.py:1259-1437), the parent of BoundaryVectorCells, ObjectVectorCells and
    AgentVectorCells: their shared tuning (``tuning_distances``, ``tuning_angles``, ``sigma_distances``, ``sigma_angles``
    from ``cell_arrangement``) and the head directions egocentric cells read in get_state."""
    default_params = {                                              # ratinabox/Neurons.py:1303-1316
        "n": 10,
        "reference_frame": "allocentric",
        "cell_arrangement": "random",
        "tuning_distance_distribution": "uniform",
        "tuning_distance": (0.05, 0.3),
        "sigma_distance_distribution": "diverging",
        "sigma_distance": (0.08, 12),
        "tuning_angle_distribution": "uniform",
        "tuning_angle": (0.0, 360),
        "angular_spread_distribution": "uniform",
        "angular_spread": (10, 30),
    }

    def _init_vector_tuning(self):
        """VectorCells.set_tuning_parameters (Neurons.py:1388-1437): tuning_distances / tuning_angles /
        sigma_distances / sigma_angles from ``cell_arrangement``."""
        from .utils import (create_random_assembly, create_uniform_radial_assembly,
                            create_diverging_radial_assembly)
        if self.reference_frame not in ("allocentric", "egocentric"):
            raise ValueError(f"unknown reference_frame {self.reference_frame!r}")
        arr = self.cell_arrangement                                   # VectorCells.set_tuning_parameters, Neurons.py:1388-1437
        if callable(arr):
            tuning = arr(**self.params)
        elif arr is None or (isinstance(arr, str) and arr[:6] == "random"):
            tuning = create_random_assembly(**self.params)
        elif arr == "uniform_manifold":
            tuning = create_uniform_radial_assembly(**self.params)
        elif arr == "diverging_manifold":
            tuning = create_diverging_radial_assembly(**self.params)
        else:
            raise ValueError("cell_arrangement must be either 'uniform_manifold' or 'diverging_manifold' or a function")
        (self.tuning_distances, self.tuning_angles, self.sigma_distances,
         self.sigma_angles) = (np.array(x, dtype=float) for x in tuning)
        assert len(self.tuning_distances) == len(self.tuning_angles) == len(self.sigma_distances) == len(self.sigma_angles), \
            "All manifold tuning parameters must be of the same length"
        self.n = len(self.tuning_distances)

    def _vector_tuning(self):
        """The four tuning arrays as contiguous float64 vectors, in the packers' order."""
        return [np.ascontiguousarray(a, dtype=np.float64).reshape(-1) for a in (
            self.tuning_distances, self.tuning_angles, self.sigma_distances, self.sigma_angles)]

    def _kernel_inputs(self, evaluate_at, n_pos, kwargs):
        if self.reference_frame != "egocentric":
            return {}
        return {"head_dir": self._head_directions(evaluate_at, n_pos, kwargs)}

    def _head_directions(self, evaluate_at, n_pos, kwargs):
        """The (n_pos, 2) float64 device head directions of egocentric cells: the agents' at "agent", else the
        ``head_direction`` kwarg (one vector for all positions, or one per position), the deprecated ``vel``, or [1,0]
        with the reference's warning (Neurons.py:1693-1706)."""
        if evaluate_at == "agent":
            return self._agent_state()["head_direction"]
        if "head_direction" in kwargs:
            hd = kwargs["head_direction"]
        elif "vel" in kwargs:
            warnings.warn("'vel' kwarg deprecated in favour of 'head_direction'")
            hd = kwargs["vel"]
        else:
            warnings.warn(self._egocentric_warning)
            hd = [1.0, 0.0]
        return self._rows(hd, n_pos)


class BoundaryVectorCells(VectorCells):
    default_params = {                                              # ratinabox/Neurons.py:1549-1555
        "n": 10,
        "name": "BoundaryVectorCells",
        "dtheta": 2,
        "max_fr": 1.0,
        "min_fr": 0.0,
    }
    _cells_kind = _lib.CELLS_BVC
    _egocentric_warning = "BVCs in egocentric plane require a head direction vector but none was passed. Using [1,0]"

    def __init__(self, Agent, params={}):
        from .utils import rotate
        super().__init__(Agent, params)
        assert self.Agent.Environment.boundary_conditions == "solid", \
            "boundary cells only possible with solid boundary conditions"      # Neurons.py:1580-1582
        self._init_vector_tuning()
        test_direction = np.array([1, 0])                           # Neurons.py:1584-1596 (duplicated-0 quirk kept)
        dirs, angs = [test_direction], [0]
        self.n_test_angles = int(360 / self.dtheta)
        for i in range(self.n_test_angles - 1):
            dirs.append(rotate(test_direction, 2 * np.pi * i * self.dtheta / 360))
            angs.append(2 * np.pi * i * self.dtheta / 360)
        self.test_directions = np.array(dirs, dtype=float)
        self.test_angles = np.array(angs, dtype=float)
        kappa = 1 / (self.sigma_angles.reshape(-1, 1) ** 2)         # Neurons.py:1599-1604
        self.cell_fr_norm = (np.exp(kappa * np.cos(self.test_angles.reshape(1, -1))) * (1 / np.exp(kappa))).sum(axis=1)
        self._scratch = None

    def _signature(self):
        return tuple(np.ascontiguousarray(a, dtype=np.float64).tobytes() for a in (
            *self._vector_tuning(), self.test_angles, self.test_directions)) + (
            float(self.min_fr), float(self.max_fr), self.reference_frame)

    def _pack(self):
        arrs = self._vector_tuning()
        self.n = arrs[0].shape[0]
        angs = np.ascontiguousarray(self.test_angles, dtype=np.float64)
        T = angs.shape[0]
        c = _lib.BvcCells()
        host = np.zeros(self._lib.riab_bvc_pack_floats(self.n, T), dtype=np.float32)
        _lib.check(self._lib.riab_bvc_pack(*[_f64p(a) for a in arrs], self.n, _f64p(angs), T, C.byref(c),
                                           host.ctypes.data_as(_lib.c_float_p)))
        self._packed = self._upload(host)
        self._dirs_dev = self._upload(np.ascontiguousarray(self.test_directions, dtype=np.float64))
        c.n_cells, c.n_test_angles = self.n, T
        c.egocentric = 1 if self.reference_frame == "egocentric" else 0
        c.min_fr, c.max_fr = float(self.min_fr), float(self.max_fr)
        c.packed_dev, c.test_dirs_dev = self._packed.data_ptr(), self._dirs_dev.data_ptr()
        return c

    def _scratch_for(self, n):
        need = self._lib.riab_bvc_scratch_floats(n, len(self.test_angles))
        if self._scratch is None or self._scratch.numel() < need:
            self._scratch = self._torch.empty(need, dtype=self._torch.float32, device=self.device)
        return self._scratch

    def _scratch_ptr(self, n):
        return self._scratch_for(n).data_ptr()

    def _rates_from_positions(self, pos_dev, n_pos, out, first_wall=None, head_dir=None):
        ag = self.Agent
        scratch = self._scratch_for(n_pos)
        _lib.check(self._lib.riab_bvc_rates(pos_dev.data_ptr(), n_pos, C.byref(ag._env_struct()),
                                            C.byref(self._cells()), scratch.data_ptr(),
                                            first_wall.data_ptr() if first_wall is not None else None,
                                            head_dir.data_ptr() if head_dir is not None else None,
                                            out.data_ptr(), out.stride(0), ag._stream()))


class FieldOfViewBVCs(BoundaryVectorCells):
    """Egocentric BVCs tiling the agent's field of view (ratinabox/Neurons.py:1847-1887)."""
    default_params = {
        "distance_range": [0.02, 0.4],
        "angle_range": [0, 75],
        "spatial_resolution": 0.02,
        "cell_arrangement": "diverging_manifold",
        "beta": 5,
        "color": [0.3, 0.3, 0.3, 1],
    }

    def __init__(self, Agent, params={}):
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        p["reference_frame"] = "egocentric"
        assert p["cell_arrangement"] is not None, "cell_arrangement must be set for FoV Neurons"
        super().__init__(Agent, p)


class ObjectVectorCells(VectorCells):
    """ratinabox.ObjectVectorCells (Neurons.py:1892-2113): vector cells tuned to the objects of the Environment.
    Same tuning machinery as the other VectorCells (cell_arrangement, tuning_distance, ...); each cell responds to the
    objects of ONE type (``object_tuning_type``: "random", an int, or one int per cell).  The rates are evaluated by
    ``riab_ovc_*`` (csrc/riab_ovc.cuh): exact float64 agent-object geometry per agent, float32 tuning per cell."""
    default_params = {
        "n": 10,
        "name": "ObjectVectorCell",
        "walls_occlude": True,          # objects behind walls cannot be seen
        "object_tuning_type": "random",
    }
    _cells_kind = _lib.CELLS_OVC

    def __init__(self, Agent, params={}):
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        env = Agent.Environment
        if len(env.objects["objects"]) == 0:                       # Neurons.py:1921-1923
            raise RuntimeError(f"Cannot initialize {p['name']}, as there are no objects in the environment.")
        if len(env.objects["objects"]) > _lib.MAX_OBJECTS:
            raise NotImplementedError(f"at most {_lib.MAX_OBJECTS} objects per environment on the CUDA path")
        super().__init__(Agent, p)
        self._init_vector_tuning()
        self.object_locations = env.objects["objects"]
        self.tuning_types = None
        self.set_tuning_types(self.object_tuning_type)
        self.wall_geometry = "line_of_sight" if self.walls_occlude == True else "euclidean"      # Neurons.py:1937-1940

    def set_tuning_types(self, tuning_types=None):                  # Neurons.py:1962-1986
        if isinstance(tuning_types, str) and tuning_types == "random":
            self.object_types = self.Agent.Environment.objects["object_types"]
            self.tuning_types = np.random.choice(np.unique(self.object_types), replace=True, size=(self.n,))
        else:
            if isinstance(tuning_types, (int, np.integer)):
                tuning_types = np.repeat(tuning_types, self.n)
            elif isinstance(tuning_types, list):
                tuning_types = np.array(tuning_types)
            assert isinstance(tuning_types, np.ndarray), "tuning_types must be an integer, list or numpy array"
            assert tuning_types.shape[0] == self.n, \
                f"Tuning types must be a vector of length of the number of neurons: ({self.n},)"
            self.tuning_types = tuning_types

    def _signature(self):
        env = self.Agent.Environment
        return tuple(np.ascontiguousarray(a, dtype=np.float64).tobytes() for a in (
            *self._vector_tuning(), np.asarray(self.tuning_types, dtype=np.float64), env.objects["objects"],
            np.asarray(env.objects["object_types"], dtype=np.float64))) + (
            float(self.min_fr), float(self.max_fr), self.reference_frame, self.wall_geometry)

    def _pack(self):
        env = self.Agent.Environment
        arrs = self._vector_tuning()
        self.n = arrs[0].shape[0]
        types = np.ascontiguousarray(self.tuning_types, dtype=np.int32).reshape(-1)
        assert types.shape[0] == self.n
        objs = np.ascontiguousarray(env.objects["objects"], dtype=np.float64).reshape(-1, 2)
        otypes = np.asarray(env.objects["object_types"], dtype=np.int32).reshape(-1)
        if len(objs) > _lib.MAX_OBJECTS:
            raise NotImplementedError(f"at most {_lib.MAX_OBJECTS} objects per environment on the CUDA path")
        c = _lib.OvcCells()
        host = np.zeros(self._lib.riab_ovc_pack_floats(self.n), dtype=np.float32)
        _lib.check(self._lib.riab_ovc_pack(*[_f64p(a) for a in arrs], types.ctypes.data_as(C.POINTER(C.c_int32)), self.n,
                                           C.byref(c), host.ctypes.data_as(_lib.c_float_p)))
        self._packed = self._upload(host)
        c.n_cells, c.n_objects = self.n, len(objs)
        for o in range(len(objs)):
            c.objects[2 * o], c.objects[2 * o + 1] = float(objs[o, 0]), float(objs[o, 1])
            c.object_types[o] = int(otypes[o])
        c.walls_occlude = 1 if self.wall_geometry == "line_of_sight" else 0
        c.egocentric = 1 if self.reference_frame == "egocentric" else 0
        c.min_fr, c.max_fr = float(self.min_fr), float(self.max_fr)
        c.packed_dev = self._packed.data_ptr()
        return c

    def _rates_from_positions(self, pos_dev, n_pos, out, head_dir=None):
        ag = self.Agent
        _lib.check(self._lib.riab_ovc_rates(pos_dev.data_ptr(), n_pos, C.byref(ag._env_struct()), C.byref(self._cells()),
                                            head_dir.data_ptr() if head_dir is not None else None,
                                            out.data_ptr(), out.stride(0), ag._stream()))

    _egocentric_warning = "OVCs in egocentric plane require a head direction vector but none was passed. Using [1,0]"


class FieldOfViewOVCs(ObjectVectorCells):
    """Egocentric ObjectVectorCells tiling the agent's field of view (ratinabox/Neurons.py:2116-2160)."""
    default_params = {
        "distance_range": [0.02, 0.4],
        "angle_range": [0, 75],
        "spatial_resolution": 0.02,
        "beta": 5,
        "cell_arrangement": "diverging_manifold",
        "object_tuning_type": None,
    }

    def __init__(self, Agent, params={}):
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        if p["object_tuning_type"] is None:
            warnings.warn("For FieldOfViewOVCs you must specify the object type they are selective for with the "
                          "'object_tuning_type' parameter. This can be 'random' (each cell in the field of view chooses a "
                          "random object type) or any integer (all cells have the same preference for this type). For now "
                          "defaulting to params['object_tuning_type'] = 0.")
            p["object_tuning_type"] = 0
        p["reference_frame"] = "egocentric"
        assert p["cell_arrangement"] is not None, "cell_arrangement must be set for FOV Neurons"
        super().__init__(Agent, p)


class AgentVectorCells(VectorCells):
    """ratinabox.AgentVectorCells (Neurons.py:2151-2320): vector cells tuned to another Agent, ``tuning_type_agent`` (the
    ``Other_Agent`` argument).  A cell fires ``gaussian(d) * von_mises(bearing)`` of the vector from the agent to its
    partner, with the other VectorCells' tuning machinery (cell_arrangement, tuning_distance, ...); ``walls_occlude`` takes
    the line-of-sight distance (1000 behind an inner wall).

    Pairing: row i of ``Agent`` sees row i of ``Other_Agent`` (``Other_Agent.n_agents == Agent.n_agents``, and under
    sharding the same ``id_offset``), or every row sees the single agent of an ``Other_Agent`` with ``n_agents == 1``.
    Passing the Agent itself pairs each agent with itself.  The partner's position is read as it stands when the rates are
    evaluated: its queued motion step runs first, and its in-place edits are uploaded.  ``Agent.run`` does not move the
    partner, like the reference's loop.  ``tuning_type_agent`` may be reassigned (another Agent, or None: zero rates).

    Away from the agents (``evaluate_at="all"`` or ``pos=...``) the partner is ``Other_Agent.pos`` when it has one agent;
    a batched partner needs the ``other_pos`` kwarg, one (2,) position or one per position.  Egocentric cells take the
    ``head_direction`` kwarg there, like ObjectVectorCells.  Rates are evaluated by ``riab_avc_*`` (csrc/riab_avc.cuh)."""
    default_params = {                                              # ratinabox/Neurons.py:2165-2168
        "name": "AgentVectorCell",
        "walls_occlude": True,          # agents behind walls cannot be seen
    }
    _cells_kind = _lib.CELLS_AVC
    _egocentric_warning = ObjectVectorCells._egocentric_warning      # the reference's own text (Neurons.py:2274-2276)
    _zeroed_state = True                                             # zeros without a partner (:2231-2232)

    def __init__(self, Agent, Other_Agent, params={}):
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        Other_Agent.agent_idx                                        # the reference reads it for its colours (:2195)
        warn_n = "n" in params and params["n"] is not None           # Neurons.py:2180-2181
        super().__init__(Agent, p)
        self._init_vector_tuning()
        if warn_n:                                                   # VectorCells.__init__, Neurons.py:1375-1379
            arr = self.params["cell_arrangement"]
            if (isinstance(arr, str) and arr.endswith("manifold")) or self.params["n"] != self.n:
                warnings.warn(f"Ignoring 'n' parameter value ({self.params['n']}) that was passed, and setting number of "
                              f"{self.name} neurons to {self.n}, inferred from the cell arrangement parameter.")
        self.wall_geometry = "line_of_sight" if self.walls_occlude == True else "euclidean"      # Neurons.py:2188-2191
        if Agent.Environment.boundary_conditions == "periodic":
            raise NotImplementedError("AgentVectorCells need solid boundary conditions on the CUDA path")
        self._check_partner(Other_Agent)
        self.tuning_type_agent = Other_Agent

    def _check_partner(self, other):
        ag = self.Agent
        if other is None or other is ag:
            return
        if other.n_agents not in (ag.n_agents, 1):
            raise ValueError(f"Other_Agent has {other.n_agents} agents, this Agent {ag.n_agents}: AgentVectorCells pair row "
                             "i with row i of Other_Agent, or every row with an Other_Agent of one agent")
        if other.n_agents > 1 and int(other.id_offset) != int(ag.id_offset):
            raise ValueError(f"Other_Agent's id_offset {other.id_offset} differs from this Agent's {ag.id_offset}: paired "
                             "shards must cover the same global agent ids")
        if other.device != ag.device:
            raise ValueError(f"Other_Agent lives on {other.device}, this Agent on {ag.device}")

    def _partner(self):
        """The partner, with its queued motion step run and its in-place edits uploaded (the position the reference's
        get_state would read now)."""
        other = self.tuning_type_agent
        if other is not None and other is not self.Agent:
            other._flush_pending()
            other._sync_user_writes()
        return other

    def _cells(self):
        self._partner()
        return super()._cells()

    def _signature(self):
        other = self.tuning_type_agent
        return tuple(a.tobytes() for a in self._vector_tuning()) + (
            float(self.min_fr), float(self.max_fr), self.reference_frame, self.wall_geometry,
            self.Agent.Environment._walls_signature(), id(other),
            None if other is None else (other.n_agents, int(other.id_offset), other._s["pos"].data_ptr()))

    def _pack(self):
        other = self.tuning_type_agent
        self._check_partner(other)
        arrs = self._vector_tuning()
        self.n = arrs[0].shape[0]
        c = _lib.AvcCells()
        host = np.zeros(self._lib.riab_avc_pack_floats(self.n), dtype=np.float32)
        _lib.check(self._lib.riab_avc_pack(*[_f64p(a) for a in arrs], self.n, C.byref(c), host.ctypes.data_as(_lib.c_float_p)))
        self._packed = self._upload(host)
        c.walls_occlude = 1 if self.wall_geometry == "line_of_sight" else 0
        c.egocentric = 1 if self.reference_frame == "egocentric" else 0
        c.partner_is_self = 1 if other is self.Agent else 0
        c.min_fr, c.max_fr = float(self.min_fr), float(self.max_fr)
        c.packed_dev = self._packed.data_ptr()
        c.other_pos_dev = None if (other is None or other is self.Agent) else other._s["pos"].data_ptr()
        c.n_other = 1 if (other is None or other is self.Agent) else other.n_agents
        return c

    def _kernel_inputs(self, evaluate_at, n_pos, kwargs):
        """The partner's positions (its agents' at "agent", else the ``other_pos`` kwarg or a one-agent partner's
        position) and, for egocentric cells, the head directions; nothing without a partner."""
        other = self.tuning_type_agent
        if other is None:
            return {}
        if evaluate_at == "agent":
            other_pos = other._s["pos"]
        elif "other_pos" in kwargs:
            other_pos = self._rows(kwargs["other_pos"])
        elif other.n_agents == 1:
            other_pos = other._s["pos"]
        else:
            raise ValueError(f"Other_Agent has {other.n_agents} agents: pass their positions away from the agents "
                             "with other_pos=, one (2,) position or one per position")
        if other_pos.shape[0] not in (1, n_pos):
            raise ValueError(f"{other_pos.shape[0]} partner positions for {n_pos} positions: pass one (2,) position or one "
                             "per position")
        return dict(super()._kernel_inputs(evaluate_at, n_pos, kwargs), other_pos=other_pos)

    def _rates_from_positions(self, pos_dev, n_pos, out, head_dir=None, other_pos=None):
        if other_pos is None:
            return                                                   # no partner: the zeros get_state allocated
        ag = self.Agent
        _lib.check(self._lib.riab_avc_rates(pos_dev.data_ptr(), n_pos, other_pos.data_ptr(),
                                            1 if other_pos.shape[0] > 1 else 0, C.byref(ag._env_struct()),
                                            C.byref(self._cells()), None if head_dir is None else head_dir.data_ptr(),
                                            out.data_ptr(), out.stride(0), ag._stream()))


class FieldOfViewAVCs(AgentVectorCells):
    """Egocentric AgentVectorCells tiling the agent's field of view (ratinabox/Neurons.py:2323-2351)."""
    default_params = {
        "distance_range": [0.02, 0.4],
        "angle_range": [0, 75],
        "spatial_resolution": 0.02,
        "beta": 5,
        "cell_arrangement": "diverging_manifold",
    }

    def __init__(self, Agent, Other_Agent, params={}):
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        p["reference_frame"] = "egocentric"
        assert p["cell_arrangement"] is not None, "cell_arrangement must be set for FOV Neurons"
        super().__init__(Agent, Other_Agent, p)


# =============================================================================
class _FflInput(dict):
    """One entry of ``FeedForwardLayer.inputs`` with the reference's keys (Neurons.py:2781-2788).  ``"I"`` is looked up
    lazily: it is the input layer's ``firingrate`` as it stands when read, so no step pays a device -> host copy."""

    def __getitem__(self, k):
        if k == "I":
            return dict.__getitem__(self, "layer").firingrate
        return dict.__getitem__(self, k)

    def get(self, k, default=None):
        return self[k] if k in self else default


class FeedForwardLayer(Neurons):
    """ratinabox.FeedForwardLayer (Neurons.py:2654-2847): firingrate = phi(sum over input layers of w . I + biases).

    Inputs are any populations of the same Agent, other FeedForwardLayers and the layer itself included.  Like the
    reference's update loop (``[Ns.update() for Ns in Ag.Neurons]``) an input registered before the layer gives this
    step's rates, one registered at or after it the previous step's (zeros before its first update).  ``inputs[name]["w"]``
    and ``biases`` are float64 NumPy arrays the user may edit between steps; they are re-packed when their bytes change.
    The activations are the premade ones of utils.activate (utils.py:919-1026); bespoke callables raise.  The contraction
    runs as an error-compensated TF32 tensor-core GEMM over the whole batch (csrc/riab_ffl.cuh)."""
    default_params = {                                              # ratinabox/Neurons.py:2699-2705
        "n": 10,
        "input_layers": [],
        "activation_function": {"activation": "linear"},
        "name": "FeedForwardLayer",
        "biases": None,
    }
    _cells_kind = _lib.CELLS_FFL

    def __init__(self, Agent, params={}):
        params = dict(params)
        if "activation_params" in params:                          # Neurons.py:2712-2715
            warnings.warn("The parameter 'activation_params' is deprecated. Use 'activation_function' instead.")
            params["activation_function"] = params.pop("activation_params")
        super().__init__(Agent, params)
        assert isinstance(self.input_layers, list), "param['input_layers'] must be a list."
        if len(self.input_layers) == 0:
            warnings.warn("No input layers have been provided. Either hand them in in the params dictionary "
                          "params['input_layers']=[list,of,inputs] or use self.add_input_layer() to add them manually.")
        self._activation()                                           # refuse bespoke activations at construction
        self.inputs = {}
        for layer in self.input_layers:
            self.add_input(layer)
        if self.biases is None:
            self.biases = np.zeros(self.n)
        self._prime = None
        self._bias_dev = None
        self._w_dev = []

    def add_input(self, input_layer, w=None, w_init_scale=1, recurrent=False, **kwargs):
        """FeedForwardLayer.add_input (Neurons.py:2758-2795), with the reference's weight draw."""
        if input_layer.Agent is not self.Agent:
            raise ValueError("a FeedForwardLayer's inputs must belong to its own Agent")
        n, name = input_layer.n, input_layer.name
        if name not in self.inputs and len(self.inputs) >= _lib.FFL_MAX_INPUTS:
            raise NotImplementedError(f"at most {_lib.FFL_MAX_INPUTS} input layers per FeedForwardLayer on the CUDA path")
        if w is None:
            w = np.random.normal(loc=0, scale=w_init_scale / np.sqrt(n), size=(self.n, n))
        entry = _FflInput(layer=input_layer, w=w, w_init=w.copy(), I=None, n=input_layer.n, recurrent=recurrent)
        entry.update(kwargs)
        self.inputs[name] = entry
        if input_layer._population_id >= self._population_id:
            input_layer._ring_min = 2           # read one step late: its previous row must survive its next update

    def _activation(self):
        """(riab_activation id, 4 float parameters) of the premade activation dict (utils.activate, utils.py:919-1026)."""
        af = self.activation_function
        if not isinstance(af, dict) or "function" in af:
            raise NotImplementedError("bespoke (callable) activation functions are not supported on the CUDA path: use one "
                                      "of the premade utils.activate dicts, e.g. {'activation': 'relu', 'gain': 1, 'threshold': 0}")
        name = af["activation"]
        assert name in _lib.ACTIVATIONS, f"unknown activation {name!r}"
        if name == "linear":
            prm = (0.0, 0.0, 0.0, 0.0)
        elif name == "sigmoid":                                      # utils.py:961-979
            a = {"max_fr": 1, "min_fr": 0, "mid_x": 1, "width_x": 2}
            a.update(af)
            prm = (a["max_fr"], a["min_fr"], a["mid_x"], np.log((1 - 0.05) / 0.05) / (0.5 * a["width_x"]))
        else:                                                        # utils.py:981-1026
            a = {"gain": 1, "threshold": 0}
            a.update(af)
            prm = (a["gain"], a["threshold"], 0.0, 0.0)
        return _lib.ACTIVATIONS[name], tuple(float(x) for x in prm)

    def _signature(self):
        sig = [self.n, repr(self.activation_function), np.ascontiguousarray(self.biases, dtype=np.float64).tobytes()]
        for name, e in self.inputs.items():
            sig += [name, id(e["layer"]), e["layer"].n, np.ascontiguousarray(e["w"], dtype=np.float64).tobytes()]
        return tuple(sig)

    def _pack(self):
        act, prm = self._activation()
        c = _lib.FflCells()
        c.n_cells, c.activation = self.n, act
        for i in range(4):
            c.act[i] = prm[i]
        b = np.ascontiguousarray(self.biases, dtype=np.float64).reshape(-1)
        assert b.shape[0] == self.n, f"biases must have shape ({self.n},)"
        self._bias_dev = self._upload(b.astype(np.float32))
        c.bias_dev = self._bias_dev.data_ptr()
        self._w_dev = []
        for i, (name, e) in enumerate(self.inputs.items()):
            n_in = e["layer"].n
            w = np.ascontiguousarray(e["w"], dtype=np.float64)
            assert w.shape == (self.n, n_in), f"inputs[{name!r}]['w'] must have shape ({self.n}, {n_in})"
            host = np.zeros(self._lib.riab_ffl_pack_floats(self.n, n_in), dtype=np.float32)
            _lib.check(self._lib.riab_ffl_pack(_f64p(w), self.n, n_in, C.byref(c.inputs[i]), host.ctypes.data_as(_lib.c_float_p)))
            dev = self._upload(host)
            self._w_dev.append(dev)
            c.inputs[i].w_dev = dev.data_ptr()
        c.n_inputs = len(self.inputs)
        return c

    def _layer_struct(self, c):
        """The riab_ffl_cells part of the struct _cells() returns."""
        return c

    def _slot_ptr(self, layer, slot):
        if slot is None:
            return None                   # never updated: the reference's initial zeros (Neurons.py:120)
        return layer._hist.data_ptr() + slot * self.Agent.n_agents * layer._ld() * 4

    def _cells(self):
        c = super()._cells()
        if self._prime is None:
            self._prime = self._torch.zeros((self.Agent.n_agents, self._ld()), dtype=self._torch.float32, device=self.device)
        c.prime_dev = self._prime.data_ptr()
        for i, e in enumerate(self.inputs.values()):
            layer, meta = e["layer"], c.inputs[i]
            meta.population = layer._population_id
            meta.lag = 0 if layer._population_id < self._population_id else 1
            meta.rows_dev, meta.ld = self._slot_ptr(layer, layer._last_slot), layer._ld()
        return c

    def _row_buffers(self):
        # update(): the struct was bound before this layer's next row was taken; a self-recurrent input reads the
        # previous row, located in the ring as it is after any growth
        prev = self._last_slot
        out = super()._row_buffers()
        for i, e in enumerate(self.inputs.values()):
            if e["layer"] is self:
                self._cstruct.inputs[i].rows_dev = self._slot_ptr(self, prev)
        return out

    def _cells_for_run(self):
        """Agent.run: the rows read one step late before the run's first step are snapshots (the run may overwrite the
        ring slot they sit in before the layer reads them)."""
        c = self._cells()
        self._run_keep = []
        for i, e in enumerate(self.inputs.values()):
            layer = e["layer"]
            if c.inputs[i].lag == 1 and layer._last_slot is not None:
                snap = layer._hist[layer._last_slot].clone()
                self._run_keep.append(snap)
                c.inputs[i].rows_dev = snap.data_ptr()
        return c

    @property
    def firingrate_prime(self):
        """phi'(V) of the last evaluation at "last" (Neurons.py:2839-2845): (n,) for one agent, else (n_agents, n)."""
        A = self.Agent.n_agents
        if self._prime is None:
            return np.zeros(self.n) if A == 1 else np.zeros((A, self.n))
        r = self._prime[:, : self.n].cpu().numpy().astype(np.float64)
        return r[0] if A == 1 else r

    def get_state(self, evaluate_at="last", max_recurrence=None, **kwargs):
        """FeedForwardLayer.get_state (Neurons.py:2797-2847).  "last" reads the inputs' current rows and refreshes
        firingrate_prime; anything else evaluates the inputs with get_state(evaluate_at, ...) on the device first (recurrent
        inputs are skipped once max_recurrence runs out).  Returns (n, n_pos) float64, or with ``return_tensor=True`` the
        (n_pos, n) float32 device tensor."""
        torch = self._torch
        return_tensor = kwargs.pop("return_tensor", False)
        c = self._cells()
        if evaluate_at == "last":
            self.Agent._flush_pending()
            n_pos = self.Agent.n_agents
            fc = self._layer_struct(c)
        else:
            fc = _lib.FflCells.from_buffer_copy(c)
            fc.prime_dev = None
            n_pos, keep = self._input_rows(fc, evaluate_at, max_recurrence, kwargs)
        out = torch.empty((n_pos, self._ld()), dtype=torch.float32, device=self.device)
        ro = _lib.RatesOut()
        ro.rates_row, ro.ld = out.data_ptr(), self._ld()
        _lib.check(self._lib.riab_ffl_rates(C.byref(fc), n_pos, None, None, C.byref(ro), self.Agent._stream()))
        r = self._result(out, return_tensor)
        return r[:, 0] if (evaluate_at == "last" and n_pos == 1 and not return_tensor) else r

    def _input_rows(self, fc, evaluate_at, max_recurrence, kwargs):
        """Point fc's inputs at their populations' get_state(evaluate_at, ...) rows, evaluated on the device.  Returns the
        row count and the tensors that must outlive the evaluation."""
        torch = self._torch
        keep = []
        n_pos = self._n_pos(evaluate_at, kwargs, self.Agent.n_agents)
        for i, e in enumerate(self.inputs.values()):
            pass_max = max_recurrence
            if max_recurrence is not None and e["recurrent"]:
                if max_recurrence <= 0:
                    fc.inputs[i].rows_dev = None                  # skipped: contributes nothing (Neurons.py:2812-2815)
                    continue
                pass_max = max_recurrence - 1
            I = e["layer"].get_state(evaluate_at, max_recurrence=pass_max, return_tensor=True, **kwargs)
            if I.dtype != torch.float32 or I.stride(1) != 1 or I.stride(0) % 4 or I.data_ptr() % 16:
                ld = (I.shape[1] + 3) // 4 * 4
                J = torch.zeros((I.shape[0], ld), dtype=torch.float32, device=self.device)
                J[:, : I.shape[1]] = I
                I = J
            assert I.shape[0] == n_pos
            keep.append(I)
            fc.inputs[i].rows_dev, fc.inputs[i].ld = I.data_ptr(), I.stride(0)
        return n_pos, keep


# =============================================================================
class RandomSpatialNeurons(Neurons):
    """ratinabox.RandomSpatialNeurons (Neurons.py:2865-2954): smooth random spatial tunings drawn from a Gaussian process.

    Set-up (host, float64, the reference's global NumPy draws in the reference's order): the sample grid ``X`` =
    ``discretise_environment(dx=min(0.05, lengthscale))``, its covariance ``Q = kernel(X, X)`` with the population's
    ``wall_geometry`` distances, and ``targets`` = sigmoid(multivariate_normal(0, Q, size=n).T) in [min_fr, max_fr].
    ``targets`` is a float64 (|X|, n) array the user may edit; it is re-packed when its bytes change.

    Rates: the kernel-weighted average of the targets, ``k(pos, X) @ targets / sum k(pos, X)``, evaluated in one fused
    kernel (csrc/riab_rsn.cuh): the kernel row is generated in registers as a PlaceCells row over X and contracted with
    the targets on the tensor cores.  NaN positions give zero rates."""
    default_params = {                                              # ratinabox/Neurons.py:2875-2881
        "lengthscale": 0.1,
        "max_fr": 1,
        "min_fr": 0,
        "n": 10,
        "wall_geometry": "geodesic",
        "name": "RandomSpatialNeurons",
    }
    _cells_kind = _lib.CELLS_RSN

    def __init__(self, Agent, params={}):
        super().__init__(Agent, params)
        self._set_up()

    def _set_up(self):
        """The host set-up of Neurons.py:2890-2913 (no device work)."""
        env = self.Agent.Environment
        if self.wall_geometry == "geodesic" and len(env.walls) > 5:    # Neurons.py:2890-2894
            print("Geodesic wall geometry only possible in environments with one or no additional walls. Using "
                  "'line_of_sight' instead. If this is slow, consider trying 'euclidean'")
            self.wall_geometry = "line_of_sight"
        assert self.lengthscale >= 0.02, "lengthscale must be greater than 0.02 m"
        self._effective_geometry()                                   # the device path's limits, before any draw
        X = env.discretise_environment(dx=min(0.05, self.lengthscale))
        self.X = X.reshape(-1, X.shape[-1])
        self.Q = self.kernel(self.X, self.X)
        with warnings.catch_warnings():                              # Neurons.py:2909-2911
            warnings.simplefilter("ignore", category=RuntimeWarning)
            targets = np.random.multivariate_normal(mean=np.zeros(self.Q.shape[0]), cov=self.Q, size=self.n).T
        from .utils import sigmoid
        self.targets = sigmoid(targets, max_fr=self.max_fr, min_fr=self.min_fr, mid_x=0, width_x=2)

    def kernel(self, x1, x2):
        """(len(x1), len(x2)) squared-exponential covariance over the environment's distances (Neurons.py:2944-2954),
        host float64, with the reference's jitter draws for the wall tests."""
        from .utils import get_distances_between___accounting_for_environment
        d = get_distances_between___accounting_for_environment(self.Agent.Environment, x1, x2, self.wall_geometry)
        return np.exp(-(d ** 2) / (2 * self.lengthscale ** 2))

    def _effective_geometry(self):
        """The device path's wall geometry: PlaceCells' limits (geodesic only in the box, at most PLACE_MAX_WI inner
        walls); without inner walls every geometry is the plain distance.  Periodic boundaries are refused by kernel()."""
        geom = PlaceCells._effective_geometry(self)
        n_inner = len(self.Agent.Environment.walls) - self.Agent.Environment.los_skip
        if geom != "euclidean" and n_inner > _lib.PLACE_MAX_WI:
            raise NotImplementedError(f"at most {_lib.PLACE_MAX_WI} inner walls with {geom} wall geometry on the CUDA path")
        return geom

    def _signature(self):
        env = self.Agent.Environment
        return (np.ascontiguousarray(self.targets, dtype=np.float64).tobytes(),
                np.ascontiguousarray(self.X, dtype=np.float64).tobytes(), float(self.lengthscale), self.wall_geometry,
                env._walls_signature(), float(self.min_fr), float(self.max_fr))

    def _pack(self):
        env = self.Agent.Environment
        X = np.ascontiguousarray(self.X, dtype=np.float64).reshape(-1, 2)
        T = np.ascontiguousarray(self.targets, dtype=np.float64)
        assert T.ndim == 2 and T.shape[0] == X.shape[0], f"targets must have shape ({X.shape[0]}, n)"
        self.n = T.shape[1]
        geom = _lib.WALL_GEOMETRIES[self._effective_geometry()]
        walls = np.ascontiguousarray(env.walls, dtype=np.float64)
        n_inner = 0 if geom == 0 else walls.shape[0] - env.los_skip
        c = _lib.RsnCells()
        host = np.zeros(self._lib.riab_rsn_pack_floats(self.n, X.shape[0], n_inner), dtype=np.float32)
        k_pad = (X.shape[0] + 31) // 32 * 32
        centres = np.zeros((k_pad, 2), dtype=np.float64)
        ext = np.ascontiguousarray(env.extent, dtype=np.float64)
        _lib.check(self._lib.riab_rsn_pack(_f64p(X), X.shape[0], _f64p(T), self.n, float(self.lengthscale), _f64p(walls),
                                           walls.shape[0], env.los_skip, _f64p(ext), geom, C.byref(c),
                                           host.ctypes.data_as(_lib.c_float_p), _f64p(centres)))
        self._packed = self._upload(host)
        self._centres_dev = self._upload(centres)
        point_floats = self._lib.riab_place_pack_floats(k_pad, c.points.n_inner_walls)
        c.points.packed_dev, c.points.centres_dev = self._packed.data_ptr(), self._centres_dev.data_ptr()
        c.targets_dev = self._packed.data_ptr() + 4 * point_floats
        c.min_fr, c.max_fr = float(self.min_fr), float(self.max_fr)
        return c

    def _rates_from_positions(self, pos_dev, n_pos, out):
        ag = self.Agent
        _lib.check(self._lib.riab_rsn_rates(pos_dev.data_ptr(), n_pos, C.byref(ag._env_struct()), C.byref(self._cells()),
                                            out.data_ptr(), out.stride(0), ag._stream()))


# =============================================================================
class _KinematicCells(Neurons):
    """Populations tuned to the agent's motion, not its position (HeadDirectionCells, VelocityCells, SpeedCell): one
    kernel kind (RIAB_CELLS_KIN, csrc/riab_kin.cuh) whose producer warps read the agent's float64 head direction,
    velocity or measured velocity."""
    _cells_kind = _lib.CELLS_KIN
    _variant = None
    one_sigma_speed = 1.0

    def _tuning(self):
        """(preferred_angles, angular_tunings) as float64 arrays, or (None, None) for a speed cell."""
        return None, None

    def _signature(self):
        pref, tun = self._tuning()
        return (None if pref is None else pref.tobytes(), None if tun is None else tun.tobytes(), float(self.min_fr),
                float(self.max_fr), float(self.one_sigma_speed), self.n)

    def _pack(self):
        pref, tun = self._tuning()
        if pref is not None:
            assert tun.shape == pref.shape, "preferred_angles and angular_tunings must have the same length"
            self.n = pref.shape[0]
        c = _lib.KinCells()
        host = np.zeros(self._lib.riab_kin_pack_floats(self.n), dtype=np.float32)
        _lib.check(self._lib.riab_kin_pack(None if pref is None else _f64p(pref), None if tun is None else _f64p(tun), self.n,
                                           self._variant, 0, float(self.min_fr), float(self.max_fr),
                                           float(self.one_sigma_speed), C.byref(c), host.ctypes.data_as(_lib.c_float_p)))
        self._packed = self._upload(host)
        c.packed_dev = self._packed.data_ptr()
        return c

    def _state(self, evaluate_at, use_velocity, vector=None, speed_scale=-1.0, **kwargs):
        """Rates at the agents (evaluate_at="agent": every agent's own head direction / velocity / measured velocity) or
        for the given ``vector``, one (2,) for every position or one per position, over the reference's n_pos: the
        discretised environment for "all", ``pos``'s rows, else 1 (Neurons.py:2476-2483).  (n, n_pos) float64, or with
        ``return_tensor=True`` the (n_pos, n) float32 device tensor."""
        torch = self._torch
        ag = self.Agent
        c = _lib.KinCells.from_buffer_copy(self._cells())
        c.use_velocity = 1 if use_velocity else 0
        if evaluate_at == "agent":
            vec = self._agent_state()["measured_velocity" if self._variant == _lib.KIN_SPEED else
                                      ("velocity" if use_velocity else "head_direction")]
            n_pos = ag.n_agents
        else:
            vec = self._rows(vector)
            n_pos = self._n_pos(evaluate_at, kwargs, int(vec.shape[0]))
            if vec.shape[0] not in (1, n_pos):
                raise ValueError(f"{vec.shape[0]} direction / velocity vectors for {n_pos} positions: pass one (2,) vector "
                                 "or one per position")
        per_position = 1 if (evaluate_at == "agent" or vec.shape[0] > 1) else 0
        out = torch.empty((n_pos, self._ld()), dtype=torch.float32, device=self.device)
        _lib.check(self._lib.riab_kin_rates(vec.data_ptr(), per_position, n_pos, float(speed_scale), C.byref(c),
                                            out.data_ptr(), out.stride(0), ag._stream()))
        return self._result(out, kwargs.get("return_tensor", False))


class HeadDirectionCells(_KinematicCells):
    """ratinabox.HeadDirectionCells (Neurons.py:2357-2485), 2D: cell i fires
    ``von_mises(get_angle(head_direction), preferred_angles[i], angular_tunings[i], norm=1) * (max_fr - min_fr) + min_fr``.
    ``preferred_angles`` / ``angular_tunings`` (radians) are float64 arrays the user may edit; they are re-packed when
    their bytes change.  Away from the agent the ``head_direction`` / ``velocity`` / ``vel`` kwargs take one (2,) vector
    or one per position."""
    default_params = {                                              # ratinabox/Neurons.py:2383-2389
        "min_fr": 0,
        "max_fr": 1,
        "n": 10,
        "angular_spread_degrees": 45,
        "name": "HeadDirectionCells",
    }
    _variant = _lib.KIN_HEAD_DIRECTION

    def __init__(self, Agent, params={}):
        if Agent.Environment.dimensionality != "2D":
            raise NotImplementedError("HeadDirectionCells in 1D environments are outside the CUDA hot path")
        super().__init__(Agent, params)
        self.preferred_angles = np.linspace(0, 2 * np.pi, self.n + 1)[:-1]           # Neurons.py:2404-2409
        self.angular_tunings = np.array([self.params["angular_spread_degrees"] * np.pi / 180] * self.n)

    def _tuning(self):
        return (np.ascontiguousarray(self.preferred_angles, dtype=np.float64).reshape(-1),
                np.ascontiguousarray(self.angular_tunings, dtype=np.float64).reshape(-1))

    def _direction_kwarg(self, use_velocity, kwargs):
        """The vector get_state reads away from the agent, with the reference's warning and prints (Neurons.py:2428-2459)."""
        if not use_velocity:
            if "head_direction" in kwargs:
                return kwargs["head_direction"]
            if "vel" in kwargs:
                warnings.warn("'vel' kwarg deprecated in favour of 'head_direction'")
                return kwargs["vel"]
            print("HeadDirection cells need a head direction but you didn't pass one. Taking ", end="")
            print("[1,0] as default", end="")
            print("Recommended to pass one in the 'head_direction' argument of get_state()")
            return [1, 0]
        if "velocity" in kwargs:
            return kwargs["velocity"]
        print("HeadDirection cells need a velocity but you didn't pass one. Taking ", end="")
        print("[1,0] as default", end="")
        print("Recommended to pass one in the 'velocity' argument of get_state()")
        return [1, 0]

    def get_state(self, evaluate_at="agent", use_velocity=False, **kwargs):
        """HeadDirectionCells.get_state (Neurons.py:2421-2485): with evaluate_at="agent" every agent's head direction
        (its normalised velocity with ``use_velocity=True``) -- any head_direction kwarg is ignored there, like the
        reference -- else the kwargs.  (n, n_pos)."""
        use_velocity = bool(use_velocity)
        vector = None if evaluate_at == "agent" else self._direction_kwarg(use_velocity, kwargs)
        return self._state(evaluate_at, use_velocity, vector, **kwargs)


class VelocityCells(HeadDirectionCells):
    """ratinabox.VelocityCells (Neurons.py:2534-2583): the use_velocity HeadDirectionCells rates times
    ``|Agent.velocity| / one_sigma_speed``, one_sigma_speed = speed_mean + speed_std at construction.  A zero velocity
    gives NaN rates like the reference.  Away from the agent the speed factor is the Agent's own velocity, which is one
    speed only for one agent: with n_agents > 1 that raises ValueError."""
    default_params = {                                              # ratinabox/Neurons.py:2552-2556
        "min_fr": 0,
        "max_fr": 1,
        "name": "VelocityCells",
    }
    _variant = _lib.KIN_VELOCITY

    def __init__(self, Agent, params={}):
        self.one_sigma_speed = Agent.speed_mean + Agent.speed_std                     # Neurons.py:2567
        super().__init__(Agent, params)

    def get_state(self, evaluate_at="agent", **kwargs):
        """VelocityCells.get_state (Neurons.py:2577-2583).  (n, n_pos)."""
        speed_scale = -1.0                               # at the agents: every agent's own |velocity| / one_sigma_speed
        if evaluate_at != "agent":
            if self.Agent.n_agents > 1:
                raise ValueError("VelocityCells.get_state away from the agent scales the rates by |Agent.velocity|, one "
                                 "speed per agent: evaluate at the agents, or use an Agent with n_agents=1")
            speed_scale = np.linalg.norm(self.Agent.velocity) / self.one_sigma_speed
        vector = None if evaluate_at == "agent" else self._direction_kwarg(True, kwargs)
        return self._state(evaluate_at, True, vector, speed_scale=speed_scale, **kwargs)


class SpeedCell(_KinematicCells):
    """ratinabox.SpeedCell (Neurons.py:2586-2651): one cell, ``|v| / one_sigma_speed * (max_fr - min_fr) + min_fr`` with
    v the measured velocity (the history's "vel", Agent.py:517) at the agent, else the ``vel`` kwarg (one (2,) vector, or
    one per position).  The population is one cell wide from the start (the reference sizes its noise, and so its rows,
    for the default n = 10 before setting n = 1)."""
    default_params = {                                              # ratinabox/Neurons.py:2603-2607
        "min_fr": 0,
        "max_fr": 1,
        "name": "SpeedCell",
    }
    _variant = _lib.KIN_SPEED

    def __init__(self, Agent, params={}):
        params = dict(params)
        n_given = params.get("n", 1)
        params["n"] = 1
        super().__init__(Agent, params)
        if n_given != 1:                                            # Neurons.py:2621-2622
            warnings.warn(f"Ignoring 'n' parameter value ({n_given}) that was passed for {self.name}. Only 1 speed cell is needed.")
        self.one_sigma_speed = self.Agent.speed_mean + self.Agent.speed_std           # Neurons.py:2625

    def get_state(self, evaluate_at="agent", **kwargs):
        """SpeedCell.get_state (Neurons.py:2632-2651).  (1, n_pos) with n_pos as for HeadDirectionCells."""
        vector = None if evaluate_at == "agent" else kwargs["vel"]
        return self._state(evaluate_at, False, vector, **kwargs)

"""ratinabox.contribs.SubAgent (contribs/SubAgent.py:10-36), ThetaSequenceAgent (:182-356), DumbAgent (:118-179),
ReplayAgent (:358-431), ShiftAgent (:466-478) and UnrelatedAgent (:480-489) on the device.

A SubAgent is an Agent over the same batch as its lead Agent (same ``n_agents``, ``id_offset`` and ``dt``) whose
``update()`` follows the lead's.  ThetaSequenceAgent's position is a theta sweep over the lead's: once per theta cycle it
runs from behind the lead, along the lead's recent path, to ahead of it, along a freshly sampled forward trajectory, at
``v_sequence`` relative to the lead.  Each ``update()`` is one kernel (riab_theta_seq_step: the sweep position of every
agent) and the forced step of Agent.update that moves the ThetaSequenceAgent there.  Populations built on it
(``PlaceCells(TSA)``) read that position like any Agent's; NaN positions give zero rates.

Where the reference raises, this returns a defined position instead (DESIGN.md, ThetaSequenceAgent):
  * look behind, when the six rows around the closest recorded distance do not bracket the target (slow agents and the
    first sweep after construction): the two recorded rows that bracket it are interpolated; NaN before the recorded rows;
  * look ahead, when the query lies past the end of the forward rollout: NaN.
The forward rollout is stepped lazily, only as far as the sweep has reached, which gives the reference's interpolated
positions bit for bit with no bound on the number of rollout steps.  ``run()`` is not available: the lead's whole-run
kernel does not drive SubAgents.

DumbAgent, ShiftAgent and ReplayAgent make one riab_subagent_step launch per ``update()`` (the position of every agent,
float64 in the reference's operation order) followed by the same forced step; UnrelatedAgent is an Agent stepped with
the lead's dt.  ReplayAgent rolls its sham agent out lazily, like the ThetaSequenceAgent's look ahead (DESIGN.md,
SubAgents).
"""
import math
import copy
import ctypes as C
import warnings

import numpy as np

from .. import _lib
from ..Agent import Agent, _STATE


def _current_state(agent):
    """The Agent's device state as it stands now: its queued motion step run and the user's in-place edits of its arrays
    uploaded (as a population reads a partner Agent)."""
    agent._flush_pending()
    agent._sync_user_writes()
    return agent._s


class SubAgent(Agent):
    """An Agent "subservient" to a lead Agent (contribs/SubAgent.py:10-36): same batch, same ``dt``, starting from the
    lead's position and velocity.  ``update(**kwargs)`` sets ``t = LeadAgent.t`` and runs Agent.update, so it ends one
    ``dt`` ahead of the lead's clock, as in the reference."""
    default_params = {}

    def __init__(self, LeadAgent, params={}):
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        self.LeadAgent = LeadAgent
        if "dt" in p:
            warnings.warn("You have passed 'dt as a parameter but this will be overwritten to match dt of the LeadAgent")
        p["dt"] = LeadAgent.dt
        p["n_agents"], p["id_offset"] = LeadAgent.n_agents, LeadAgent.id_offset
        known = set()
        for cls in type(self).__mro__:
            known.update(getattr(cls, "default_params", {}).keys())
        unexpected = [k for k in params if k not in known]
        if unexpected:
            warnings.warn(f"Found {len(unexpected)} unexpected params key(s) while initializing {type(self).__name__}: "
                          f"{unexpected}")
        super().__init__(LeadAgent.Environment, {k: v for k, v in p.items() if k in Agent.default_params})
        for k, v in p.items():
            setattr(self, k, v)
        self.params.update(p)
        lead = _current_state(LeadAgent)
        self._s["pos"].copy_(lead["pos"])                           # :29-31
        self._s["velocity"].copy_(lead["velocity"])

    def update(self, **kwargs):                                      # :33-36
        self.t = self.LeadAgent.t
        super().update(**kwargs)

    def run(self, n_steps, **kwargs):
        raise NotImplementedError(f"{type(self).__name__}.run(): the lead Agent's whole-run kernel does not drive "
                                  "SubAgents; step the lead and the SubAgent with update()")


class ThetaSequenceAgent(SubAgent):
    """ratinabox.contribs.SubAgent.ThetaSequenceAgent: a theta sweep over the lead Agent's position, for every agent of the
    lead's batch.  Per theta cycle, as a fraction phi of it:

    * phi < 1/2 - theta_frac/2, phi >= 1/2 + theta_frac/2: NaN;
    * look behind, up to phi = 1/2: the lead's recent path, interpolated by distance travelled;
    * look ahead: a forward trajectory sampled from the lead's position and velocity with this Agent's motion
      parameters (``forward_agent_update_kwargs`` apply), at ``dt * v_sequence / LeadAgent.average_measured_speed``.

    Construction resets ``LeadAgent.distance_travelled`` to 0, as the reference does; the lead's history rows written
    before keep the distances they had.  The lead's recent positions and distances are kept in a private float64 ring
    (3 x ``lookback`` x ``n_agents`` doubles, ``lookback = int(5 d_half / (dt average_measured_speed))``: 1.2 GB at
    65 536 agents and dt = 0.01 s), so the lead's history ring may be small or switched off.
    """
    default_params = {                                              # contribs/SubAgent.py:205-209
        "v_sequence": 5.0,
        "theta_freq": 10.0,
        "theta_frac": 0.5,
    }

    def __init__(self, LeadAgent, params={}):
        import torch
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        super().__init__(LeadAgent, p)
        Lead = self.LeadAgent
        Lead.distance_travelled = 0                                   # :220
        self.T_theta = 1 / self.theta_freq                            # :228-230
        self.d_half = ((self.theta_frac / 2) * self.T_theta * self.v_sequence)
        self.last_theta_phase = 0
        self.n_half = int(2 * self.d_half / (Lead.speed_mean * Lead.dt))    # :233-240
        self.keep_count = max(1, (20 * self.n_half))
        self.counter = 1
        assert (Lead.dt <= self.T_theta / 10), f"params['dt'] for the LeadAgent is too large. It must be < 10% of theta time period., i.e. smaller than {self.T_theta/10:.5f}"
        assert (self.v_sequence >= 4*Lead.speed_mean), f"params['v_sequence'] is too small. It must be > 4*LeadAgent.speed_mean, i.e. larger than {4*Lead.speed_mean:.2f}"

        A = self.n_agents
        f64 = dict(dtype=torch.float64, device=self.device)
        lead = _current_state(Lead)
        # the forward agent (:222-225): its state on the device, one row per agent
        self._fwd = {k: lead[k].clone() for k in _STATE}
        self._fwd_c = _lib.Agents()
        self._fwd_c.n_agents, self._fwd_c.id_offset = A, int(self.id_offset)
        for k in _STATE:
            setattr(self._fwd_c, k, self._fwd[k].data_ptr())
        self._fwd_pair = torch.zeros((A, 3), **f64)
        self._fwd_stop = torch.zeros(A, **f64)
        self._fwd_steps = torch.zeros(A, dtype=torch.int64, device=self.device)
        self._fwd_mp = _lib.MotionParams()
        self._fill_motion_params(Lead.dt * self.v_sequence / Lead.average_measured_speed, {}, mp=self._fwd_mp)
        self._rollout = -1
        self._out = torch.empty((A, 2), **f64)
        self._ring = None
        self._ring_rows = 0
        self._ring_head = -1
        self._ring_held = 0
        self._reserve_ring(self._lookback())
        self._ts = _lib.ThetaSeq()

    def _lookback(self):
        Lead = self.LeadAgent
        return int(5 * self.d_half / (Lead.dt * Lead.average_measured_speed))      # :283

    def _reserve_ring(self, lookback):
        """Grow the look-behind ring to `lookback` rows (at least one), keeping the rows it holds."""
        import torch
        rows = max(1, int(lookback))
        if rows <= self._ring_rows:
            return
        A = self.n_agents
        need = 3 * rows * A * 8
        free, _ = torch.cuda.mem_get_info(self.device)
        if need > free:
            raise MemoryError(f"ThetaSequenceAgent: the look-behind ring of {rows} lead steps x {A} agents needs "
                              f"{need / 2**30:.2f} GiB of device memory, {free / 2**30:.2f} GiB are free")
        ring = torch.empty((3, rows, A), dtype=torch.float64, device=self.device)
        if self._ring_held > 0:
            order = [(self._ring_head - self._ring_held + 1 + j) % self._ring_rows for j in range(self._ring_held)]
            ring[:, : self._ring_held].copy_(self._ring[:, order])
            self._ring_head = self._ring_held - 1
        self._ring, self._ring_rows = ring, rows

    def update(self, dt=None, drift_velocity=None, drift_to_random_strength_ratio=1, forward_agent_update_kwargs={},
               **kwargs):
        """ThetaSequenceAgent.update (contribs/SubAgent.py:245-350) for every agent.  As in the reference, dt,
        drift_velocity and drift_to_random_strength_ratio are ignored; the motion keywords of forward_agent_update_kwargs
        apply to the forward rollouts that start at this call.  ``_xi_forward`` (n_agents, K, 2): injected standard
        normals of rollout steps 0..K-1 of the current rollout (parity tap, like Agent.update's ``_xi``)."""
        import torch
        fkw = dict(forward_agent_update_kwargs)
        if fkw.get("drift_velocity", None) is not None:
            raise NotImplementedError("ThetaSequenceAgent: drift_velocity in forward_agent_update_kwargs is not supported")
        Lead = self.LeadAgent
        lead = _current_state(Lead)

        # :258-264 -- the stash's counter rule; the window is the last min(lookback, counter) lead rows
        if self.counter == self.keep_count:
            self.counter = 10 * self.n_half
        lookback = self._lookback()
        self._reserve_ring(lookback)
        self._ring_head = (self._ring_head + 1) % self._ring_rows
        self._ring_held = min(self._ring_held + 1, self._ring_rows)

        self.t = Lead.t
        theta_phase = (self.t % (1 / self.theta_freq)) / ((1 / self.theta_freq))     # :267
        ts = self._ts
        ts.phase, ts.offset, ts.window = _lib.THETA_NONE, 0.0, 1
        if (theta_phase >= (0.5 - self.theta_frac / 2)) and (theta_phase < 0.5):      # :274-300
            c = self.d_half / self.theta_frac
            m = -2 * c
            distance_back = (m * theta_phase + c)
            ts.phase, ts.offset = _lib.THETA_BEHIND, -distance_back
            ts.window = max(1, min(lookback, self.counter, self._ring_held))
        if (theta_phase >= 0.5) and (theta_phase < 0.5 + self.theta_frac / 2):        # :303-334
            ts.phase = _lib.THETA_AHEAD
            if (theta_phase >= 0.5 and self.last_theta_phase < 0.5):
                ts.phase = _lib.THETA_AHEAD_FIRST
                self._rollout += 1
                recent_speed = Lead.average_measured_speed
                ts.forward_distance = (self.d_half + 100 * recent_speed * (self.theta_frac / 2) * self.T_theta)
                self._fill_motion_params(Lead.dt * self.v_sequence / Lead.average_measured_speed, fkw, mp=self._fwd_mp)
            c = -self.d_half / self.theta_frac
            m = -2 * c
            distance_ahead = (m * theta_phase + c)
            ts.offset = distance_ahead
        xi = kwargs.get("_xi_forward", None)
        xi_keep = None
        ts.xi_forward, ts.xi_steps = None, 0
        if xi is not None:
            xi_keep = torch.as_tensor(np.ascontiguousarray(xi, dtype=np.float64), device=self.device).reshape(self.n_agents, -1, 2)
            ts.xi_forward, ts.xi_steps = xi_keep.data_ptr(), int(xi_keep.shape[1])

        ts.n_agents, ts.id_offset = self.n_agents, int(self.id_offset)
        ts.lead_pos, ts.lead_velocity = lead["pos"].data_ptr(), lead["velocity"].data_ptr()
        ts.lead_rotational_velocity, ts.lead_distance = lead["rotational_velocity"].data_ptr(), lead["distance_travelled"].data_ptr()
        ts.ring, ts.ring_rows, ts.ring_head = self._ring.data_ptr(), self._ring_rows, self._ring_head
        ts.fwd = self._fwd_c
        ts.fwd_pair, ts.fwd_stop, ts.fwd_steps = self._fwd_pair.data_ptr(), self._fwd_stop.data_ptr(), self._fwd_steps.data_ptr()
        ts.seed = int(self.seed) & 0xFFFFFFFFFFFFFFFF
        ts.rollout = max(self._rollout, 0)
        ts.d_half = float(self.d_half)
        ts.out_pos = self._out.data_ptr()
        _lib.check(self._lib.riab_theta_seq_step(C.byref(ts), C.byref(self._env_struct()), C.byref(self._fwd_mp),
                                                 self._stream()))
        self._xi_keep = xi_keep                   # the launch reads it asynchronously
        self.last_theta_phase = theta_phase       # :345-346
        self.counter += 1
        SubAgent.update(self, forced_next_position=self._out)


def _tensor_tap(agent, value, shape):
    """A parity tap (injected draws) as a contiguous float64 device tensor of `shape`, or None."""
    import torch
    if value is None:
        return None
    return torch.as_tensor(np.ascontiguousarray(value, dtype=np.float64), device=agent.device).reshape(shape)


class DumbAgent(SubAgent):
    """ratinabox.contribs.SubAgent.DumbAgent (contribs/SubAgent.py:118-179): the lead's position plus a displacement on a
    stochastic spring.  Per step the displacement velocity takes an Ornstein-Uhlenbeck step (noise sigma, timescale tau_v)
    plus the spring's -acceleration_scale * displacement * dt; a displacement that crosses a wall is cut back to 0.95 of
    the nearest crossing; the boundary conditions apply, and the displacement is re-measured through the environment.

    ``displacement`` and ``displacement_velocity`` are (n_agents, 2) float64 device state, read and written like the
    Agent's own state arrays.  ``sigma``, ``tau_v`` and ``acceleration_scale`` are fixed at construction, as in the
    reference.
    """
    default_params = {                                              # contribs/SubAgent.py:134-136
        "drift_distance": 0.05,
        "drift_timescale": 3.0,
    }
    _VEC_NAMES = Agent._VEC_NAMES | {"displacement", "displacement_velocity"}

    def __init__(self, LeadAgent, params={}):
        import torch
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        super().__init__(LeadAgent, p)
        f64 = dict(dtype=torch.float64, device=self.device)
        self._s["displacement"] = torch.zeros((self.n_agents, 2), **f64)            # :145-146
        self._s["displacement_velocity"] = torch.zeros((self.n_agents, 2), **f64)
        self.tau_v = self.drift_timescale / 2                                         # :147-149
        self.sigma = np.pi**2 * self.drift_distance / (self.drift_timescale**2)
        self.acceleration_scale = self.sigma / self.drift_distance
        self._sa = _lib.SubAgentStep()
        self._out = torch.empty((self.n_agents, 2), **f64)
        self._updates = 0

    displacement = property(lambda self: self._get_state("displacement"),
                            lambda self, v: self._set_state("displacement", v))
    displacement_velocity = property(lambda self: self._get_state("displacement_velocity"),
                                     lambda self, v: self._set_state("displacement_velocity", v))

    def update(self, **kwargs):
        """DumbAgent.update (contribs/SubAgent.py:151-179) for every agent.  Parity taps: ``_xi_displacement``
        (n_agents, 2) standard normals of the OU step, ``_resample_pos`` (n_agents, 2) the positions a polygon or hole
        re-draws."""
        Lead = self.LeadAgent
        lead = _current_state(Lead)
        self._flush_pending()
        self._sync_user_writes()
        dt = float(Lead.dt)
        xi = _tensor_tap(self, kwargs.get("_xi_displacement"), (self.n_agents, 2))
        rs = _tensor_tap(self, kwargs.get("_resample_pos"), (self.n_agents, 2))
        sa = self._sa
        sa.n_agents, sa.id_offset, sa.kind = self.n_agents, int(self.id_offset), _lib.SUBAGENT_DUMB
        sa.seed, sa.step = int(self.seed) & 0xFFFFFFFFFFFFFFFF, self._updates
        sa.lead_pos, sa.dt = lead["pos"].data_ptr(), dt
        sa.displacement, sa.displacement_velocity = self._s["displacement"].data_ptr(), self._s["displacement_velocity"].data_ptr()
        s = float(self.sigma)                                          # utils.ornstein_uhlenbeck (utils.py:363-366)
        sa.ou_theta = 1 / float(self.tau_v)
        sa.ou_sigma = math.sqrt((2 * (s * s)) / (float(self.tau_v) * dt))
        sa.acceleration_scale = float(self.acceleration_scale)
        sa.xi_displacement = xi.data_ptr() if xi is not None else None
        sa.resample_pos = rs.data_ptr() if rs is not None else None
        sa.out_pos = self._out.data_ptr()
        _lib.check(self._lib.riab_subagent_step(C.byref(sa), C.byref(self._env_struct()), None, self._stream()))
        self._taps = (xi, rs)                     # the launch reads them asynchronously
        self._updates += 1
        SubAgent.update(self, forced_next_position=self._out)


class ShiftAgent(SubAgent):
    """ratinabox.contribs.SubAgent.ShiftAgent (contribs/SubAgent.py:466-478): the lead's position shifted by ``shift_m``
    along the lead's head direction (negative: behind it).  No boundary condition applies, as in the reference: in a
    periodic box the position may lie outside the box."""
    default_params = {                                              # contribs/SubAgent.py:471-473
        "shift_m": 0.01,
    }

    def __init__(self, LeadAgent, params={}):
        import torch
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        super().__init__(LeadAgent, p)
        self._sa = _lib.SubAgentStep()
        self._out = torch.empty((self.n_agents, 2), dtype=torch.float64, device=self.device)

    def update(self, **kwargs):
        """ShiftAgent.update (contribs/SubAgent.py:475-478) for every agent."""
        lead = _current_state(self.LeadAgent)
        self._flush_pending()
        sa = self._sa
        sa.n_agents, sa.id_offset, sa.kind = self.n_agents, int(self.id_offset), _lib.SUBAGENT_SHIFT
        sa.lead_pos, sa.lead_head_direction = lead["pos"].data_ptr(), lead["head_direction"].data_ptr()
        sa.shift_m = float(self.shift_m)
        sa.out_pos = self._out.data_ptr()
        _lib.check(self._lib.riab_subagent_step(C.byref(sa), C.byref(self._env_struct()), None, self._stream()))
        SubAgent.update(self, forced_next_position=self._out)


def _replay_attr(name, col):
    """A ReplayAgent attribute the reference overwrites per replay: the (n_agents,) device column (a scalar when
    n_agents == 1).  Before the device state exists (construction) it holds the parameter's value."""
    def get(self):
        if "_replay_state" not in self.__dict__:
            return self.__dict__["_init_" + name]
        v = self._replay_state[:, col].cpu().numpy()
        return float(v[0]) if self.n_agents == 1 else v

    def set(self, v):
        if "_replay_state" in self.__dict__:
            raise AttributeError(f"ReplayAgent.{name} is per-agent device state and is read-only")
        self.__dict__["_init_" + name] = v
    return property(get, set)


class ReplayAgent(SubAgent):
    """ratinabox.contribs.SubAgent.ReplayAgent (contribs/SubAgent.py:358-431): tracks the lead, except during replays.
    While not replaying, each agent starts a replay with probability replay_freq * dt per step: it jumps to a random
    position and follows a fresh random-motion trajectory of a sham agent at a Rayleigh-drawn ``replay_speed`` (mean
    parameter ``replay_speed``) for a Rayleigh-drawn ``replay_duration`` (at least half its mean parameter), then returns
    to the lead.

    The sham agent's rollout is stepped lazily on the device, only as far as each step's query, which gives the
    reference's interpolated positions with O(1) state per agent.  The sham agent moves with this agent's motion
    parameters and the lead's dt; it is not registered in the Environment.  ``is_undergoing_replay``,
    ``replay_speed``, ``replay_duration``, ``replay_start_time`` and ``replay_end_time`` are read-only (n_agents,)
    arrays (scalars when n_agents == 1); ``history["replay"]`` holds the replay flag after each step.
    """
    default_params = {                                              # contribs/SubAgent.py:360-364
        "replay_freq": 0.3,
        "replay_duration": 0.1,
        "replay_speed": 1.0,
    }
    replay_speed = _replay_attr("replay_speed", 0)
    replay_duration = _replay_attr("replay_duration", 1)
    replay_start_time = _replay_attr("replay_start_time", 2)
    replay_end_time = _replay_attr("replay_end_time", 3)

    def __init__(self, LeadAgent, params={}):
        import torch
        p = copy.deepcopy(__class__.default_params)
        p.update(params)
        super().__init__(LeadAgent, p)
        A = self.n_agents
        self.mean_replay_speed = self.replay_speed                                   # :370-373
        self.mean_replay_duration = self.replay_duration
        f64 = dict(dtype=torch.float64, device=self.device)
        state = torch.full((A, _lib.REPLAY_FIELDS), float("nan"), **f64)
        state[:, 0], state[:, 1] = float(self.mean_replay_speed), float(self.mean_replay_duration)
        self._replaying = torch.zeros(A, dtype=torch.uint8, device=self.device)
        self._replay_count = torch.zeros((A, 2), dtype=torch.int64, device=self.device)
        self._flags = None                        # (history capacity, A) uint8, rows aligned with the history ring's
        # the sham agent (:376-378): Agent.__init__'s initial state; its measured velocity, head direction and distance
        # carry over between replays
        pos = self.Environment.sample_positions(n=A, method="random")
        direction = np.random.uniform(0, 2 * np.pi, size=A)
        vel = self.speed_mean * np.stack((np.cos(direction), np.sin(direction)), axis=1)
        self._sham = {k: torch.zeros_like(self._s[k]) for k in _STATE}
        self._sham["pos"].copy_(torch.as_tensor(pos, **f64))
        self._sham["velocity"].copy_(torch.as_tensor(vel, **f64))
        self._sham["measured_velocity"].copy_(torch.as_tensor(vel, **f64))
        self._sham["head_direction"].copy_(torch.as_tensor(vel / np.linalg.norm(vel, axis=1, keepdims=True), **f64))
        self._sham["distance_to_closest_wall"].fill_(float("inf"))
        self._sham_c = _lib.Agents()
        self._sham_c.n_agents, self._sham_c.id_offset = A, int(self.id_offset)
        for k in _STATE:
            setattr(self._sham_c, k, self._sham[k].data_ptr())
        self._sham_mp = _lib.MotionParams()
        self._sa = _lib.SubAgentStep()
        self._out = torch.empty((A, 2), **f64)
        self._updates = 0
        self._replay_state = state                # from here on the replay attributes read the device

    @property
    def is_undergoing_replay(self):
        v = self._replaying.cpu().numpy().astype(bool)
        return bool(v[0]) if self.n_agents == 1 else v

    def update(self, **kwargs):
        """ReplayAgent.update (contribs/SubAgent.py:380-426) for every agent.  Parity taps: ``_replay_draws``
        (n_agents, 6) = the uniform, replay_speed, the Rayleigh duration before its clamp, the start position (x, y) and
        the start direction, used by agents that are not replaying; ``_xi_replay`` (n_agents, K, 2) standard normals of
        rollout steps 0..K-1 of the current replay."""
        t_before = float(self.t)                   # :399 reads self.t before SubAgent.update sets it
        lead = _current_state(self.LeadAgent)
        self._flush_pending()
        self._sync_user_writes()
        A = self.n_agents
        draws = _tensor_tap(self, kwargs.get("_replay_draws"), (A, 6))
        xi = kwargs.get("_xi_replay")
        xi = _tensor_tap(self, xi, (A, -1, 2)) if xi is not None else None
        self._fill_motion_params(self.dt, {}, mp=self._sham_mp)
        sa = self._sa
        sa.n_agents, sa.id_offset, sa.kind = A, int(self.id_offset), _lib.SUBAGENT_REPLAY
        sa.seed, sa.step = int(self.seed) & 0xFFFFFFFFFFFFFFFF, self._updates
        sa.lead_pos, sa.dt, sa.t = lead["pos"].data_ptr(), float(self.dt), t_before
        sa.p_start = self.replay_freq * self.dt
        sa.mean_speed, sa.mean_duration = float(self.mean_replay_speed), float(self.mean_replay_duration)
        sa.replaying, sa.replay_state = self._replaying.data_ptr(), self._replay_state.data_ptr()
        sa.replay_count, sa.sham = self._replay_count.data_ptr(), self._sham_c
        sa.replay_draws = draws.data_ptr() if draws is not None else None
        sa.xi_replay, sa.xi_steps = (xi.data_ptr(), int(xi.shape[1])) if xi is not None else (None, 0)
        sa.out_pos = self._out.data_ptr()
        _lib.check(self._lib.riab_subagent_step(C.byref(sa), C.byref(self._env_struct()), C.byref(self._sham_mp),
                                                self._stream()))
        self._taps = (draws, xi)                  # the launch reads them asynchronously
        self._updates += 1
        SubAgent.update(self, forced_next_position=self._out)
        if self.save_history:                     # save_to_history (:428-431): the flag after this step
            self._flag_row().copy_(self._replaying)

    def _flag_row(self):
        """The flag ring's row of the history row this step wrote; the ring grows with the Agent's (same capacity,
        rows copied the same way), so its rows wrap in lockstep."""
        import torch
        cap = self._hist_cap
        if self._flags is None or self._flags.shape[0] != cap:
            new = torch.zeros((cap, self.n_agents), dtype=torch.uint8, device=self.device)
            if self._flags is not None:
                new[: self._flags.shape[0]].copy_(self._flags)
            self._flags = new
        return self._flags[(self._hist_rows - 1) % cap]

    def _history_keys(self):
        return super()._history_keys() + ["replay"]

    def get_history_arrays(self):
        """Agent.get_history_arrays plus ``replay``: bool (T,), or (T, n_agents) with more than one agent."""
        import torch
        fresh = self._last_history_array_cache_time != (self.t, self._hist_rows)
        arrays = super().get_history_arrays()
        if fresh or "replay" not in arrays:
            n = min(self._hist_rows, self._hist_cap)
            if n == 0 or self._flags is None:
                flags = np.zeros((n, self.n_agents), dtype=bool)
            else:
                start = self._hist_rows % self._hist_cap if self._hist_rows > self._hist_cap else 0
                idx = (torch.arange(n, device=self.device) + start) % self._hist_cap
                flags = self._flags[idx].cpu().numpy().astype(bool)
            arrays["replay"] = flags[:, 0] if self.n_agents == 1 else flags
        return arrays


class UnrelatedAgent(SubAgent):
    """ratinabox.contribs.SubAgent.UnrelatedAgent (contribs/SubAgent.py:480-489): an independent random walker with the
    lead's dt (and its batch).  It starts from the lead's position and velocity, so with the lead's seed it would repeat
    the lead's path step for step; without a ``seed`` parameter it takes one derived from the lead's."""
    default_params = {}

    def __init__(self, LeadAgent, params={}):
        p = dict(params)
        if "seed" not in p:
            p["seed"] = (int(LeadAgent.seed) * 0x9E3779B97F4A7C15 + 0x554E52454C) & 0xFFFFFFFFFFFFFFFF
        super().__init__(LeadAgent, p)

    def update(self, **kwargs):
        """SubAgent.update() (contribs/SubAgent.py:487-489): the random-motion step; Agent.update's parity tap ``_xi``
        passes through."""
        SubAgent.update(self, **kwargs)

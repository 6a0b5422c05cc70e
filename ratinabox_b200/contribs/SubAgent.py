"""ratinabox.contribs.SubAgent (contribs/SubAgent.py:10-36) and ThetaSequenceAgent (:182-356) on the device.

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
"""
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

"""TEST INFRASTRUCTURE -- NumPy restatement of DumbAgent.update (ratinabox/contribs/SubAgent.py:151-179), ShiftAgent.update
(:475-478) and ReplayAgent.update (:380-426) for one agent, driven by a recorded (or teacher-forced) lead Agent, with
the reference's draws injected.

    dumb = OracleDumb(env, params);            pos = dumb.step(lead_pos, lead_dt, normals, resample_pos=None)
    pos = shift_position(lead_pos, lead_head_direction, shift_m)
    rep = OracleReplay(env, params, dt, sham); pos = rep.step(lead_pos, lead_t, draws, rollout_normals)

``OracleReplay(mode="eager")`` rolls the sham agent out at the start of a replay to its stop distance, as the
reference does; ``mode="lazy"`` (the device's) advances it only as far as each step's query and keeps the last two
samples; on the step the replay ends it finishes the rollout to the stop distance, because the sham agent's state
(its distance travelled above all) carries over into the next replay.  Both give the same positions
(tests/test_oracle_subagents.py).
"""
import numpy as np

from riab_oracle import OracleAgent, TapeRNG, ornstein_uhlenbeck, vector_intercepts
from riab_oracle_tsa import interp_linear

REPLAY_KEYS = ("replay_freq", "replay_duration", "replay_speed")


class OracleDumb:
    def __init__(self, env, params=None):
        p = {"drift_distance": 0.05, "drift_timescale": 3.0, **(params or {})}          # :134-136
        self.env = env
        self.drift_distance, self.drift_timescale = p["drift_distance"], p["drift_timescale"]
        self.displacement = np.zeros(2)                                                  # :145-149
        self.displacement_velocity = np.zeros(2)
        self.tau_v = self.drift_timescale / 2
        self.sigma = np.pi**2 * self.drift_distance / (self.drift_timescale**2)
        self.acceleration_scale = self.sigma / self.drift_distance
        self.cuts = 0                             # steps on which a wall cut the displacement

    def step(self, lead_pos, dt, normals, resample_pos=None):
        """:151-179 with the OU draw's two standard normals; resample_pos: the position a polygon / hole re-draws."""
        lead_pos = np.asarray(lead_pos, dtype=float)
        ou = ornstein_uhlenbeck(dt, self.displacement_velocity, 0.0, self.sigma, self.tau_v, TapeRNG(agent_xi=normals))
        spring = -self.acceleration_scale * self.displacement * dt
        self.displacement_velocity = self.displacement_velocity + (ou + spring)
        self.displacement = self.displacement + self.displacement_velocity * dt
        walls = self.env.walls
        if len(walls):                                                                   # :165-173
            seg = np.array([lead_pos, lead_pos + self.displacement])
            l = vector_intercepts(walls, seg, TapeRNG())[:, 0, :]
            hit = (l[:, 0] > 0) & (l[:, 0] < 1) & (l[:, 1] > 0) & (l[:, 1] < 1)
            if hit.any():
                self.displacement = self.displacement * (0.95 * np.min(l[hit, 1]))
                self.cuts += 1
        pos = lead_pos + self.displacement
        if not self.env.contains(pos):                                                   # Environment.py:855-894
            if not (self.env.is_rectangular and not self.env.holes):
                pos = np.array(resample_pos, dtype=float)
            else:
                pos = self.env.apply_boundary_conditions(pos)
        self.displacement = self.env.vectors_between(pos, lead_pos)[0, 0, :]
        return pos


def shift_position(lead_pos, lead_head_direction, shift_m):
    """:476, with no boundary condition."""
    return np.asarray(lead_pos, dtype=float) + np.asarray(lead_head_direction, dtype=float) * shift_m


class OracleReplay:
    def __init__(self, env, params, dt, sham_state0, mode="lazy"):
        """sham_state0: (measured_velocity, head_direction, distance_travelled) of the sham agent at construction."""
        p = {"replay_freq": 0.3, "replay_duration": 0.1, "replay_speed": 1.0, **params}   # :360-364
        self.env, self.mode, self.dt = env, mode, dt
        self.replay_freq = p["replay_freq"]
        self.mean_replay_speed, self.mean_replay_duration = p["replay_speed"], p["replay_duration"]
        self.replay_speed, self.replay_duration = p["replay_speed"], p["replay_duration"]
        self.replay_start_time = self.replay_end_time = np.nan
        motion = {k: v for k, v in p.items() if k not in REPLAY_KEYS + ("dt",)}
        self.sham = OracleAgent(env, [0.5, 0.5], [1.0, 0.0], {**motion, "dt": dt})           # :376-378
        mv, hd, dist = sham_state0
        self.sham.measured_velocity, self.sham.head_direction = np.array(mv, dtype=float), np.array(hd, dtype=float)
        self.sham.distance_travelled = float(dist)
        self.t = 0.0
        self.is_undergoing_replay = False
        self.max_rollout = 0

    def step(self, lead_pos, lead_t, draws, normals):
        """One update.  draws: (u, replay_speed, Rayleigh duration, x0, y0, direction) (used when not replaying);
        normals: (K, 2) standard normals of the current replay's rollout steps."""
        t = self.t
        pos = np.array(lead_pos, dtype=float)
        if self.is_undergoing_replay is False:
            u, speed, dur, x0, y0, direction = (float(x) for x in draws)
            if not (u > self.replay_freq * self.dt):                                       # :395-414
                self.is_undergoing_replay = True
                self.replay_speed = speed
                self.replay_duration = max(dur, self.mean_replay_duration / 2)
                self.replay_start_time = t
                self.replay_end_time = t + self.replay_duration
                sh = self.sham                                   # initialise_position_and_velocity (Agent.py:523-535)
                sh.pos = np.array([x0, y0])
                sh.velocity = sh.speed_mean * np.array([np.cos(direction), np.sin(direction)])
                sh.rotational_velocity = 0
                self.start = sh.distance_travelled
                self.stop = self.start + 1.1 * self.replay_speed * self.replay_duration
                self.normals = np.asarray(normals, dtype=float).reshape(-1, 2)
                self.k = 0
                self.fd, self.fp = [sh.distance_travelled], [sh.pos.copy()]
                pos = sh.pos.copy()
                if self.mode == "eager":
                    while self.sham.distance_travelled < self.stop:
                        self._advance()
        else:
            if t < self.replay_end_time:                                                  # :416-418
                q = self.replay_speed * (t - self.replay_start_time)
                if self.mode == "eager":
                    out = interp_linear(q, np.array(self.fd) - self.start, np.array(self.fp))
                else:
                    while self.k == 0 or (self.fd[-1] - self.start < q and self.fd[-1] < self.stop):
                        self._advance()
                    d = np.array(self.fd[-2:]) - self.start
                    out = interp_linear(q, d, np.array(self.fp[-2:])) if d[-1] >= q >= d[0] else None
                pos = np.full(2, np.nan) if out is None else out
            else:                                                                         # :420-423
                self.is_undergoing_replay = False
                # the reference's rollout ran to its stop: the sham's state carries over into the next replay
                while self.mode == "lazy" and self.sham.distance_travelled < self.stop:
                    self._advance()
        self.t = lead_t + self.dt                                 # SubAgent.update: t = Lead.t, then t += dt
        return np.asarray(pos, dtype=float)

    def _advance(self):
        xi = self.normals[self.k] if self.k < len(self.normals) else np.zeros(2)
        self.sham.update(TapeRNG(agent_xi=xi))
        self.k += 1
        self.fd.append(self.sham.distance_travelled)
        self.fp.append(self.sham.pos.copy())
        self.max_rollout = max(self.max_rollout, self.k)
        if self.mode == "lazy":                   # O(1): only the last two samples are needed
            del self.fd[:-2], self.fp[:-2]

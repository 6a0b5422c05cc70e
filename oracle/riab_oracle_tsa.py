"""TEST INFRASTRUCTURE -- NumPy restatement of ThetaSequenceAgent.update (ratinabox/contribs/SubAgent.py:245-350) for one
agent, driven by a recorded (or teacher-forced) lead Agent, with the forward rollout's standard normals injected.

    tsa = OracleTSA(env, params, lead_dt, lead_speed_mean, lead_avg_speed, lead_pos0, lead_dist0=0.0)
    pos, raised = tsa.step(lead_pos, lead_vel, lead_rot, lead_dist, lead_t, rollout_normals)

``mode="lazy"`` is the device's semantics: where the reference raises the position is defined (look behind: the two
window rows that bracket the target, NaN before the window; look ahead: NaN past the rollout's end), and the forward
rollout advances only as far as the query.  ``mode="eager"`` rolls the forward agent out to its stop distance at the
first look-ahead step and interpolates in the whole rollout, as the reference does; ``raised`` reports the steps on
which the reference raises.  Both return the same positions where the reference returns (tests/test_oracle_tsa.py).
"""
import numpy as np

from riab_oracle import OracleAgent, TapeRNG

NAN2 = np.array([np.nan, np.nan])


def interp_linear(x, xs, ys):
    """scipy 1.18 interp1d(kind="linear", bounds_error=True)(x) on sorted xs: None where it raises."""
    if len(xs) < 2 or x < xs[0] or x > xs[-1]:
        return None
    j = int(np.searchsorted(xs, x, side="left"))
    j = min(max(j, 1), len(xs) - 1)
    x_lo, x_hi, y_lo, y_hi = xs[j - 1], xs[j], ys[j - 1], ys[j]
    with np.errstate(invalid="ignore", divide="ignore"):
        return ((x - x_lo) / (x_hi - x_lo)) * y_hi + ((x_hi - x) / (x_hi - x_lo)) * y_lo


class OracleTSA:
    def __init__(self, env, params, lead_dt, lead_speed_mean, lead_avg_speed, lead_pos0, lead_dist0=0.0, mode="lazy",
                 fwd_state0=None):
        self.env, self.mode = env, mode
        self.v_sequence = params.get("v_sequence", 5.0)
        self.theta_freq = params.get("theta_freq", 10.0)
        self.theta_frac = params.get("theta_frac", 0.5)
        self.motion = {k: v for k, v in params.items() if k not in ("v_sequence", "theta_freq", "theta_frac", "dt")}
        self.lead_dt, self.avg = lead_dt, lead_avg_speed
        self.T_theta = 1 / self.theta_freq
        self.d_half = ((self.theta_frac / 2) * self.T_theta * self.v_sequence)
        self.last_theta_phase = 0
        self.n_half = int(2 * self.d_half / (lead_speed_mean * lead_dt))
        self.keep_count = max(1, (20 * self.n_half))
        self.counter = 1
        self.rows = []                   # every lead (distance, x, y) row appended since construction
        self.fwd = None
        self.fwd_state0 = fwd_state0     # (measured_velocity, head_direction) the first rollout starts from
        self.rollouts = []               # per rollout: (distances, positions) of the steps taken

    def window(self):
        lookback = int(5 * self.d_half / (self.lead_dt * self.avg))
        w = min(lookback, self.counter)
        r = np.array(self.rows[len(self.rows) - w:]) if w > 0 else np.zeros((0, 3))
        return r[:, 0], r[:, 1:]

    def look_behind(self, target):
        d, p = self.window()
        if len(d) == 0:
            return NAN2.copy(), True
        idx = int(np.argmin(np.abs(d - target)))
        raised = True
        if idx >= 3:
            out = interp_linear(target, d[idx - 3: idx + 3], p[idx - 3: idx + 3])
            if out is not None:
                return out, False
        elif len(d) < 6:
            sl = slice(idx - 3, idx + 3)
            raised = interp_linear(target, d[sl], p[sl]) is None
            assert raised, "a window of fewer than 6 rows that the reference interpolates: not modelled"
        out = interp_linear(target, d, p)
        return (NAN2.copy() if out is None else out), raised

    def _forward_step(self, xi):
        self.fwd.update(TapeRNG(agent_xi=xi), dt=self.lead_dt * self.v_sequence / self.avg, **self.fwd_kwargs)

    def step(self, lead_pos, lead_vel, lead_rot, lead_dist, lead_t, normals, fwd_kwargs=None):
        """One update.  normals: (K, 2) standard normals of the current rollout's steps (used from its first step)."""
        if self.counter == self.keep_count:
            self.counter = 10 * self.n_half
        self.rows.append((float(lead_dist), float(lead_pos[0]), float(lead_pos[1])))
        theta_phase = (lead_t % (1 / self.theta_freq)) / ((1 / self.theta_freq))
        pos, raised = NAN2.copy(), False
        if (theta_phase >= (0.5 - self.theta_frac / 2)) and (theta_phase < 0.5):
            if lead_dist < self.d_half:
                pos = np.array(lead_pos, dtype=float)
            else:
                c = self.d_half / self.theta_frac
                m = -2 * c
                distance_back = (m * theta_phase + c)
                pos, raised = self.look_behind(lead_dist - distance_back)
        if (theta_phase >= 0.5) and (theta_phase < 0.5 + self.theta_frac / 2):
            if (theta_phase >= 0.5 and self.last_theta_phase < 0.5):
                self.fwd_kwargs = dict(fwd_kwargs or {})
                prev = self.fwd
                self.fwd = OracleAgent(self.env, lead_pos, lead_vel, {"dt": self.lead_dt, **self.motion})
                if prev is not None:
                    self.fwd.measured_velocity, self.fwd.head_direction = prev.measured_velocity, prev.head_direction
                elif self.fwd_state0 is not None:
                    self.fwd.measured_velocity, self.fwd.head_direction = (np.array(v, dtype=float) for v in self.fwd_state0)
                self.fwd.rotational_velocity = float(lead_rot)
                self.fwd.distance_travelled = float(lead_dist)
                self.stop = lead_dist + (self.d_half + 100 * self.avg * (self.theta_frac / 2) * self.T_theta)
                self.k = 0
                self.fd, self.fp = [self.fwd.distance_travelled], [self.fwd.pos.copy()]
                self.normals = np.asarray(normals, dtype=float).reshape(-1, 2)
                self.rollouts.append((self.fd, self.fp))
                if self.mode == "eager":
                    while self.fwd.distance_travelled < self.stop:
                        self._advance()
            c = -self.d_half / self.theta_frac
            m = -2 * c
            distance_ahead = (m * theta_phase + c)
            q = lead_dist + distance_ahead
            if self.mode == "eager":
                out = interp_linear(q, np.array(self.fd), np.array(self.fp))
                pos, raised = (NAN2.copy(), True) if out is None else (out, False)
            else:
                while self.k == 0 or (self.fd[-1] < q and self.fd[-1] < self.stop):
                    self._advance()
                raised = q > self.fd[-1] or q < self.fd[0]
                if self.fd[-1] >= q and q >= self.fd[-2]:
                    pos = interp_linear(q, np.array(self.fd[-2:]), np.array(self.fp[-2:]))
        if not np.isnan(pos).any():
            dist = np.linalg.norm(self.env.vectors_between(pos, lead_pos), axis=-1)[0, 0]
            if dist > self.d_half:
                pos = NAN2.copy()
        self.last_theta_phase = theta_phase
        self.counter += 1
        return np.asarray(pos, dtype=float), raised

    def _advance(self):
        xi = self.normals[self.k] if self.k < len(self.normals) else np.zeros(2)
        self._forward_step(xi)
        self.k += 1
        self.fd.append(self.fwd.distance_travelled)
        self.fp.append(self.fwd.pos.copy())

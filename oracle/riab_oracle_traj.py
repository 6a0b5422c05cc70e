"""Float64 restatement of the imported / forced branches of Agent.update (ratinabox/Agent.py:202-259, :444-507) and of
Agent.import_trajectory (:543-659), on top of the random-motion oracle (riab_oracle.OracleAgent).

The trajectory is interpolated with scipy's interp1d(kind="cubic", fill_value="extrapolate") as the reference does.  The
zero-displacement fall-back (the reference's ``1e-8 * np.random.randn(2)``, :460-461) is an input, like mode A's injected
normals: ``update(fallback=v)`` uses v (already scaled) when the measured velocity is exactly zero.
"""
import numpy as np
from scipy.interpolate import interp1d

from riab_oracle import OracleAgent, get_angle, pi_domain


class OracleTrajAgent(OracleAgent):
    use_imported_trajectory = False

    def import_trajectory(self, times, positions):
        """Agent.py:543-659 with arrays, interpolate=True, 2D, solid boundaries."""
        assert self.env.boundary_conditions == "solid", "Only solid boundary conditions are supported"
        times, positions = np.array(times, dtype=float), np.array(positions, dtype=float)
        assert len(positions) == len(times), "time and position arrays must have same length"
        times = times - min(times)
        positions = positions.reshape(-1, 2)
        self.t_interp = times
        self.pos_interp = interp1d(times, positions, axis=0, kind="cubic", fill_value="extrapolate")
        self.use_imported_trajectory = True
        self.pos = self.pos_interp(0)
        self.prev_pos = self.pos.copy()

    def update(self, rng=None, dt=None, drift_velocity=None, drift_to_random_strength_ratio=1, fallback=(0.0, 0.0),
               **kwargs):
        """Agent.update; the random branch is OracleAgent.update (it needs ``rng``)."""
        forced = kwargs.get("forced_next_position", None)
        if not self.use_imported_trajectory and forced is None:
            return OracleAgent.update(self, rng, dt, drift_velocity, drift_to_random_strength_ratio, **kwargs)
        dt = dt or self.dt
        self.dt = dt
        self.prev_t = self.t
        self.t += dt
        self.pos = np.array(self.pos, dtype=float)
        self.velocity = np.array(self.velocity, dtype=float)
        self.prev_pos = self.pos.copy()
        self.prev_measured_velocity = self.measured_velocity.copy()
        if self.use_imported_trajectory:                                     # Agent.py:223-225, :255-259
            self.pos = self.pos_interp(self.t % max(self.t_interp))
        else:                                                                # Agent.py:229-232, :244-253
            assert isinstance(forced, np.ndarray), "forced_next_position must be an np.array"
            assert forced.shape == (2,), "forced_next_position must be an np.array of shape Env.D"
            self.pos = forced
        self._measure_overwrite(np.asarray(fallback, dtype=float))
        self._update_head_direction()
        if not (np.isnan(self.pos).any() or np.isnan(self.prev_pos).any()):   # Agent.py:502-507
            self._update_distance_travelled()
        if self.save_history:
            self._save_to_history()
        return {}

    def _measure_overwrite(self, fallback):
        """_measure_velocity_of_step_taken(overwrite_velocity=True), Agent.py:444-472."""
        if np.isnan(self.pos).any() or np.isnan(self.prev_pos).any():
            self.measured_velocity = np.full((2,), np.nan)
            self.measured_rotational_velocity = np.nan
            return
        self.measured_velocity = self.env.vectors_between(self.pos, self.prev_pos).reshape(-1) / self.dt
        if np.linalg.norm(self.measured_velocity) == 0:
            self.measured_velocity = fallback.copy()
        self.velocity = self.measured_velocity.copy()
        now, before = get_angle(self.measured_velocity), get_angle(self.prev_measured_velocity)
        self.measured_rotational_velocity = float(pi_domain(now - before)) / self.dt
        self.rotational_velocity = self.measured_rotational_velocity

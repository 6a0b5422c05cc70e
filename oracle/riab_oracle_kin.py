"""Float64 restatement of the kinematic cells, HeadDirectionCells (ratinabox/Neurons.py:2357-2485), VelocityCells
(:2534-2583) and SpeedCell (:2586-2651), with utils.get_angle (utils.py:231-273) and utils.von_mises (:441-457) in the
reference's operation order.  One vector (2,) per call, like the reference; ``*_rows`` apply it per row."""
import numpy as np


def get_angle(v):
    """utils.get_angle of one (2,) vector: mod(arctan2(y, x + 1e-6), 2 pi)."""
    s = np.array(v).reshape(1, 2)
    return np.mod(np.arctan2(s[:, 1], (s[:, 0] + 1e-6)), 2 * np.pi)[0]


def von_mises_norm1(theta, mu, sigma):
    """utils.von_mises(theta, mu, sigma, norm=1): exp(kappa cos(theta - mu)) * (1 / exp(kappa)), kappa = 1 / sigma^2."""
    kappa = 1 / (sigma ** 2)
    v = np.exp(kappa * np.cos(theta - mu))
    norm = 1 / np.exp(kappa)
    return v * norm


def default_tuning(n, angular_spread_degrees):
    """Neurons.py:2405-2409."""
    return np.linspace(0, 2 * np.pi, n + 1)[:-1], np.array([angular_spread_degrees * np.pi / 180] * n)


def head_direction_rates(direction, preferred_angles, angular_tunings, min_fr=0, max_fr=1, n_pos=1, use_velocity=False):
    """HeadDirectionCells.get_state (2D) for one head direction (or, with use_velocity, one velocity) -> (n, n_pos)."""
    direction = np.asarray(direction)
    if use_velocity:
        direction = direction / np.linalg.norm(direction)
    fr = von_mises_norm1(get_angle(direction), preferred_angles, angular_tunings)
    fr = fr * (max_fr - min_fr) + min_fr
    return np.tile(fr, (n_pos, 1)).T


def velocity_rates(velocity, agent_velocity, one_sigma_speed, preferred_angles, angular_tunings, min_fr=0, max_fr=1,
                   n_pos=1):
    """VelocityCells.get_state: the use_velocity rates of `velocity` times |agent_velocity| / one_sigma_speed."""
    fr = head_direction_rates(velocity, preferred_angles, angular_tunings, min_fr, max_fr, n_pos, use_velocity=True)
    return fr * (np.linalg.norm(agent_velocity) / one_sigma_speed)


def speed_rate(vel, one_sigma_speed, min_fr=0, max_fr=1):
    """SpeedCell.get_state -> (1,): the norm is taken over the whole array."""
    fr = np.array([np.linalg.norm(np.array(vel)) / one_sigma_speed])
    return fr * (max_fr - min_fr) + min_fr


def head_direction_rows(directions, preferred_angles, angular_tunings, min_fr=0, max_fr=1, use_velocity=False):
    """One column per row of `directions` (m, 2) -> (n, m)."""
    return np.stack([head_direction_rates(d, preferred_angles, angular_tunings, min_fr, max_fr, 1, use_velocity)[:, 0]
                     for d in np.asarray(directions).reshape(-1, 2)], axis=1)


def velocity_rows(velocities, one_sigma_speed, preferred_angles, angular_tunings, min_fr=0, max_fr=1, scale_by=None):
    """VelocityCells per row; the speed factor is each row's own |velocity| (the rates at the agents) unless scale_by gives
    the agent velocity of every row."""
    cols = []
    for v in np.asarray(velocities).reshape(-1, 2):
        cols.append(velocity_rates(v, v if scale_by is None else scale_by, one_sigma_speed, preferred_angles, angular_tunings,
                                   min_fr, max_fr)[:, 0])
    return np.stack(cols, axis=1)


def speed_rows(velocities, one_sigma_speed, min_fr=0, max_fr=1):
    return np.stack([speed_rate(v, one_sigma_speed, min_fr, max_fr) for v in np.asarray(velocities).reshape(-1, 2)], axis=1)

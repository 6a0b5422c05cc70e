"""Float64 restatement of PhasePrecessingPlaceCells (ratinabox/contribs/PhasePrecessingPlaceCells.py:10-119): the PlaceCells
rate of riab_oracle.place_cells_get_state times the theta modulation factor, with utils.von_mises (utils.py:441-457) and
utils.get_vectors_between (utils.py:203-215) in the reference's operation order.  Per agent: one position, one velocity and
the Agent's clock ``t``."""
import numpy as np

import riab_oracle as O

DEFAULTS = {"n": 10, "min_fr": 0, "max_fr": 1, "theta_freq": 10, "kappa": 1, "precess_fraction": 0.5,
            "description": "gaussian_threshold", "name": "PhasePrecessingPlaceCell"}          # :33-42
MESSAGE = ("Since you are not evaluating hte firing rate using the current state of the agent no phase precession modulation "
           "has been applied (since this requires a velocity). Ignore this if you are plotting receptive field. ")   # :88-90


def von_mises(theta, mu, sigma):
    """utils.von_mises(theta, mu, sigma, norm=None): the normalised density (utils.py:452-457)."""
    from scipy.special import i0
    kappa = 1 / (sigma ** 2)
    v = np.exp(kappa * np.cos(theta - mu))
    norm = np.exp(kappa) / (2 * np.pi * i0(kappa))
    norm = norm / np.exp(kappa)
    return v * norm


def theta_modulation_factors(pos, velocity, t, centres, widths, description, theta_freq, sigma, precess_fraction):
    """:94-119 for one agent -> (n, 1)."""
    position = np.asarray(pos, dtype=float)
    velocity = np.asarray(velocity, dtype=float)
    direction = velocity / (1e-8 + np.linalg.norm(velocity))                                 # :99
    theta_phase = theta_freq * (t % (1 / theta_freq)) * 2 * np.pi                            # :100-102
    s = np.array(widths, dtype=float).copy()                                                 # :103-105
    if description == "gaussian":
        s *= 2
    vectors_to_cells = position.reshape(-1, 2)[:, None, :] - np.asarray(centres, dtype=float).reshape(-1, 2)[None, :, :]
    sigmas_to_cell_midline = np.dot(vectors_to_cells, direction) / s                          # :107-110
    prefered_theta_phase = np.pi - sigmas_to_cell_midline * precess_fraction * np.pi        # :111-113
    phase_diff = prefered_theta_phase - theta_phase
    return (von_mises(phase_diff, mu=0, sigma=sigma) * 2 * np.pi).T                           # :115-117


def get_state_agent(env, pos, velocity, t, centres, widths, rng, description, wall_geometry, min_fr, max_fr, theta_freq,
                    sigma, precess_fraction, scalar_width=None):
    """get_state(evaluate_at="agent") for one agent -> (n, 1): the PlaceCells rate times the factors (:82-86)."""
    fr = O.place_cells_get_state(env, centres, widths, pos, rng, description, wall_geometry, min_fr, max_fr,
                                 scalar_width=scalar_width)
    return fr * theta_modulation_factors(pos, velocity, t, centres, widths, description, theta_freq, sigma, precess_fraction)


def get_state_rows(env, pos, velocity, t, centres, widths, rng, description, wall_geometry, min_fr, max_fr, theta_freq,
                   sigma, precess_fraction, scalar_width=None):
    """One column per agent row of pos / velocity (m, 2) -> (n, m)."""
    return np.concatenate([get_state_agent(env, p, v, t, centres, widths, rng, description, wall_geometry, min_fr, max_fr,
                                           theta_freq, sigma, precess_fraction, scalar_width)
                           for p, v in zip(np.asarray(pos).reshape(-1, 2), np.asarray(velocity).reshape(-1, 2))], axis=1)


def peak_factor(sigma):
    """M = exp(kappa) / I0(kappa), kappa = 1 / sigma^2: the largest factor (phase difference 0)."""
    return float(von_mises(0.0, 0.0, sigma) * 2 * np.pi)

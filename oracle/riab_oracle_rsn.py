"""Float64 restatement of RandomSpatialNeurons (ratinabox/Neurons.py:2865-2954) on top of riab_oracle's geometry:
the sample grid, the covariance of the set-up, and get_state's kernel-weighted average of the targets.  ``rng`` is
riab_oracle.GlobalRNG (the reference's jitter draws) or TapeRNG (zero jitter, the configuration the device is held to)."""
import numpy as np

import riab_oracle as O


def sample_grid(extent, lengthscale):
    """Environment.discretise_environment(dx=min(0.05, lengthscale)) (Environment.py:635-655) flattened to (|X|, 2)."""
    dx = min(0.05, lengthscale)
    x = np.arange(extent[0] + dx / 2, extent[1], dx)
    y = np.arange(extent[2] + dx / 2, extent[3], dx)[::-1]
    xm, ym = np.meshgrid(x, y)
    return np.stack((xm, ym), axis=-1).reshape(-1, 2)


def distances(env, x1, x2, wall_geometry, rng):
    """Environment.py:677-779, with the reference's assertion for walls in a periodic environment (:711-713, :733-735)."""
    if wall_geometry != "euclidean":
        assert env.boundary_conditions == "solid", f"{wall_geometry} geometry is not available for periodic boundary conditions"
    return O.distances_accounting_for_environment(env, x1, x2, wall_geometry, rng)


def kernel(env, x1, x2, lengthscale, wall_geometry, rng):
    """Neurons.py:2944-2954: exp(-d^2 / (2 l^2))."""
    d = distances(env, x1, x2, wall_geometry, rng)
    return np.exp(-(d ** 2) / (2 * lengthscale ** 2))


def targets_from(Q, n, min_fr=0.0, max_fr=1.0):
    """Neurons.py:2909-2913: multivariate_normal(0, Q, size=n).T through utils.activate's sigmoid (mid_x 0, width_x 2)."""
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", category=RuntimeWarning)
        t = np.random.multivariate_normal(mean=np.zeros(Q.shape[0]), cov=Q, size=n).T
    beta = np.log((1 - 0.05) / 0.05) / (0.5 * 2)
    return ((max_fr - min_fr) / (1 + np.exp(-beta * (t - 0)))) + min_fr


def get_state(env, X, targets, lengthscale, wall_geometry, pos, rng):
    """Neurons.py:2923-2941 -> (n, n_pos)."""
    k = kernel(env, np.asarray(pos, dtype=float).reshape(-1, 2), X, lengthscale, wall_geometry, rng)
    k = k / np.sum(k, axis=1, keepdims=True)
    return (k @ targets).T

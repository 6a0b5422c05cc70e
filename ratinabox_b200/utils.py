"""Host-side set-up helpers (one-off parameter sampling; not on the per-step path).

These follow the semantics of the reference's helpers so that populations built
with the same params and NumPy seed get the same parameters:
``utils.rotate`` (ratinabox/utils.py:293-301), ``utils.distribution_sampler``
(:460-538) and ``utils.create_random_assembly`` (:1115-1219).
"""
import numpy as np


def rotate(vector, theta):
    c, s = np.cos(theta), np.sin(theta)
    return np.matmul(np.array([[c, -s], [s, c]]), vector)


def distribution_sampler(distribution_name="uniform", distribution_parameters=(1,), shape=(10,)):
    prm = distribution_parameters
    prm = tuple(prm) if isinstance(prm, (list, tuple)) else (prm,)
    if distribution_name == "uniform":
        low, high = (0.5 * prm[0], 1.5 * prm[0]) if len(prm) == 1 else (prm[0], prm[1])
        return np.random.uniform(low, high, size=shape)
    if distribution_name == "rayleigh":
        return np.random.rayleigh(scale=prm[0], size=shape)
    if distribution_name == "normal":
        return np.random.normal(loc=prm[0], scale=prm[1], size=shape)
    if distribution_name == "logarithmic":
        assert len(shape) == 1, "Logarithmic distribution only works for 1D arrays"
        return np.logspace(np.log10(prm[0]), np.log10(prm[1]), num=shape[0], base=10)
    if distribution_name == "delta":
        return prm[0] * np.ones(shape)
    if distribution_name == "modules":
        assert len(shape) == 1, "Modules distribution only works for 1D arrays"
        per = shape[0] // len(prm)
        out = prm[-1] * np.ones(shape)          # remainder goes to the last module
        for i, val in enumerate(prm):
            out[i * per:(i + 1) * per] = val
        return out
    if distribution_name == "truncnorm":
        import scipy.stats
        lower, upper, mu, sigma = prm[:4]
        return scipy.stats.truncnorm.rvs((lower - mu) / sigma, (upper - mu) / sigma, scale=sigma, loc=mu, size=shape)
    raise ValueError("This distribution is not recognised")


def create_random_assembly(tuning_distance_distribution="uniform", tuning_distance=(0.02, 0.3),
                           tuning_angle_distribution="uniform", tuning_angle=(0.0, 360.0),
                           sigma_angle_distribution="uniform", sigma_angle=(10, 30),
                           sigma_distance_distribution="diverging", sigma_distance=(0.08, 12), n=10, **kwargs):
    """Random vector-cell tuning: (tuning_distance, tuning_angle [rad], sigma_distance, sigma_angle [rad]).
    Draw order (distance, [sigma_d], angle, sigma_angle) matches the reference so seeds line up."""
    given = [p for p in (tuning_distance, tuning_angle, sigma_distance, sigma_angle) if type(p) in (list, np.ndarray)]
    if given:
        lengths = {len(p) for p in given}
        assert len(lengths) == 1, "If more than one parameter is passed as a list, they must all have the same length"
        n = lengths.pop()

    def draw(value, dist):
        if type(value) in (list, np.ndarray):
            return np.array(value, dtype=float)
        return distribution_sampler(dist, value, (n,))

    mu_d = np.abs(draw(tuning_distance, tuning_distance_distribution))
    if type(sigma_distance) in (list, np.ndarray):
        sg_d = np.array(sigma_distance, dtype=float)
    elif sigma_distance_distribution == "diverging":
        sg_d = sigma_distance[0] + mu_d / sigma_distance[1]        # Hartley: xi + mu/beta
    else:
        sg_d = distribution_sampler(sigma_distance_distribution, sigma_distance, (n,))
    mu_t = draw(tuning_angle, tuning_angle_distribution) * (np.pi / 180)
    sg_t = draw(sigma_angle, sigma_angle_distribution) * (np.pi / 180)
    return mu_d, mu_t, sg_d, sg_t


def create_uniform_radial_assembly(distance_range=(0.0, 0.2), angle_range=(0, 90), spatial_resolution=0.04, **kwargs):
    """Concentric rows of equally sized receptive fields tiling a field of view (the reference's
    utils.create_uniform_radial_assembly, ratinabox/utils.py:1033-1070)."""
    lo, hi = (a * np.pi / 180 for a in angle_range)
    mu_d, mu_t, sg_d, sg_t = [], [], [], []
    for radius in np.arange(max(0.01, distance_range[0]), distance_range[1], spatial_resolution):
        dtheta = spatial_resolution / radius
        right = np.arange(lo + dtheta / 2, hi, dtheta)
        for theta in np.concatenate((-right[::-1], right)):
            mu_d.append(radius); mu_t.append(theta); sg_d.append(spatial_resolution); sg_t.append(spatial_resolution / radius)
    return mu_d, mu_t, sg_d, sg_t


def create_diverging_radial_assembly(distance_range=(0.01, 0.2), angle_range=(0, 90), spatial_resolution=0.04,
                                     beta=5, **kwargs):
    """Rows whose receptive fields grow with radius (Hartley et al. 2000): sigma_d = xi + radius/beta with xi fixed
    by the innermost row (the reference's utils.create_diverging_radial_assembly, ratinabox/utils.py:1073-1112)."""
    lo, hi = (a * np.pi / 180 for a in angle_range)
    mu_d, mu_t, sg_d, sg_t = [], [], [], []
    radius = max(0.01, distance_range[0])
    xi = spatial_resolution - radius / beta
    while radius < distance_range[1]:
        res = xi + radius / beta
        dtheta = res / radius
        right = np.array([lo + dtheta / 2]) if dtheta / 2 > hi else np.arange(lo + dtheta / 2, hi, dtheta)
        for theta in np.concatenate((-right[::-1], right)):
            mu_d.append(radius); mu_t.append(theta); sg_d.append(res); sg_t.append(res / radius)
        radius = (2 * radius + res + xi) / (2 - 1 / beta)      # next row just touches this one
    return mu_d, mu_t, sg_d, sg_t


def bin_data_for_histogramming(data, extent, dx, weights=None, norm_by_bincount=False, return_zero_bins=False):
    """ratinabox.utils.bin_data_for_histogramming, 2D branch (utils.py:544-589): np.histogram2d over
    np.arange(extent[0], extent[1] + dx, dx) x np.arange(extent[2], extent[3] + dx, dx), optionally weighted and
    divided by the bin count, returned `.T[::-1, :]`.  Host NumPy; the device path over the history rings is
    ``Agent.get_position_heatmap`` / ``Neurons.get_history_rate_maps``."""
    assert len(extent) == 4, "2D only"
    data = np.asarray(data, dtype=float)
    bins_x = np.arange(extent[0], extent[1] + dx, dx)
    bins_y = np.arange(extent[2], extent[3] + dx, dx)
    heatmap, _, _ = np.histogram2d(data[:, 0], data[:, 1], bins=[bins_x, bins_y], weights=weights)
    zero_bins = None
    if norm_by_bincount:
        bincount, _, _ = np.histogram2d(data[:, 0], data[:, 1], bins=[bins_x, bins_y])
        zero_bins = (bincount == 0)
        bincount[zero_bins] = 1
        heatmap = heatmap / bincount
    heatmap = heatmap.T[::-1, :]
    if return_zero_bins:
        return (heatmap, zero_bins.T[::-1, :])
    return heatmap


# ------------------------------------------------------------------------------------------------- environment geometry
# Host float64 restatements of the reference's pairwise-distance helpers, for set-up computations that must consume the
# same global NumPy draws as the reference (RandomSpatialNeurons' covariance): same operations, same order, same draws.
def vector_intercepts(vector_list_a, vector_list_b, return_collisions=False):
    """utils.vector_intercepts (utils.py:30-118): the intersection parameters (l_a, l_b) of every pair of segments
    a (N_a,2,2) and b (N_b,2,2) -> (N_a,N_b,2), or with ``return_collisions`` the mask 0 < l_a, l_b < 1.  Both lists
    are jittered by N(0, 1e-9) draws first, a's then b's, like the reference."""
    a = np.asarray(vector_list_a, dtype=float).reshape(-1, 2, 2)
    b = np.asarray(vector_list_b, dtype=float).reshape(-1, 2, 2)
    a = a + np.random.normal(scale=1e-9, size=a.shape)
    b = b + np.random.normal(scale=1e-9, size=b.shape)
    d0 = b[None, :, 0, :] - a[:, None, 0, :]                  # (N_a,N_b,2)
    sa = (a[:, 1, :] - a[:, 0, :])[:, None, :]
    sb = (b[:, 1, :] - b[:, 0, :])[None, :, :]
    sa_px, sa_py = -sa[..., 1], sa[..., 0]                    # [x,y]_p = [-y,x]
    sb_px, sb_py = -sb[..., 1], sb[..., 0]
    with np.errstate(divide="ignore", invalid="ignore"):     # parallel segments: inf / nan, never inside (0, 1)
        l_a = (d0[..., 0] * sb_px + d0[..., 1] * sb_py) / (sa[..., 0] * sb_px + sa[..., 1] * sb_py)
        l_b = ((-d0[..., 0]) * sa_px + (-d0[..., 1]) * sa_py) / (sb[..., 0] * sa_px + sb[..., 1] * sa_py)
    if return_collisions:
        return (l_a > 0) & (l_a < 1) & (l_b > 0) & (l_b < 1)
    return np.stack((l_a, l_b), axis=-1)


def get_distances_between___accounting_for_environment(env, pos1, pos2, wall_geometry="euclidean"):
    """Environment.get_distances_between___accounting_for_environment (Environment.py:677-779), 2D: (N,M) distances
    from pos1 (N,2) to pos2 (M,2).  Periodic boundaries wrap the difference vectors; line_of_sight sets the distance of
    pairs whose segment crosses one of ``walls[4:]`` to 1000; geodesic (at most one wall after the first four) replaces
    a blocked distance by the shortest detour via an end of that wall that lies inside the environment."""
    pos1 = np.asarray(pos1, dtype=float).reshape(-1, 2)
    pos2 = np.asarray(pos2, dtype=float).reshape(-1, 2)
    vectors = pos1[:, None, :] - pos2[None, :, :]
    if env.boundary_conditions == "periodic":
        flip = np.abs(vectors) > (env.scale / 2)
        vectors[flip] = -np.sign(vectors[flip]) * (env.scale - np.abs(vectors[flip]))
    distances = np.linalg.norm(vectors, axis=-1)
    if wall_geometry == "euclidean":
        return distances
    segments = np.stack((np.broadcast_to(pos1[:, None, :], vectors.shape),
                         np.broadcast_to(pos2[None, :, :], vectors.shape)), axis=-2).reshape(-1, 2, 2)
    walls = env.walls
    if wall_geometry == "line_of_sight":
        assert env.boundary_conditions == "solid", "line of sight geometry not available for periodic boundary conditions"
        blocked = vector_intercepts(segments, walls[4:], return_collisions=True)
        blocked = (blocked.sum(axis=-1) != 0).reshape(distances.shape)
        distances[blocked] = 1000
        return distances
    if wall_geometry == "geodesic":
        assert env.boundary_conditions == "solid", "geodesic geometry is not available for periodic boundary conditions"
        assert len(walls) <= 5, ("unfortunately geodesic geometry is only defined in closed rooms with one additional "
                                 "wall. Try using \"line_of_sight\" or \"euclidean\" instead.")
        if len(walls) == 4:
            return distances
        wall = walls[4]
        via = []
        for end in wall:
            if env.check_if_position_is_in_environment(end):
                e = end.reshape(1, 2)
                via.append(np.linalg.norm(pos1[:, None, :] - e[None, :, :], axis=-1)
                           + np.linalg.norm(e[:, None, :] - pos2[None, :, :], axis=-1))
        via = np.array(via)
        blocked = vector_intercepts(segments, np.expand_dims(wall, axis=0), return_collisions=True).reshape(distances.shape)
        distances[blocked] = np.amin(via, axis=0)[blocked]
        return distances
    raise ValueError(f"unknown wall_geometry {wall_geometry!r}")


def sigmoid(x, max_fr=1, min_fr=0, mid_x=1, width_x=2):
    """utils.activate(x, "sigmoid") (utils.py:961-977): (max_fr - min_fr) / (1 + exp(-beta (x - mid_x))) + min_fr with
    beta = log(19) / (width_x / 2), so that width_x spans the 5 % to 95 % rise."""
    beta = np.log((1 - 0.05) / 0.05) / (0.5 * width_x)
    return ((max_fr - min_fr) / (1 + np.exp(-beta * (x - mid_x)))) + min_fr

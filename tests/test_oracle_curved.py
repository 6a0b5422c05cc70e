"""Curved environments made of many short walls (tests/golden/curved.npz, from the live reference): the README's
100-wall circular arena and the successor-features demo's 200-wall loop track.  The NumPy oracle reproduces the
reference bit for bit there, and the host mirror's vectorised in-environment test decides exactly as the scalar one."""
import numpy as np
import pytest

import riab_oracle as O


def circle(r, n=100):
    return [[r * np.cos(t), r * np.sin(t)] for t in np.linspace(0, 2 * np.pi, n)]


CURVED_CASES = {"circle": dict(boundary=circle(0.5)), "annulus": dict(boundary=circle(0.5), holes=[circle(0.4)])}


@pytest.mark.parametrize("name", sorted(CURVED_CASES))
def test_curved_environment_golden(golden, name):
    """The oracle against the reference in the circle / annulus: wall list, a native 1000-step run (global RNG, jitter
    on) with Euclidean PlaceCells and BVCs bit for bit, and 384 teacher-forced single steps (half of them at an edge at
    speed, some at the 1.2e-16 m closing edge) with the rates at their start positions."""
    g = golden("curved.npz")
    env = O.OracleEnvironment(**CURVED_CASES[name])
    assert np.array_equal(env.walls, g[f"{name}_walls"]) and np.array_equal(env.extent, g[f"{name}_extent"])
    assert len(env.walls) == (100 if name == "circle" else 200)
    assert 0.0 < np.linalg.norm(env.walls[99, 0] - env.walls[99, 1]) < 1e-15          # the closing edge
    assert str(g[f"{name}_default_geom"]) == "line_of_sight"
    prm = {"dt": 0.02, "speed_mean": 0.25}
    ag = O.OracleAgent(env, g[f"{name}_pos0"], g[f"{name}_vel0"], prm)
    rng = O.GlobalRNG()
    td, ta, sd, sa = g[f"{name}_bvc"]
    pcs = O.OracleNeurons(ag, 24, lambda p, r: O.place_cells_get_state(env, g[f"{name}_centres"], g[f"{name}_widths"], p, r,
                                                                       "gaussian", "euclidean"))
    bvcs = O.OracleNeurons(ag, 6, lambda p, r: O.bvc_get_state(env, td, ta, sd, sa, p, r))
    np.random.set_state(("MT19937", g[f"{name}_rng_keys"], int(g[f"{name}_rng_pos"]), int(g[f"{name}_rng_has_gauss"]),
                         float(g[f"{name}_rng_cached"])))
    for _ in range(1000):
        ag.update(rng); pcs.update(rng); bvcs.update(rng)
    assert np.array_equal(np.array(ag.history["pos"]), g[f"{name}_pos"])
    assert np.array_equal(np.array(ag.history["vel"]), g[f"{name}_vel"])
    assert np.array_equal(np.array(pcs.history["firingrate"]), g[f"{name}_pc_fr"])
    assert np.array_equal(np.array(bvcs.history["firingrate"]), g[f"{name}_bvc_fr"])
    assert all(env.contains(p) for p in g[f"{name}_pos"])
    for a in range(len(g[f"{name}_A_pos0"])):
        assert env.contains(g[f"{name}_A_pos0"][a])
        oa = O.OracleAgent(env, g[f"{name}_A_pos0"][a], g[f"{name}_A_vel0"][a], prm)
        oa.update(O.TapeRNG(agent_xi=g[f"{name}_A_xi"][a]))
        assert np.array_equal(oa.pos, g[f"{name}_A_pos"][a]) and np.array_equal(oa.velocity, g[f"{name}_A_vel"][a])
        assert np.array_equal(oa.measured_velocity, g[f"{name}_A_mv"][a])
    bounced = np.abs(np.linalg.norm(g[f"{name}_A_vel"], axis=1) - 0.5 * 0.25) < 1e-12
    assert bounced.sum() >= 40
    fr = O.place_cells_get_state(env, g[f"{name}_centres"], g[f"{name}_widths"], g[f"{name}_A_pos0"], O.TapeRNG(),
                                 "gaussian", "euclidean")
    assert np.array_equal(fr, g[f"{name}_A_pc"])
    assert np.array_equal(O.bvc_get_state(env, td, ta, sd, sa, g[f"{name}_A_pos0"], O.TapeRNG()), g[f"{name}_A_bvc"])


def _probe_points(verts, rs):
    """About 10^5 points that stress the predicate: every vertex, edge midpoints, points 1 ulp off the edges and
    vertices, points on the edges' lines, the closing edge, and uniform points in and around the polygon."""
    v = np.asarray(verts, dtype=float)
    nxt = np.roll(v, -1, axis=0)
    mids = 0.5 * (v + nxt)
    pts = [v, mids, nxt]
    for p in (v, mids):
        for dx in (-1, 0, 1):
            for dy in (-1, 0, 1):
                pts.append(np.stack((np.nextafter(p[:, 0], p[:, 0] + dx) if dx else p[:, 0],
                                     np.nextafter(p[:, 1], p[:, 1] + dy) if dy else p[:, 1]), axis=1))
    t = rs.uniform(0, 1, size=(len(v), 64))
    on = v[:, None, :] + t[..., None] * (nxt - v)[:, None, :]
    pts.append(on.reshape(-1, 2))
    pts.append(np.array([[0.5, 0.0], [0.5, -1.2246467991473532e-16], [np.nextafter(0.5, 0), 0.0], [np.nextafter(0.5, 1), 0.0],
                         [0.5, np.nextafter(0.0, 1)], [0.5, np.nextafter(0.0, -1)], [0.4, 0.0], [np.nextafter(0.4, 1), 0.0]]))
    pts.append(rs.uniform(-0.55, 0.55, size=(60000, 2)))
    pts.append(np.array([[np.nan, 0.0], [0.0, np.nan], [np.inf, 0.0]]))
    return np.concatenate(pts)


@pytest.mark.parametrize("name", sorted(CURVED_CASES))
def test_vectorised_polygon_predicate_equals_scalar(name):
    from ratinabox_b200.Environment import Environment, _polygon_contains_strict, _polygon_contains_strict_many
    rs = np.random.RandomState(11)
    E = Environment(dict(CURVED_CASES[name]))
    polys = [E.boundary] + list(E.holes)
    pts = np.concatenate([_probe_points(p, rs) for p in polys])
    assert len(pts) >= 60000
    for verts in polys:
        many = _polygon_contains_strict_many(verts, pts)
        one = np.array([_polygon_contains_strict(verts, p) for p in pts])
        assert np.array_equal(many, one)
        assert 0 < many.sum() < len(pts)
    scalar = np.array([E.check_if_position_is_in_environment(p) for p in pts])
    assert np.array_equal(E._in_environment(pts), scalar)


def _scalar_sample_random(E, n):
    """Environment.sample_positions(method="random") as the reference writes it: one point at a time."""
    ex = E.extent
    positions = np.zeros((n, 2))
    positions[:, 0] = np.random.uniform(ex[0], ex[1], size=n)
    positions[:, 1] = np.random.uniform(ex[2], ex[3], size=n)
    for i, pos in enumerate(positions):
        if E.check_if_position_is_in_environment(pos) == False:          # noqa: E712
            positions[i] = _scalar_sample_random(E, 1).reshape(-1)
    return positions


@pytest.mark.parametrize("name", sorted(CURVED_CASES))
def test_sample_positions_curved(golden, name):
    """sample_positions keeps the reference's draw tape: the n initial draws, then each outside point re-drawn on its
    own in index order -- equal to the scalar loop and to the reference's output."""
    import ratinabox_b200 as rb
    g = golden("curved.npz")
    E = rb.Environment(dict(CURVED_CASES[name]))
    assert np.array_equal(E.walls, g[f"{name}_walls"])
    np.random.seed(8)
    got = E.sample_positions(n=500, method="random")
    assert np.array_equal(got, g[f"{name}_samples_random"])
    np.random.seed(8)
    assert np.array_equal(_scalar_sample_random(E, 500), got)
    np.random.seed(3)
    uj = E.sample_positions(n=50, method="uniform_jitter")
    # the hole's area (the grid spacing) sums the shoelace terms in another order than the reference's polygon area:
    # the annulus' points may differ in the last bit
    assert np.abs(uj - g[f"{name}_samples_uj"]).max() <= (0.0 if name == "circle" else 1e-15)
    np.random.seed(21)
    big = E.sample_positions(n=2000, method="random")
    np.random.seed(21)
    assert np.array_equal(_scalar_sample_random(E, 2000), big)
    assert E._in_environment(big).all()

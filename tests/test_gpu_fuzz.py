"""Seeded differential fuzzing of the CUDA path against the oracle: random wall layouts (0..7 inner walls, some
touching the boundary or each other), random Agent parameters, random cell populations; teacher-forced steps
(injected normals, zero jitter) so positions are comparable to 1e-12 step by step, then every cell type's rates at the
reached positions, and geodesic PlaceCells there in a box holding only the first wall.  GPU only."""
import numpy as np
import pytest

import riab_oracle as O

pytestmark = pytest.mark.gpu


def _random_walls(rs):
    k = rs.randint(0, 8)
    walls = []
    for _ in range(k):
        kind = rs.randint(0, 4)
        if kind == 0:                                   # from a boundary wall into the room
            x = rs.uniform(0.1, 0.9)
            walls.append([[x, 0.0], [x + rs.uniform(-0.1, 0.1), rs.uniform(0.2, 0.7)]])
        elif kind == 1:
            y = rs.uniform(0.1, 0.9)
            walls.append([[1.0, y], [rs.uniform(0.3, 0.8), y + rs.uniform(-0.1, 0.1)]])
        elif kind == 2 and walls:                       # T-junction on an earlier wall
            w = np.array(walls[rs.randint(len(walls))])
            p = w[0] + rs.uniform(0.2, 0.8) * (w[1] - w[0])
            q = np.clip(p + rs.uniform(-0.3, 0.3, size=2), 0.05, 0.95)
            walls.append([p.tolist(), q.tolist()])
        else:                                           # free-standing
            p = rs.uniform(0.1, 0.9, size=2)
            q = np.clip(p + rs.uniform(-0.35, 0.35, size=2), 0.05, 0.95)
            walls.append([p.tolist(), q.tolist()])
    return walls


@pytest.mark.parametrize("seed", range(24))
def test_random_environment_motion_and_rates(seed):
    import ratinabox_b200 as rb
    rs = np.random.RandomState(1000 + seed)
    walls = _random_walls(rs)
    prm = {"dt": float(rs.choice([0.005, 0.01, 0.03])), "speed_mean": float(rs.uniform(0.05, 0.4)),
           "speed_std": float(rs.choice([0.0, 0.08])), "thigmotaxis": float(rs.uniform(0, 1)),
           "wall_repel_distance": float(rs.uniform(0.05, 0.2)), "wall_repel_strength": float(rs.choice([0.0, 1.0, 2.0])),
           "rotational_velocity_std": float(rs.uniform(1, 4)), "speed_coherence_time": float(rs.uniform(0.1, 1.0)),
           "rotational_velocity_coherence_time": float(rs.uniform(0.03, 0.3)),
           "head_direction_smoothing_timescale": float(rs.choice([0.004, 0.15]))}
    A, steps = 48, 4
    np.random.seed(seed)
    E = rb.Environment()
    for w in walls:
        E.add_wall(w)
    Ag = rb.Agent(E, dict(prm, n_agents=A))
    env = O.OracleEnvironment(walls=walls)
    pos0 = rs.uniform(0.01, 0.99, size=(A, 2))
    hug = rs.choice(A, A // 2, replace=False)           # half of the agents start within millimetres of a wall
    wl = env.walls[rs.randint(0, len(env.walls), size=len(hug))]
    pos0[hug] = np.clip(wl[:, 0] + rs.uniform(0, 1, size=(len(hug), 1)) * (wl[:, 1] - wl[:, 0])
                        + rs.normal(scale=3e-3, size=(len(hug), 2)), 0.001, 0.999)
    ang = rs.uniform(0, 2 * np.pi, size=A)
    vel0 = (rs.rayleigh(prm["speed_mean"], size=A) * rs.choice([1.0, 4.0], size=A))[:, None] * np.stack((np.cos(ang), np.sin(ang)), 1)
    Ag.pos, Ag.velocity, Ag.measured_velocity = pos0, vel0, vel0
    Ag.head_direction = vel0 / np.linalg.norm(vel0, axis=1, keepdims=True)
    Ag.rotational_velocity = np.zeros(A)
    oas = []
    for a in range(A):
        oa = O.OracleAgent(env, pos0[a], vel0[a], prm)
        oa.head_direction = vel0[a] / np.linalg.norm(vel0[a])
        oas.append(oa)
    use_drift = seed % 3 == 0
    for s in range(steps):
        xi = rs.normal(size=(A, 2))
        drift = rs.normal(scale=0.2, size=(A, 2))
        if use_drift:
            Ag.update(drift_velocity=drift, drift_to_random_strength_ratio=1.5, _xi=xi)
        else:
            Ag.update(_xi=xi)
        for a, oa in enumerate(oas):
            if use_drift:
                oa.update(O.TapeRNG(agent_xi=xi[a]), drift_velocity=drift[a].copy(), drift_to_random_strength_ratio=1.5)
            else:
                oa.update(O.TapeRNG(agent_xi=xi[a]))
        ref = np.array([oa.pos for oa in oas])
        err = np.abs(Ag.pos - ref).max()
        assert err <= 1e-11, (seed, s, err, len(walls))
        assert np.abs(Ag.velocity - np.array([oa.velocity for oa in oas])).max() <= 1e-10
    pos = Ag.pos
    rng = O.TapeRNG()
    n_inner = len(walls)
    if n_inner <= 8:
        geom = "line_of_sight" if n_inner else "euclidean"
        desc = ["gaussian", "gaussian_threshold", "diff_of_gaussians", "top_hat"][seed % 4]
        per_cell = (seed % 2 == 1) and desc != "top_hat"     # top_hat compares with the SCALAR `widths` (Neurons.py:975-976)
        widths = rs.uniform(0.08, 0.3, size=40) if per_cell else 0.18
        P = rb.PlaceCells(Ag, {"n": 40, "description": desc, "widths": widths, "wall_geometry": geom})
        ref = O.place_cells_get_state(env, P.place_cell_centres, P.place_cell_widths, pos, rng, desc, geom,
                                      scalar_width=(None if per_cell else 0.18)).T
        assert np.abs(P.get_state(evaluate_at=None, pos=pos).T - ref).max() <= 1e-5, (seed, desc, geom)
    if walls:
        # geodesic PlaceCells in a box holding only the seed's first wall (from the boundary or free-standing)
        rg = np.random.RandomState(2000 + seed)
        E1 = rb.Environment()
        E1.add_wall(walls[0])
        env1 = O.OracleEnvironment(walls=walls[:1])
        desc = ["gaussian", "gaussian_threshold", "diff_of_gaussians", "top_hat", "one_hot"][rg.randint(5)]
        per_cell = rg.randint(2) == 1 and desc not in ("top_hat", "one_hot")
        w = float(rg.uniform(0.08, 0.3))
        widths = rg.uniform(0.08, 0.3, size=40) if per_cell else w
        P = rb.PlaceCells(rb.Agent(E1, {"n_agents": 1}), {"n": 40, "description": desc, "widths": widths})
        assert P.wall_geometry == "geodesic" and P._effective_geometry() == "geodesic"
        ref = O.place_cells_get_state(env1, P.place_cell_centres, P.place_cell_widths, pos, rng, desc, "geodesic",
                                      scalar_width=(None if per_cell else w)).T
        assert np.abs(P.get_state(evaluate_at=None, pos=pos).T - ref).max() <= 1e-5, (seed, desc, "geodesic", walls[0])
    G = rb.GridCells(Ag, {"n": 20})
    assert np.abs(G.get_state(evaluate_at=None, pos=pos) - O.grid_cells_get_state(G.gridscales, G.phase_offsets, G.w, pos)).max() <= 1e-5
    B = rb.BoundaryVectorCells(Ag, {"n": 12})
    refb = O.bvc_get_state(env, B.tuning_distances, B.tuning_angles, B.sigma_distances, B.sigma_angles, pos, rng)
    assert np.abs(B.get_state(evaluate_at=None, pos=pos) - refb).max() <= 1e-5, seed

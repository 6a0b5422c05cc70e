"""Environments with more than 64 walls on the device: the README's 100-wall circular arena, the successor-features
demo's 200-wall loop track (tests/golden/curved.npz, from the live reference) and 1024-wall mazes.  Motion, BVC rays,
every wall-free population, riab_run and the fused step; the populations that keep the 64-wall limit refuse it before
any launch.  GPU only."""
import numpy as np
import pytest

import riab_oracle as O
from test_gpu_parity import assert_rates_close
from test_oracle_curved import CURVED_CASES, circle

pytestmark = pytest.mark.gpu


def _modeA_agent(rb, g, name, E):
    A = len(g[f"{name}_A_pos0"])
    Ag = rb.Agent(E, {"dt": 0.02, "speed_mean": 0.25, "n_agents": A})
    v0 = g[f"{name}_A_vel0"]
    Ag.pos, Ag.velocity, Ag.measured_velocity = g[f"{name}_A_pos0"], v0, v0
    Ag.rotational_velocity = np.zeros(A)
    Ag.head_direction = v0 / np.linalg.norm(v0, axis=1, keepdims=True)
    Ag.distance_travelled = np.zeros(A)
    return Ag


@pytest.mark.parametrize("name", sorted(CURVED_CASES))
def test_curved_modeA_against_the_reference(golden, name):
    """Teacher-forced steps (half of them bouncing off the short edges, some at the 1.2e-16 m closing edge), Euclidean
    PlaceCells and BVCs at their start positions, against the live reference; then a free run stays strictly inside."""
    import ratinabox_b200 as rb
    g = golden("curved.npz")
    E = rb.Environment(dict(CURVED_CASES[name]))
    assert np.array_equal(E.walls, g[f"{name}_walls"]) and len(E.walls) > 64
    Ag = _modeA_agent(rb, g, name, E)
    PCs = rb.PlaceCells(Ag, {"place_cell_centres": g[f"{name}_centres"], "widths": 0.1, "wall_geometry": "euclidean"})
    td, ta, sd, sa = g[f"{name}_bvc"]
    BVCs = rb.BoundaryVectorCells(Ag, {"tuning_distance": td, "tuning_angle": np.degrees(ta), "sigma_distance": sd,
                                       "sigma_angle": np.degrees(sa)})
    assert_rates_close(PCs.get_state(evaluate_at=None, pos=g[f"{name}_A_pos0"]), g[f"{name}_A_pc"], 1.0, f"{name} pc")
    assert_rates_close(BVCs.get_state(evaluate_at=None, pos=g[f"{name}_A_pos0"]), g[f"{name}_A_bvc"], 1.0, f"{name} bvc")
    assert np.isfinite(BVCs.get_state(evaluate_at="all")).all()
    Ag.update(_xi=g[f"{name}_A_xi"])
    assert np.abs(Ag.pos - g[f"{name}_A_pos"]).max() <= 1e-12
    assert np.abs(Ag.velocity - g[f"{name}_A_vel"]).max() <= 1e-12
    assert np.abs(Ag.measured_velocity - g[f"{name}_A_mv"]).max() <= 1e-10
    PCs.update(); BVCs.update()
    env = O.OracleEnvironment(**CURVED_CASES[name])
    pos = Ag.pos
    assert_rates_close(BVCs.firingrate, O.bvc_get_state(env, td, ta, sd, sa, pos, O.TapeRNG()).T, 1.0, f"{name} bvc update")
    Ag.run(300)
    assert E._in_environment(Ag.pos).all()
    assert np.isfinite(Ag.get_history_arrays()["pos"]).all()


@pytest.mark.parametrize("name", sorted(CURVED_CASES))
def test_curved_collision_taps_equal_the_oracle(golden, name):
    """Parity taps of the motion kernel over 100 / 200 walls: per-iteration collision masks, first-hit wall indices and
    iteration counts equal the float64 oracle's exactly."""
    import ratinabox_b200 as rb
    g = golden("curved.npz")
    E = rb.Environment(dict(CURVED_CASES[name]))
    Ag = _modeA_agent(rb, g, name, E)
    Ag.update(_xi=g[f"{name}_A_xi"], _record_collisions=True)
    info = Ag.last_collision_info()
    env = O.OracleEnvironment(**CURVED_CASES[name])
    W = len(env.walls)
    n_hits = 0
    for a in range(len(g[f"{name}_A_pos0"])):
        oa = O.OracleAgent(env, g[f"{name}_A_pos0"][a], g[f"{name}_A_vel0"][a], {"dt": 0.02, "speed_mean": 0.25})
        rec = oa.update(O.TapeRNG(agent_xi=g[f"{name}_A_xi"][a]))
        n = len(rec["collisions"])
        assert info["n_iters"][a] == n, a
        fh = np.full(info["first_hit"].shape[1], -1)
        fh[:len(rec["first_hit"])] = rec["first_hit"]
        assert np.array_equal(info["first_hit"][a], fh), a
        m = np.zeros(info["mask"].shape[1:], dtype=bool)
        m[:n] = np.array(rec["collisions"]).reshape(n, W)
        assert np.array_equal(info["mask"][a].astype(bool), m), a
        n_hits += len(rec["first_hit"])
    assert n_hits >= 40


def _run_state(Ag):
    out = {k: np.asarray(getattr(Ag, k)).copy() for k in ("pos", "velocity", "head_direction", "distance_travelled",
                                                             "distance_to_closest_wall")}
    for k, v in Ag.get_history_arrays().items():
        out["agent." + k] = np.asarray(v)
    for i, N in enumerate(Ag.Neurons):
        out[f"{i}.firingrate"] = np.asarray(N.firingrate).copy()
        for k, v in N.get_history_arrays().items():
            out[f"{i}.{k}"] = np.asarray(v)
    return out


def _assert_same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), f"{what}: {k}"


def _circle_pops(rb, params, fused=False, seed=3, A=2048):
    np.random.seed(seed)
    E = rb.Environment(dict(params))
    Ag = rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": seed, "fused_step": fused})
    rb.PlaceCells(Ag, {"n": 64, "widths": 0.1, "wall_geometry": "euclidean", "save_spikes": True})
    rb.GridCells(Ag, {"n": 32})
    rb.BoundaryVectorCells(Ag, {"n": 16})
    rb.HeadDirectionCells(Ag, {"n": 8})
    return Ag


@pytest.mark.parametrize("name", sorted(CURVED_CASES))
def test_run_equals_stepped_and_fused_equals_unfused(name):
    """Euclidean PlaceCells + GridCells + BVCs + HeadDirectionCells on one Agent: Agent.run(n), the stepped loop and
    fused_step=True give the same state, rates, spikes and history rows, bit for bit."""
    import ratinabox_b200 as rb
    res = {}
    for way in ("step", "run", "step_fused", "run_fused"):
        Ag = _circle_pops(rb, CURVED_CASES[name], fused=way.endswith("fused"))
        if way.startswith("run"):
            Ag.run(12)
        else:
            for _ in range(12):
                Ag.update()
                for N in Ag.Neurons:
                    N.update()
        res[way] = _run_state(Ag)
    for way in ("run", "step_fused", "run_fused"):
        _assert_same(res[way], res["step"], f"{name} {way}")
    assert any(v.any() for k, v in res["step"].items() if k.endswith("spikes"))


def test_readme_circular_arena():
    """The README's quick tour: 65 536 agents and default BVCs in the 100-wall arena, Ag.run(1000)."""
    import ratinabox_b200 as rb
    Env = rb.Environment({"boundary": [[0.5 * np.cos(t), 0.5 * np.sin(t)] for t in np.linspace(0, 2 * np.pi, 100)]})
    Ag = rb.Agent(Env, {"n_agents": 65536})
    BVCs = rb.BoundaryVectorCells(Ag)
    Ag.run(1000)
    assert Env._in_environment(Ag.pos).all()
    fr = BVCs.firingrate
    assert fr.shape == (65536, BVCs.n) and np.isfinite(fr).all() and fr.max() > 0.1


def test_successor_features_in_the_loop_track():
    """The demo's loop: Euclidean PlaceCells on its centres, SuccessorFeatures and the tangential drift, stepped with
    update_weights -- the trace and the learning step against the float64 TD oracle on the device's own state."""
    import riab_oracle_td as T
    import ratinabox_b200 as rb
    from ratinabox_b200.contribs import SuccessorFeatures
    EPS32 = np.finfo(np.float32).eps
    np.random.seed(0)
    E = rb.Environment(dict(CURVED_CASES["annulus"]))
    A, dt = 256, 0.1
    Ag = rb.Agent(E, {"dt": dt, "n_agents": A, "seed": 4})
    centres = np.array([[0.45 * np.cos(t), 0.45 * np.sin(t)] for t in np.linspace(0, 2 * np.pi, 100)])
    feat = rb.PlaceCells(Ag, {"n": 100, "widths": 0.1, "place_cell_centres": centres, "wall_geometry": "euclidean",
                              "name": "PlaceCells"})
    sf = SuccessorFeatures(Ag, {"features": feat, "input_layers": [feat], "tau": 10, "tau_e": 0.5, "eta": 0.02})
    sf.inputs["PlaceCells"]["w"] *= 0.1
    dev = lambda x, n: x[:, :n].double().cpu().numpy()                                  # noqa: E731
    prev = None
    for t in range(30):
        Ag.update(drift_velocity=0.5 * np.stack((-Ag.pos[:, 1], Ag.pos[:, 0]), axis=1), drift_to_random_strength_ratio=2)
        feat.update(); sf.update()
        n = sf.n
        s = {"fr": dev(sf._fr_prev, n), "deriv": dev(sf._deriv, n), "prime": dev(sf._prime, n),
             "e": dev(sf._trace["PlaceCells"], 100), "W": sf._master["PlaceCells"].cpu().numpy().copy()}
        I = dev(feat._hist[feat._last_slot], 100)
        if prev is not None:
            want = T.td_trace(prev["e"], I, dt, sf.tau_e)
            assert np.all(np.abs(s["e"] - want) <= 3 * EPS32 * (np.abs(dt * I) + np.abs(prev["e"]))), t
        r = I
        sf.update_weights()
        after = {"td": dev(sf._td, n), "W": sf._master["PlaceCells"].cpu().numpy().copy()}
        W = s["W"].copy()
        td = T.td_learn([W], [s["e"]], r, s["fr"], s["deriv"], s["prime"], dt, sf.tau, sf.eta, sf.L2)
        assert np.all(np.abs(after["td"] - td) <= 4 * EPS32 * (np.abs(r) + np.abs(s["deriv"]) + np.abs(s["fr"]))), t
        b, = T.td_learn_bound([s["e"]], r, s["fr"], s["deriv"], s["prime"], sf.tau)
        err = np.abs((after["W"] - s["W"]) - (W - s["W"]))
        assert np.all(err <= sf.eta * dt * 1e-5 * b + 1e-15 * np.abs(s["W"])), t
        prev = {"e": dev(sf._trace["PlaceCells"], 100)}
    assert E._in_environment(Ag.pos).all()


def test_forced_and_imported_motion_in_the_loop_track():
    """Forced positions and an imported trajectory need no walls: in the 200-wall loop they run through update(), run()
    and the populations like in the box, run() equal to the stepped loop bit for bit."""
    import ratinabox_b200 as rb
    E = rb.Environment(dict(CURVED_CASES["annulus"]))
    A = 64
    Ag = rb.Agent(E, {"dt": 0.05, "n_agents": A})
    PCs = rb.PlaceCells(Ag, {"n": 20, "wall_geometry": "euclidean"})
    rs = np.random.RandomState(1)
    for _ in range(5):
        ang = rs.uniform(0, 2 * np.pi, A)
        p = 0.45 * np.stack((np.cos(ang), np.sin(ang)), axis=1)
        Ag.update(forced_next_position=p.copy())
        PCs.update()
        assert np.array_equal(Ag.pos, p)
        env = O.OracleEnvironment(**CURVED_CASES["annulus"])
        ref = O.place_cells_get_state(env, PCs.place_cell_centres, PCs.place_cell_widths, p, O.TapeRNG(), "gaussian",
                                      "euclidean").T
        assert np.abs(PCs.firingrate - ref).max() <= 1e-5
    times = np.arange(0, 20.0, 0.1)
    traj = 0.45 * np.stack((np.cos(times), np.sin(times)), axis=1)
    res = []
    for way in ("step", "run"):
        np.random.seed(5)
        Ag = rb.Agent(E, {"dt": 0.05, "n_agents": A, "seed": 6})
        rb.PlaceCells(Ag, {"n": 20, "wall_geometry": "euclidean", "place_cell_centres": PCs.place_cell_centres})
        Ag.import_trajectory(times=times, positions=traj)
        if way == "run":
            Ag.run(40)
        else:
            for _ in range(40):
                Ag.update()
                Ag.Neurons[0].update()
        res.append(_run_state(Ag))
    _assert_same(res[1], res[0], "imported run vs step")
    assert np.abs(np.linalg.norm(res[0]["pos"], axis=1) - 0.45).max() < 1e-3


def _replay_draws_inside(S, seed, agent, step, env):
    """The ReplayAgent's draws of one (agent, update) with the start position of a polygonal environment: the first of
    the uniform draws 2, 3, ... inside it (k_subagent's sample_positions(n=1))."""
    d = S._replay_draws(seed, agent, step, 1.0, 0.1, env.extent)
    ext, a = env.extent, np.array([agent], dtype=np.uint64)
    for k in range(1024):
        ux, uy = S._uniforms(seed, a, 2 + k, step, 7)
        d[3], d[4] = ext[0] + (ext[1] - ext[0]) * ux[0], ext[2] + (ext[3] - ext[2]) * uy[0]
        if env.contains(d[3:5]):
            break
    return d


def test_subagents_in_curved_environments(monkeypatch):
    """DumbAgent and ReplayAgent over a lead Agent in the 200-wall loop against their oracles on the device's Philox
    draws (as tests/test_gpu_subagents.py does in the box); ThetaSequenceAgent's forward rollouts likewise in the
    100-wall circle.  In the 10 cm wide loop a fast replay rollout can leave the environment, where the reference re-draws
    at random and the oracle stops: such an agent is compared up to there."""
    import ratinabox_b200 as rb
    from ratinabox_b200.contribs import DumbAgent, ReplayAgent
    from riab_oracle_subagents import OracleDumb, OracleReplay
    import test_gpu_subagents as S
    import test_gpu_theta_sequence as TS
    A, T = 1024, 200
    sample = np.array([0, 3, 100, 200, 311, 400, 513, 640, 777, 900, 1000, 1023])
    np.random.seed(5)
    Lead = rb.Agent(rb.Environment(dict(CURVED_CASES["annulus"])), {"dt": 0.01, "n_agents": A, "seed": 2,
                                                                     "speed_mean": 0.3, "speed_std": 0.3})
    D = DumbAgent(Lead, {"seed": 21, "drift_distance": 0.2})
    R = ReplayAgent(Lead, {"seed": 22, "replay_freq": 5.0})
    env = O.OracleEnvironment(**CURVED_CASES["annulus"])
    sham = R._sham
    od = [OracleDumb(env, {"drift_distance": 0.2}) for _ in sample]
    orr = [OracleReplay(env, {"replay_freq": 5.0}, 0.01, (sham["measured_velocity"][a].cpu().numpy(),
                                                         sham["head_direction"][a].cpu().numpy(), 0.0)) for a in sample]
    idx = np.zeros(len(sample), dtype=int)
    left = np.zeros(len(sample), dtype=bool)
    worst_d = worst_r = 0.0
    n_rep = n_cmp = 0
    for s in range(T):
        Lead.update()
        lp, lt = Lead.pos[sample], Lead.t
        D.update(); R.update()
        dp, rp, flags = D.pos[sample], R.pos[sample], R.is_undergoing_replay[sample]
        for j, a in enumerate(sample):
            ag = np.array([a], dtype=np.uint64)
            if left[j]:
                continue
            try:
                want = od[j].step(lp[j], 0.01, S._normals(21, ag, 0, s, 6)[0])
            except RuntimeError:
                left[j] = True
                continue
            worst_d = max(worst_d, float(np.abs(want - dp[j]).max()))
            was = orr[j].is_undergoing_replay
            draws = _replay_draws_inside(S, 22, a, s, env)
            xi = S._normals(22, np.full(4096, a, dtype=np.uint64), idx[j], np.arange(4096), 8) if not was else None
            try:
                want = orr[j].step(lp[j], lt, draws, xi)
            except RuntimeError:
                left[j] = True
                continue
            n_cmp += 1
            if not was and orr[j].is_undergoing_replay:
                idx[j] += 1
                n_rep += 1
            assert orr[j].is_undergoing_replay == flags[j], (s, a)
            if np.isfinite(want).all():
                worst_r = max(worst_r, float(np.abs(want - rp[j]).max()))
    assert n_rep > 5 and n_cmp >= 300, (n_rep, n_cmp)
    assert worst_d <= 1e-5 and worst_r <= 1e-5, (worst_d, worst_r)
    monkeypatch.setattr(TS, "HOLED", dict(CURVED_CASES["circle"]))
    worst, nan_diff, finite, _ = TS._philox_run("holed", 256, 300, np.array([0, 5, 77, 200, 255]),
                                                O.OracleEnvironment(**CURVED_CASES["circle"]),
                                                {"speed_mean": 0.2, "speed_std": 0.2})
    assert finite > 0.3 * 300 * 5
    assert nan_diff <= 2 and worst <= 1e-5, (nan_diff, worst)


def _maze(n_walls, seed=0):
    """The unit box and n_walls - 4 short random walls."""
    rs = np.random.RandomState(seed)
    c = rs.uniform(0.05, 0.95, size=(n_walls - 4, 2))
    ang = rs.uniform(0, np.pi, size=n_walls - 4)
    h = 0.01 * np.stack((np.cos(ang), np.sin(ang)), axis=1)
    return np.stack((c - h, c + h), axis=1)


def test_1024_walls_65536_agents():
    """The largest environment the motion kernel takes: 1024 walls, 65 536 agents, one teacher-forced step; a fixed
    sample of agents against the float64 oracle."""
    import ratinabox_b200 as rb
    walls = _maze(1024)
    E = rb.Environment()
    for w in walls:
        E.add_wall(w)
    assert len(E.walls) == 1024
    A = 65536
    np.random.seed(1)
    Ag = rb.Agent(E, {"dt": 0.05, "n_agents": A, "speed_mean": 0.3})
    pos0, vel0 = Ag.pos.copy(), Ag.velocity.copy()
    xi = np.random.RandomState(2).normal(size=(A, 2))
    Ag.update(_xi=xi)
    env = O.OracleEnvironment(walls=walls)
    pos = Ag.pos
    for a in np.random.RandomState(3).choice(A, 128, replace=False):
        oa = O.OracleAgent(env, pos0[a], vel0[a], {"dt": 0.05, "speed_mean": 0.3})
        oa.update(O.TapeRNG(agent_xi=xi[a]))
        assert np.abs(oa.pos - pos[a]).max() <= 1e-12, a
    BVCs = rb.BoundaryVectorCells(Ag, {"n": 8})
    BVCs.update()
    td, ta, sd, sa = BVCs.tuning_distances, BVCs.tuning_angles, BVCs.sigma_distances, BVCs.sigma_angles
    smp = np.arange(0, A, 4096)
    assert_rates_close(BVCs.firingrate[smp], O.bvc_get_state(env, td, ta, sd, sa, pos[smp], O.TapeRNG()).T, 1.0, "maze bvc")
    Ag.run(20)
    assert np.isfinite(Ag.pos).all()


def test_refusals():
    """1025 walls: refused before any launch.  In the circle, the populations whose kernels read at most 64 walls refuse;
    their Euclidean / non-occluding variants run."""
    import ratinabox_b200 as rb
    from ratinabox_b200 import _lib
    from ratinabox_b200.contribs import PhasePrecessingPlaceCells, SpatialGoalEnvironment
    lib = _lib.load()
    E = rb.Environment()
    for w in _maze(1025):
        E.add_wall(w)
    c0 = lib.riab_launch_count()
    with pytest.raises(_lib.RiabError, match="1025"):
        Ag = rb.Agent(E, {"n_agents": 16})
        Ag.update()
        Ag.pos
    assert lib.riab_launch_count() == c0

    refused = (_lib.RiabError, NotImplementedError)
    Env = rb.Environment(dict(CURVED_CASES["circle"]))
    Env.add_object([0.1, 0.1])
    Ag = rb.Agent(Env, {"n_agents": 32})
    Other = rb.Agent(Env, {"n_agents": 32})
    makers = {
        "place_los": lambda: rb.PlaceCells(Ag, {"n": 10, "wall_geometry": "line_of_sight"}),
        "ovc": lambda: rb.ObjectVectorCells(Ag, {"walls_occlude": True}),
        "avc": lambda: rb.AgentVectorCells(Ag, Other, {"walls_occlude": True}),
        "pppc": lambda: PhasePrecessingPlaceCells(Ag, {"n": 10, "wall_geometry": "line_of_sight"}),
        "rsn": lambda: rb.RandomSpatialNeurons(Ag, {"n": 4, "wall_geometry": "line_of_sight"}),
    }
    for k, make in makers.items():
        with pytest.raises(refused):
            P = make()
            Ag.update()
            P.update()
            np.asarray(P.firingrate)
    with pytest.raises(refused):
        G = SpatialGoalEnvironment(params=dict(CURVED_CASES["circle"]), n_agents=4)
        G.reset()
        G.step()
    Ag = rb.Agent(Env, {"n_agents": 32})
    Other = rb.Agent(Env, {"n_agents": 32})
    ok = [rb.PlaceCells(Ag, {"n": 10, "wall_geometry": "euclidean"}),
          rb.PlaceCells(Ag, {"n": 10, "wall_geometry": "euclidean", "description": "one_hot"}),
          rb.ObjectVectorCells(Ag, {"walls_occlude": False}),
          rb.AgentVectorCells(Ag, Other, {"walls_occlude": False}),
          PhasePrecessingPlaceCells(Ag, {"n": 10, "wall_geometry": "euclidean"}),
          rb.RandomSpatialNeurons(Ag, {"n": 4, "wall_geometry": "euclidean"}),
          rb.GridCells(Ag, {"n": 8}), rb.VelocityCells(Ag), rb.SpeedCell(Ag), rb.FieldOfViewBVCs(Ag)]
    for _ in range(3):
        Ag.update(); Other.update()
        for P in ok:
            P.update()
    for P in ok:
        assert np.isfinite(np.asarray(P.firingrate)).all(), type(P).__name__
    Ag.run(5)


@pytest.mark.parametrize("n_walls", [64, 65])
def test_64_and_65_walls(n_walls):
    """On both sides of the step kernels' wall block: motion against the oracle, run() equal to the stepped loop and
    fused_step=True equal to False; occluding ObjectVectorCells run at 64 walls and refuse at 65."""
    import ratinabox_b200 as rb
    from ratinabox_b200 import _lib
    walls = _maze(n_walls, seed=4)
    res = {}
    for way in ("step", "run", "step_fused"):
        E = rb.Environment()
        for w in walls:
            E.add_wall(w)
        np.random.seed(6)
        Ag = rb.Agent(E, {"dt": 0.02, "n_agents": 1000, "seed": 8, "fused_step": way.endswith("fused")})
        rb.PlaceCells(Ag, {"n": 40, "wall_geometry": "euclidean", "save_spikes": True})
        rb.BoundaryVectorCells(Ag, {"n": 8})
        if way == "run":
            Ag.run(6)
        else:
            for _ in range(6):
                Ag.update()
                for N in Ag.Neurons:
                    N.update()
        res[way] = _run_state(Ag)
    for way in ("run", "step_fused"):
        _assert_same(res[way], res["step"], f"{n_walls} walls {way}")
    E = rb.Environment()
    for w in walls:
        E.add_wall(w)
    E.add_object([0.5, 0.5])
    Ag = rb.Agent(E, {"n_agents": 64})
    xi = np.random.RandomState(0).normal(size=(64, 2))
    pos0, vel0 = Ag.pos.copy(), Ag.velocity.copy()
    Ag.update(_xi=xi)
    env = O.OracleEnvironment(walls=walls)
    for a in range(64):
        oa = O.OracleAgent(env, pos0[a], vel0[a], {"dt": Ag.dt})
        oa.update(O.TapeRNG(agent_xi=xi[a]))
        assert np.abs(oa.pos - Ag.pos[a]).max() <= 1e-12
    OVC = rb.ObjectVectorCells(Ag, {"walls_occlude": True})
    if n_walls <= 64:
        OVC.update()
        assert np.isfinite(OVC.firingrate).all()
    else:
        with pytest.raises(_lib.RiabError, match="at most 64 walls"):
            OVC.update()
            np.asarray(OVC.firingrate)

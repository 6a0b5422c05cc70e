"""AgentVectorCells and FieldOfViewAVCs on the GPU (csrc/riab_avc.cuh, k_step<AvcPolicy>): rates against the float64
oracle (oracle/riab_oracle_avc.py) at the agents and away from them for every cell tile and batch size with pairwise,
broadcast and self partners; the line-of-sight decisions of the live reference's placed partners (tests/golden/avc.npz);
bit equality of the stepped API, the fused stepped API and Agent.run with pinned launch counts; a two-Agent stepped loop
in every fused_step combination with edits of the partner's positions; spikes against the Philox mirror; NaN own and
partner positions, no partner and retargeting; a FeedForwardLayer fed by AVCs; head-direction averages; the raises; and
the staged live reference."""
import warnings

import numpy as np
import pytest

import philox_np as PX
import riab_oracle as O
import riab_oracle_avc as V

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                      # noqa: E402

WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
STATE = ("pos", "velocity", "rotational_velocity", "measured_velocity", "measured_rotational_velocity",
         "head_direction", "distance_travelled", "distance_to_closest_wall")
WAYS = ("run", "run_fused", "step", "step_fused")


def _env():
    E = rb.Environment()
    for w in WALLS:
        E.add_wall(w)
    return E


def _bound(N):
    return 1e-5 * abs(N.max_fr - N.min_fr)


def _close(got, want, bound):
    assert got.shape == want.shape, (got.shape, want.shape)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    err = np.abs(np.nan_to_num(got) - np.nan_to_num(want))
    assert np.all(err <= bound), float(np.max(err - bound))


def _rows(Ag, name):
    return np.asarray(getattr(Ag, name), dtype=float).reshape(Ag.n_agents, 2)


def _tuning(N):
    return (N.tuning_distances, N.tuning_angles, N.sigma_distances, N.sigma_angles)


def _oracle(N, partner, pos, hd=None):
    return V.avc_get_state(O.OracleEnvironment(walls=WALLS), partner, _tuning(N), pos, O.TapeRNG(), N.wall_geometry,
                           head_direction=hd, min_fr=N.min_fr, max_fr=N.max_fr)


def _set_tuning(N, t):
    N.tuning_distances, N.tuning_angles, N.sigma_distances, N.sigma_angles = (np.array(x, dtype=float) for x in t)


# ---- rates against the oracle
@pytest.mark.parametrize("A", [1, 33, 4099])
@pytest.mark.parametrize("n", [1, 4, 10, 58, 63, 64, 300])
def test_rates_match_the_oracle(n, A):
    np.random.seed(n + A)
    E = _env()
    Ag = rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": 3})
    Ag2 = rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": 4, "speed_mean": 0.15})
    Ag3 = rb.Agent(E, {"dt": 0.02, "seed": 5})
    P = rb.AgentVectorCells(Ag, Ag2, {"n": n, "min_fr": 0.1, "max_fr": 1.3})                      # pairwise, occluded
    Q = rb.AgentVectorCells(Ag, Ag3, {"n": n, "walls_occlude": False, "reference_frame": "egocentric"})   # broadcast
    S = rb.AgentVectorCells(Ag, Ag, {"n": n, "max_fr": 2.0})                                       # self
    for _ in range(3):
        Ag.update()
        Ag2.update()
        Ag3.update()
        for N in (P, Q, S):
            N.update()
    pos, hd, pos2, pos3 = _rows(Ag, "pos"), _rows(Ag, "head_direction"), _rows(Ag2, "pos"), _rows(Ag3, "pos")[0]
    for N, partner, h in ((P, pos2, None), (Q, pos3, hd), (S, pos, None)):
        fr = N.get_history_arrays()["firingrate"][-1].reshape(A, N.n)
        _close(fr, _oracle(N, partner, pos, h).T, _bound(N))
        assert np.array_equal(N.get_state().T, fr)                      # get_state() at the agents gives the update rows
    # away from the agents: a batched partner takes other_pos, a single one is read from the Agent
    rs = np.random.RandomState(n)
    X, Y = rs.uniform(0.02, 0.98, (50, 2)), rs.uniform(0.02, 0.98, (50, 2))
    H = rs.normal(size=(50, 2))
    _close(P.get_state(evaluate_at=None, pos=X, other_pos=Y), _oracle(P, Y, X), _bound(P))
    _close(P.get_state(evaluate_at=None, pos=X, other_pos=Y[0]), _oracle(P, Y[0], X), _bound(P))
    _close(Q.get_state(evaluate_at=None, pos=X, head_direction=H), _oracle(Q, pos3, X, H), _bound(Q))
    got = Q.get_state(evaluate_at="all", head_direction=H[0], return_tensor=True).double().cpu().numpy().T
    _close(got, _oracle(Q, pos3, E.flattened_discrete_coords, H[0]), _bound(Q))


# ---- the live reference's placed partners (mode A)
def _fixture_population(g, k, Ag, other):
    cls = rb.FieldOfViewAVCs if k == "fov" else rb.AgentVectorCells
    prm = {"fov": {}, "allo": {"n": 12}, "eucl": {"n": 6, "walls_occlude": False, "min_fr": 0.2, "max_fr": 1.5}}[k]
    N = cls(Ag, other, prm)
    _set_tuning(N, g[f"{k}1_tuning"])
    return N


def test_the_reference_fixture_and_its_line_of_sight_decisions(golden):
    g = golden("avc.npz")
    E = _env()
    Ag, Ag2 = rb.Agent(E, {"dt": 0.02}), rb.Agent(E, {"dt": 0.02})
    pos, partner = g["A_pos"], g["A_partner"]
    for k in ("allo", "eucl", "fov"):
        N = _fixture_population(g, k, Ag, Ag2)
        kw = {"head_direction": g["A_hd"]} if k == "fov" else {}
        _close(N.get_state(evaluate_at=None, pos=pos, other_pos=partner, **kw), g[f"A_{k}"], _bound(N))
    N = _fixture_population(g, "allo", Ag, Ag2)
    Ag2.pos = g["B_partner"]
    _close(N.get_state(evaluate_at=None, pos=pos), g["B_allo"], _bound(N))
    F = _fixture_population(g, "fov", Ag, Ag2)
    with pytest.warns(UserWarning) as rec:
        got = F.get_state(evaluate_at=None, pos=pos[:16])
    assert [str(w.message) for w in rec] == list(g["B_fov_warnings"])
    _close(got, g["B_fov_default_hd"], _bound(F))
    # the decisions themselves: a cell tuned to d = 1000 with a flat angular tuning fires ~1 exactly when blocked
    probe = rb.AgentVectorCells(Ag, Ag2, {"n": 1})
    _set_tuning(probe, ([1000.0], [0.0], [1.0], [1e3]))
    blocked = probe.get_state(evaluate_at=None, pos=pos, other_pos=partner)[0] > 0.5
    d = O.distances_accounting_for_environment(O.OracleEnvironment(walls=WALLS), pos, partner, "line_of_sight",
                                               O.TapeRNG()).diagonal()
    assert np.array_equal(blocked, d == 1000)
    assert blocked[g["A_kind"] == 4].any() and not blocked[g["A_kind"] == 3].any()


def test_self_nan_none_and_retargeting(golden):
    g = golden("avc.npz")
    E = _env()
    Ag, Ag2, Ag3 = rb.Agent(E, {"dt": 0.02}), rb.Agent(E, {"dt": 0.02}), rb.Agent(E, {"dt": 0.02})
    # the Agent as its own partner
    Ag.pos, Ag.head_direction = g["self_pos"], g["self_hd"]
    S = rb.AgentVectorCells(Ag, Ag, {"n": 9, "min_fr": 0.1})
    _set_tuning(S, g["self_tuning"])
    F = rb.FieldOfViewAVCs(Ag, Ag, {"spatial_resolution": 0.05})
    _set_tuning(F, g["self_fov_tuning"])
    _close(S.get_state(), g["self_rates"], _bound(S))
    _close(F.get_state(), g["self_fov_rates"], _bound(F))
    # a NaN partner: NaN rates, NaN rows and no spikes
    N = _fixture_population(g, "allo", Ag, Ag2)
    Ag2.pos = np.array([np.nan, np.nan])
    assert np.all(np.isnan(N.get_state())) and np.all(np.isnan(_fixture_population(g, "fov", Ag, Ag2).get_state()))
    N.update()
    assert np.all(np.isnan(N.firingrate)) and not N.get_history_arrays()["spikes"][-1].any()
    assert np.all(np.isnan(g["nan_update_fr"])) and not g["nan_update_spikes"].any()
    # no partner: exact zeros, at the agents, away from them and through update()
    N.tuning_type_agent = None
    N.update()
    assert np.array_equal(N.firingrate, np.zeros(12)) and np.array_equal(N.get_state(), np.zeros((12, 1)))
    assert np.array_equal(N.get_state(evaluate_at=None, pos=g["A_pos"][:5]), np.zeros((12, 5)))
    # retargeted to another Agent
    Ag3.pos = np.array([0.2, 0.8])
    N.tuning_type_agent = Ag3
    N.update()
    _close(N.firingrate[:, None], _oracle(N, _rows(Ag3, "pos")[0], _rows(Ag, "pos")), _bound(N))
    # NaN own position: zeros (Neurons.update's guard)
    Ag.pos = np.array([np.nan, np.nan])
    N.update()
    assert np.array_equal(N.firingrate, np.zeros(12))
    # get_head_direction_averaged_state of a FieldOfViewAVCs population
    F2 = _fixture_population(g, "fov", Ag, Ag2)
    Ag2.pos = g["avg_partner"]
    _close(F2.get_head_direction_averaged_state(evaluate_at=None, pos=g["avg_P"], angular_resolution_degrees=30),
           g["avg_fov"], 2e-5)


def test_raises():
    E = _env()
    Ag = rb.Agent(E, {"n_agents": 5})
    with pytest.raises(ValueError, match="pair row"):
        rb.AgentVectorCells(Ag, rb.Agent(E, {"n_agents": 3}))
    with pytest.raises(ValueError, match="id_offset"):
        rb.AgentVectorCells(Ag, rb.Agent(E, {"n_agents": 5, "id_offset": 5}))
    with pytest.raises(AttributeError):
        rb.AgentVectorCells(Ag, None)
    P = rb.Environment({"boundary_conditions": "periodic"})
    with pytest.raises(NotImplementedError):
        rb.AgentVectorCells(rb.Agent(P), rb.Agent(P))
    N = rb.AgentVectorCells(Ag, rb.Agent(E, {"n_agents": 5}))
    with pytest.raises(ValueError, match="other_pos"):
        N.get_state(evaluate_at=None, pos=np.zeros((4, 2)) + 0.5)
    with pytest.raises(ValueError, match="partner positions"):
        N.get_state(evaluate_at=None, pos=np.zeros((4, 2)) + 0.5, other_pos=np.zeros((3, 2)) + 0.5)
    N.tuning_type_agent = rb.Agent(E, {"n_agents": 2})
    with pytest.raises(ValueError, match="pair row"):
        N.update()
    with pytest.warns(UserWarning, match=r"Ignoring 'n' parameter value \(7\) that was passed, and setting number of "
                                         r"AgentVectorCell neurons to 58"):
        assert rb.FieldOfViewAVCs(Ag, Ag, {"n": 7}).n == 58


# ---- stepped / fused / run
def _agents(fused, A=257):
    np.random.seed(9)
    E = _env()
    Ag = rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": 5, "fused_step": fused})
    Ag2 = rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": 6})
    Ag2.update()
    return Ag, Ag2


def avc_first(fused):
    Ag, Ag2 = _agents(fused)
    rb.AgentVectorCells(Ag, Ag2, {"n": 12, "max_fr": 3.0})
    rb.FieldOfViewAVCs(Ag, Ag2, {"spatial_resolution": 0.05})
    return Ag, Ag2


def behind_place(fused):
    Ag, Ag2 = _agents(fused)
    rb.PlaceCells(Ag, {"n": 64, "wall_geometry": "line_of_sight"})
    rb.AgentVectorCells(Ag, Ag2, {"n": 70, "noise_std": 0.05, "walls_occlude": False})
    return Ag, Ag2


def imported(fused):
    Ag, Ag2 = _agents(fused)
    rng = np.random.default_rng(8)
    Ag.import_trajectory(times=np.cumsum(rng.uniform(0.05, 0.2, 20)), positions=rng.uniform(0.05, 0.95, (20, 2)))
    rb.AgentVectorCells(Ag, Ag2, {"n": 10, "max_fr": 3.0})
    rb.AgentVectorCells(Ag, Ag, {"n": 10, "max_fr": 3.0})
    return Ag, Ag2


SETUPS = {
    # skewed: motion(0), then per step population 1 and the skewed launch of population 0
    "avc_first": (avc_first, lambda n: {"run": 1 + 2 * n, "run_fused": 1 + 2 * n, "step": 3 * n, "step_fused": 2 * n}),
    "behind_place": (behind_place, lambda n: {"run": 1 + 2 * n, "run_fused": 1 + 2 * n, "step": 3 * n, "step_fused": 2 * n}),
    # a motion source: the motion kernel, then every population
    "imported": (imported, lambda n: dict.fromkeys(WAYS, 3 * n)),
}


def _collect(Ag):
    out = {k: np.asarray(getattr(Ag, k)).copy() for k in STATE}
    for k, v in Ag.get_history_arrays().items():
        out["agent." + k] = np.asarray(v)
    for i, N in enumerate(Ag.Neurons):
        for k, v in N.get_history_arrays().items():
            out[f"{i}.{k}"] = np.asarray(v)
    return out


@pytest.mark.parametrize("name", list(SETUPS))
def test_run_fused_and_stepped_are_bit_identical(name):
    from ratinabox_b200 import _lib
    lib = _lib.load()
    build, launches = SETUPS[name]
    n = 5
    res, counts = {}, {}
    for way in WAYS:
        Ag, Ag2 = build(way.endswith("fused"))
        Ag.update()
        for N in Ag.Neurons:
            N.update()
        c0 = lib.riab_launch_count()
        if way.startswith("run"):
            Ag.run(n)
        else:
            for _ in range(n):
                Ag.update()
                for N in Ag.Neurons:
                    N.update()
        res[way] = _collect(Ag)
        counts[way] = lib.riab_launch_count() - c0
        if way == "step":
            # the last step's rows against the oracle and the Philox mirror of the dense spike stream
            pos, hd, pos2 = _rows(Ag, "pos"), _rows(Ag, "head_direction"), _rows(Ag2, "pos")
            for N in Ag.Neurons:
                if not isinstance(N, rb.AgentVectorCells):
                    continue
                h = N.get_history_arrays()
                fr = h["firingrate"][-1].reshape(Ag.n_agents, N.n)
                if N.noise_std == 0:
                    partner = pos if N.tuning_type_agent is Ag else pos2
                    ego = N.reference_frame == "egocentric"
                    _close(fr, _oracle(N, partner, pos, hd if ego else None).T, _bound(N))
                    sp = PX.expected_spikes(5, N._upd - 1, np.arange(Ag.n_agents), fr.astype(np.float32), 0.02,
                                            pop=N._population_id)
                    assert np.array_equal(h["spikes"][-1].reshape(Ag.n_agents, N.n), sp)
    assert counts == launches(n), counts
    ref = res["step"]
    for way in WAYS:
        for k in ref:
            x, y = np.asarray(res[way][k]), np.asarray(ref[k])
            assert x.shape == y.shape and np.array_equal(x, y, equal_nan=True), f"{name}: {way} vs step: {k}"
    assert any(np.asarray(v).any() for k, v in ref.items() if k.endswith(".spikes"))


@pytest.mark.parametrize("fused1", [False, True])
@pytest.mark.parametrize("fused2", [False, True])
def test_two_agent_stepped_loop(fused1, fused2):
    """``Ag1.update(); Ag2.update()`` then AVCs both ways for 200 steps, with in-place edits and assignments of Ag2.pos
    between Ag2's step and the rates that read it: every row against the oracle at the positions of that step."""
    A = 64
    np.random.seed(12)
    E = _env()
    Ag1 = rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": 1, "fused_step": fused1})
    Ag2 = rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": 2, "fused_step": fused2, "speed_mean": 0.2})
    N1 = rb.AgentVectorCells(Ag1, Ag2, {"n": 16, "min_fr": 0.1})
    N2 = rb.FieldOfViewAVCs(Ag2, Ag1, {"spatial_resolution": 0.05})
    rs = np.random.RandomState(0)
    worst = 0.0
    for s in range(200):
        Ag1.update()
        Ag2.update()
        if s % 50 == 25:
            p = Ag2.pos
            p += 0.01                                                    # in place: uploaded before it is read
        elif s % 50 == 40:
            Ag2.pos = rs.uniform(0.05, 0.95, (A, 2))
        N1.update()
        N2.update()
        p1, p2, h2 = _rows(Ag1, "pos"), _rows(Ag2, "pos"), _rows(Ag2, "head_direction")
        for N, own, other, hd in ((N1, p1, p2, None), (N2, p2, p1, h2)):
            fr = N.get_history_arrays()["firingrate"][-1].reshape(A, N.n)
            err = np.abs(fr - _oracle(N, other, own, hd).T)
            assert np.all(err <= _bound(N)), (s, float(err.max()))
            worst = max(worst, float(err.max()))
    assert worst > 0.0 and (N1.get_history_arrays()["firingrate"] > 0.2).any()


def test_feedforward_layer_fed_by_avcs():
    A = 300
    res = []
    for way in ("run", "step"):
        np.random.seed(2)
        E = _env()
        Ag2 = rb.Agent(E, {"dt": 0.05, "n_agents": A, "seed": 7})
        Ag = rb.Agent(E, {"dt": 0.05, "n_agents": A, "seed": 1})
        P = rb.AgentVectorCells(Ag, Ag2, {"n": 16, "name": "AVC"})
        F = rb.FieldOfViewAVCs(Ag, Ag2, {"spatial_resolution": 0.05, "name": "FoV"})
        L = rb.FeedForwardLayer(Ag, {"n": 20, "input_layers": [P, F], "name": "social"})
        if way == "run":
            Ag.run(6)
        else:
            for _ in range(6):
                Ag.update()
                for N in Ag.Neurons:
                    N.update()
        res.append([N.get_history_arrays()["firingrate"] for N in (P, F, L)])
        p, f, out = (N.get_history_arrays()["firingrate"][-1].reshape(A, N.n) for N in (P, F, L))
        want = p @ L.inputs[P.name]["w"].T + f @ L.inputs[F.name]["w"].T + L.biases
        scale = np.abs(p) @ np.abs(L.inputs[P.name]["w"]).T + np.abs(f) @ np.abs(L.inputs[F.name]["w"]).T
        assert np.all(np.abs(out - want) <= 1e-5 * max(scale.max(), 1.0)), float(np.abs(out - want).max())
        X = np.random.RandomState(3).uniform(0.05, 0.95, (40, 2))
        Y = np.random.RandomState(4).uniform(0.05, 0.95, (40, 2))
        got = L.get_state(evaluate_at=None, pos=X, other_pos=Y, head_direction=[0.0, 1.0])
        pw = P.get_state(evaluate_at=None, pos=X, other_pos=Y)
        fw = F.get_state(evaluate_at=None, pos=X, other_pos=Y, head_direction=[0.0, 1.0])
        want = L.inputs[P.name]["w"] @ pw + L.inputs[F.name]["w"] @ fw + L.biases[:, None]
        assert np.all(np.abs(got - want) <= 1e-5 * max(np.abs(want).max(), 1.0))
    for a, b in zip(*res):
        assert np.array_equal(a, b)


def test_matches_the_staged_live_reference():
    import ref_shim
    if ref_shim.import_reference() is None:
        pytest.skip("the reference is not staged under oracle/_ref")
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import AgentVectorCells, FieldOfViewAVCs
    np.random.seed(21)
    RE = Environment()
    for w in WALLS:
        RE.add_wall(w)
    R1, R2 = Agent(RE, {"dt": 0.05}), Agent(RE, {"dt": 0.05, "speed_mean": 0.2})
    RP = AgentVectorCells(R1, R2, {"n": 17, "min_fr": 0.3, "max_fr": 1.1})
    RF = FieldOfViewAVCs(R1, R2)
    E = _env()
    Ag1, Ag2 = rb.Agent(E, {"dt": 0.05}), rb.Agent(E, {"dt": 0.05})
    P = rb.AgentVectorCells(Ag1, Ag2, {"n": 17, "min_fr": 0.3, "max_fr": 1.1})
    F = rb.FieldOfViewAVCs(Ag1, Ag2)
    _set_tuning(P, _tuning(RP))
    _set_tuning(F, _tuning(RF))
    for _ in range(25):
        R1.update()
        R2.update()
        Ag1.pos, Ag1.head_direction, Ag2.pos = R1.pos, R1.head_direction, R2.pos
        _close(P.get_state(), RP.get_state(), _bound(P))
        _close(F.get_state(), RF.get_state(), _bound(F))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            X = np.random.RandomState(1).uniform(0.05, 0.95, (30, 2))
            _close(P.get_state(evaluate_at=None, pos=X), RP.get_state(evaluate_at=None, pos=X), _bound(P))

"""PhasePrecessingPlaceCells on the GPU (csrc/riab_pppc.cuh, k_step<PppcPolicy>): rates at the agents against the float64
oracle (oracle/riab_oracle_pppc.py) for every description and wall geometry, cell tiles and batch sizes, at kappa 1 and 4,
with and without min_fr > 0, through update()'s history row and get_state(); the line-of-sight classification of
PlaceCells; PlaceCells rates and the reference's message away from the agents; bit equality of Agent.run, the fused run,
the stepped and the fused stepped API with pinned launch counts and wrapped rings, as population 0, behind a PlaceCells
population and under an imported trajectory; spikes against the Philox mirror; OU noise statistics; NaN positions;
parameter edits between steps; a FeedForwardLayer reading the cells in run(); and the staged live reference."""
import numpy as np
import pytest

import philox_np as PX
import riab_oracle as O
import riab_oracle_pppc as P

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                                  # noqa: E402
from ratinabox_b200.contribs import PhasePrecessingPlaceCells as PPPC  # noqa: E402

WALLS2 = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
WALLS8 = WALLS2 + [[[0.1, 0.8], [0.4, 0.8]], [[0.5, 0.1], [0.5, 0.35]], [[0.85, 0.2], [0.85, 0.6]],
                   [[0.2, 0.6], [0.45, 0.55]], [[0.6, 0.75], [0.9, 0.9]], [[0.15, 0.3], [0.22, 0.12]]]
WALL1 = [[[0.5, 0.2], [0.5, 0.8]]]
GEOMS = {"euclidean": ([], "euclidean"), "los2": (WALLS2, "line_of_sight"), "los8": (WALLS8, "line_of_sight"),
         "geodesic1": (WALL1, "geodesic")}
DESCS = ("gaussian", "gaussian_threshold", "diff_of_gaussians", "top_hat")
STATE = ("pos", "velocity", "rotational_velocity", "measured_velocity", "measured_rotational_velocity",
         "head_direction", "distance_travelled", "distance_to_closest_wall")
WAYS = ("run", "run_fused", "step", "step_fused")


def _env(walls):
    E = rb.Environment()
    for w in walls:
        E.add_wall(w)
    return E


def _rows(Ag, name):
    return np.asarray(getattr(Ag, name), dtype=float).reshape(Ag.n_agents, 2)


def _bound(N):
    return 1e-5 * max(abs(N.min_fr), abs(N.max_fr)) * P.peak_factor(N.sigma)


def _factors(N, pos, vel, t):
    """theta_modulation_factors of every row (the reference's expression, vectorised over the rows) -> (n, A)."""
    d = vel / (1e-8 + np.linalg.norm(vel, axis=1, keepdims=True))
    phi = N.theta_freq * (t % (1 / N.theta_freq)) * 2 * np.pi
    s = np.array(N.place_cell_widths, dtype=float) * (2 if N.description == "gaussian" else 1)
    v = pos[:, None, :] - np.asarray(N.place_cell_centres, dtype=float)[None, :, :]
    x = np.pi - ((v * d[:, None, :]).sum(-1) / s) * N.precess_fraction * np.pi - phi
    return (P.von_mises(x, 0, N.sigma) * 2 * np.pi).T


def _oracle(N, walls, pos, vel, t):
    geom = N._effective_geometry()
    place = O.place_cells_get_state(O.OracleEnvironment(walls=walls), N.place_cell_centres, N.place_cell_widths, pos,
                                    O.TapeRNG(), N.description, geom, N.min_fr, N.max_fr, scalar_width=N.widths)
    return place * _factors(N, pos, vel, t)


def _close(got, want, bound):
    assert got.shape == want.shape, (got.shape, want.shape)
    err = np.abs(got - want)
    assert np.all(err <= bound), float(err.max() / bound)


# ---- rates against the oracle
CASES = [(1, 1), (33, 4), (4099, 10), (33, 63), (4099, 64), (33, 300), (1, 1024)]


@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("desc", DESCS)
def test_rates_match_the_oracle(geom, desc):
    """Per (A, n): kappa 1 or 4 and min_fr 0 or 0.3 in turn; the update() history row and get_state()."""
    walls, wg = GEOMS[geom]
    for c, (A, n) in enumerate(CASES):
        np.random.seed(100 + c)
        Ag = rb.Agent(_env(walls), {"dt": 0.05, "n_agents": A, "seed": c})
        kappa, min_fr = (1.0, 4.0)[c % 2], (0.0, 0.3)[(c // 2) % 2]
        N = PPPC(Ag, {"n": n, "description": desc, "wall_geometry": wg, "widths": 0.15 + 0.02 * c, "kappa": kappa,
                      "min_fr": min_fr, "max_fr": 2.0, "theta_freq": 8.0, "precess_fraction": 0.7})
        if c % 3 == 1:
            N.place_cell_widths = np.random.uniform(0.1, 0.3, n)          # per-cell widths (top_hat still uses `widths`)
        for _ in range(3):
            Ag.update()
            N.update()
        pos, vel = _rows(Ag, "pos"), _rows(Ag, "velocity")
        want = _oracle(N, walls, pos, vel, Ag.t)
        hist = N.get_history_arrays()["firingrate"][-1].reshape(A, n).T
        _close(hist, want, _bound(N))
        _close(N.get_state(), want, _bound(N))
        f = N.theta_modulation_factors()
        assert f.shape == (n, A) and np.allclose(f, _factors(N, pos, vel, Ag.t), rtol=1e-12, atol=0)


def test_line_of_sight_classification_is_place_cells():
    """With min_fr = 0 a rate is 0 exactly where the PlaceCells rate of the same parameters is (blocked pairs): the
    factor is positive everywhere."""
    np.random.seed(3)
    Ag = rb.Agent(_env(WALLS8), {"dt": 0.05, "n_agents": 2048})
    prm = {"n": 300, "description": "gaussian", "wall_geometry": "line_of_sight", "widths": 0.2}
    N = PPPC(Ag, prm)
    Pc = rb.PlaceCells(Ag, dict(prm, place_cell_centres=N.place_cell_centres))
    Ag.update()
    N.update()
    Pc.update()
    a = N.get_history_arrays()["firingrate"][-1]
    b = Pc.get_history_arrays()["firingrate"][-1]
    assert np.array_equal(a == 0, b == 0) and (b == 0).any() and (b > 0).any()


def test_away_from_the_agents_is_place_cells_and_prints(capsys):
    np.random.seed(4)
    Ag = rb.Agent(_env(WALLS2), {"dt": 0.05, "n_agents": 7})
    prm = {"n": 50, "wall_geometry": "line_of_sight", "min_fr": 0.1, "max_fr": 3.0}
    N = PPPC(Ag, prm)
    Pc = rb.PlaceCells(Ag, dict(prm, description=N.description, place_cell_centres=N.place_cell_centres))
    X = np.random.RandomState(1).uniform(0.05, 0.95, (40, 2))
    capsys.readouterr()
    assert np.array_equal(N.get_state(evaluate_at=None, pos=X), Pc.get_state(evaluate_at=None, pos=X))
    assert capsys.readouterr().out == P.MESSAGE + "\n"
    assert np.array_equal(N.get_state(evaluate_at="all"), Pc.get_state(evaluate_at="all"))
    assert capsys.readouterr().out == P.MESSAGE + "\n"
    N.get_state()
    assert capsys.readouterr().out == ""


# ---- launch paths
def _base(fused, A=257):
    np.random.seed(9)
    return rb.Agent(_env(WALLS2), {"dt": 0.02, "n_agents": A, "seed": 5, "fused_step": fused})


def _limit(A, n, rows=3):
    return rows * A * ((n + 3) // 4 * 4) * 4                # history rings of 3 rows: 5 steps wrap them


def pppc_first(fused):
    Ag = _base(fused)
    PPPC(Ag, {"n": 40, "wall_geometry": "line_of_sight", "max_fr": 5.0, "history_bytes_limit": _limit(257, 40)})
    rb.PlaceCells(Ag, {"n": 64})
    return Ag


def behind_place(fused):
    Ag = _base(fused)
    rb.PlaceCells(Ag, {"n": 64, "wall_geometry": "line_of_sight"})
    PPPC(Ag, {"n": 130, "description": "gaussian", "kappa": 3, "max_fr": 4.0, "history_bytes_limit": _limit(257, 130)})
    PPPC(Ag, {"n": 20, "noise_std": 0.05})
    return Ag


def imported(fused):
    Ag = _base(fused)
    rng = np.random.default_rng(8)
    Ag.import_trajectory(times=np.cumsum(rng.uniform(0.05, 0.2, 20)), positions=rng.uniform(0.05, 0.95, (20, 2)))
    PPPC(Ag, {"n": 36, "description": "top_hat", "max_fr": 3.0})
    rb.PlaceCells(Ag, {"n": 12})
    return Ag


SETUPS = {
    # skewed: motion(0), then per step population 1 and the skewed launch of population 0
    "pppc_first": (pppc_first, lambda n: {"run": 1 + 2 * n, "run_fused": 1 + 2 * n, "step": 3 * n, "step_fused": 2 * n}),
    "behind_place": (behind_place, lambda n: {"run": 1 + 3 * n, "run_fused": 1 + 3 * n, "step": 4 * n, "step_fused": 3 * n}),
    # a motion source: the motion kernel, then every population
    "imported": (imported, lambda n: dict.fromkeys(WAYS, 3 * n)),
}


def _collect(Ag):
    out = {k: np.asarray(getattr(Ag, k)).copy() for k in STATE}
    out["t"] = np.array(Ag.t)
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
        Ag = build(way.endswith("fused"))
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
            pos, vel = _rows(Ag, "pos"), _rows(Ag, "velocity")
            for N in Ag.Neurons:
                if not isinstance(N, PPPC):
                    continue
                h = N.get_history_arrays()
                fr = h["firingrate"][-1].reshape(Ag.n_agents, N.n)
                if N.noise_std == 0:
                    _close(fr.T, _oracle(N, WALLS2, pos, vel, Ag.t), _bound(N))
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
    wrapped = [N for N in Ag.Neurons if N._hist_rows > N._hist_cap]
    assert len(wrapped) == (0 if name == "imported" else 1)


def test_ou_noise_statistics():
    """OU noise on top of the modulated rate: the difference to a noiseless copy of the population has mean 0 and the
    stationary standard deviation of the discrete OU update, noise_std sqrt(2 / (2 - dt / tau))."""
    np.random.seed(5)
    Ag = rb.Agent(_env([]), {"dt": 0.05, "n_agents": 4096, "seed": 3})
    prm = {"n": 16, "description": "gaussian", "max_fr": 2.0}
    N0 = PPPC(Ag, dict(prm, save_history=False))
    Nn = PPPC(Ag, dict(prm, place_cell_centres=N0.place_cell_centres, noise_std=0.3, noise_coherence_time=0.5,
                       save_history=False))
    Ag.run(100)
    diff = Nn.firingrate - N0.firingrate
    want = 0.3 * np.sqrt(2 / (2 - 0.05 / 0.5))
    assert abs(diff.std() / want - 1) < 0.02 and abs(diff.mean()) < 0.01, (diff.std(), want, diff.mean())


def test_nan_positions_give_zeros():
    np.random.seed(6)
    Ag = rb.Agent(_env(WALLS2), {"dt": 0.05, "n_agents": 66})
    N = PPPC(Ag, {"n": 64, "min_fr": 0.2, "wall_geometry": "line_of_sight"})
    Ag.update()
    pos = Ag.pos.copy()
    pos[[3, 40, 41]] = np.nan
    Ag.pos = pos
    N.update()
    fr = N.get_history_arrays()["firingrate"][-1]
    assert np.all(fr[[3, 40, 41]] == 0) and np.all(fr[[0, 1, 2, 4, 42]] > 0)


def test_edits_between_steps():
    """theta_freq, precess_fraction, sigma, widths and centres are read on every call; kappa is not."""
    np.random.seed(7)
    Ag = rb.Agent(_env(WALLS2), {"dt": 0.05, "n_agents": 129})
    N = PPPC(Ag, {"n": 70, "description": "gaussian", "wall_geometry": "line_of_sight", "max_fr": 2.0})
    Ag.update()
    N.update()
    pos, vel = _rows(Ag, "pos"), _rows(Ag, "velocity")
    last = N.firingrate.copy()

    def check(changed=True):
        nonlocal last
        N.update()
        fr = N.firingrate
        _close(fr.T, _oracle(N, WALLS2, pos, vel, Ag.t), _bound(N))
        assert (not np.array_equal(fr, last)) == changed
        last = fr.copy()

    N.kappa = 9.0
    check(changed=False)
    N.theta_freq = 6.0
    check()
    N.precess_fraction = 0.2
    check()
    N.sigma = np.sqrt(1 / 3.0)
    check()
    N.place_cell_widths = N.place_cell_widths * 1.3
    check()
    N.place_cell_centres = N.place_cell_centres + 0.02
    check()


def test_feedforward_layer_reads_the_cells_in_run():
    A = 300
    res = []
    for way in ("run", "step"):
        np.random.seed(2)
        Ag = rb.Agent(_env(WALLS2), {"dt": 0.05, "n_agents": A, "seed": 1})
        N = PPPC(Ag, {"n": 40, "wall_geometry": "line_of_sight", "max_fr": 3.0})
        L = rb.FeedForwardLayer(Ag, {"n": 20, "input_layers": [N], "name": "readout"})
        if way == "run":
            Ag.run(6)
        else:
            for _ in range(6):
                Ag.update()
                for M in Ag.Neurons:
                    M.update()
        res.append([M.get_history_arrays()["firingrate"] for M in (N, L)])
        p, out = (M.get_history_arrays()["firingrate"][-1].reshape(A, M.n) for M in (N, L))
        want = p @ L.inputs[N.name]["w"].T + L.biases
        scale = np.abs(p) @ np.abs(L.inputs[N.name]["w"]).T
        assert np.all(np.abs(out - want) <= 1e-5 * max(scale.max(), 1.0)), float(np.abs(out - want).max())
    for a, b in zip(*res):
        assert np.array_equal(a, b)


def test_raises_for_one_hot():
    Ag = rb.Agent(_env([]), {"dt": 0.05})
    with pytest.raises(AssertionError):
        PPPC(Ag, {"description": "one_hot"})


def test_matches_the_staged_live_reference():
    import ref_shim
    if ref_shim.import_reference() is None:
        pytest.skip("the reference is not staged under oracle/_ref")
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.contribs.PhasePrecessingPlaceCells import PhasePrecessingPlaceCells
    np.random.seed(21)
    RE = Environment()
    for w in WALLS2:
        RE.add_wall(w)
    RA = Agent(RE, {"dt": 0.05})
    prm = {"n": 30, "widths": 0.3, "theta_freq": 5, "precess_fraction": 1, "kappa": 2, "max_fr": 10.0,
           "description": "gaussian", "wall_geometry": "line_of_sight"}
    R = PhasePrecessingPlaceCells(RA, prm)
    Ag = rb.Agent(_env(WALLS2), {"dt": 0.05, "n_agents": 16, "seed": 4})
    N = PPPC(Ag, dict(prm, place_cell_centres=R.place_cell_centres))
    for _ in range(20):
        Ag.update()
        N.update()
        fr = N.firingrate
        for a in (0, 7, 15):
            RA.pos, RA.velocity, RA.t = _rows(Ag, "pos")[a], _rows(Ag, "velocity")[a], Ag.t
            _close(fr[a][:, None], R.get_state(), _bound(N))

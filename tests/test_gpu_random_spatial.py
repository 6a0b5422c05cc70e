"""RandomSpatialNeurons on the GPU (csrc/riab_rsn.cuh): the fused kernel-weighted average against the float64 oracle
and the live reference's fixture (tests/golden/rsn.npz) in every fixture environment, blocked decisions next to the
walls, an independent check through the existing PlaceCells kernel, NaN positions, bit equality of the stepped API,
the fused step and Agent.run (launch counts pinned), and the population as a FeedForwardLayer input.

The fixture's targets are loaded into the populations, so that LAPACK differences between machines drop out."""
import numpy as np
import pytest

import philox_np as PX
import riab_oracle as O
import riab_oracle_rsn as R

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                      # noqa: E402
from test_oracle_rsn import ENVS, _mirror_env, _oracle_env   # noqa: E402


def _population(name, g, n=None, **kw):
    """An Agent in fixture environment `name` with a RandomSpatialNeurons population holding the fixture's targets
    (or, for another n, targets drawn here in [min_fr, max_fr])."""
    spec, prm, seed = ENVS[name]
    np.random.seed(seed)
    Ag = rb.Agent(_mirror_env(spec), kw.pop("agent", {}))
    N = rb.RandomSpatialNeurons(Ag, dict(prm, name=name, **kw))
    assert np.array_equal(N.X, g[f"{name}_X"])
    if n is None:
        N.targets = g[f"{name}_targets"].copy()
    else:
        lo, hi = prm.get("min_fr", 0), prm.get("max_fr", 1)
        N.targets = np.random.RandomState(n).uniform(lo, hi, (N.X.shape[0], n))
    return Ag, N


def _bound(N):
    return 1e-5 * (N.max_fr - N.min_fr)


@pytest.mark.parametrize("name", list(ENVS))
def test_rates_match_the_oracle_and_the_reference(golden, name):
    g = golden("rsn.npz")
    Ag, N = _population(name, g)
    P = g[f"{name}_P"]
    got = N.get_state(evaluate_at=None, pos=P)
    want = R.get_state(_oracle_env(ENVS[name][0]), N.X, N.targets, N.lengthscale, N.wall_geometry, P, O.TapeRNG())
    assert np.array_equal(want, g[f"{name}_gs"])
    err = np.abs(got - want)
    print(name, N.X.shape[0], f"max |err| = {err.max():.2e}")
    assert got.shape == want.shape and np.all(err <= _bound(N)), float(err.max())


@pytest.mark.parametrize("n", [1, 10, 63, 64, 300])
@pytest.mark.parametrize("name", ["c2", "wall21", "holed"])
def test_rates_for_every_n_tile(golden, name, n):
    g = golden("rsn.npz")
    Ag, N = _population(name, g, n=n)
    P = g[f"{name}_P"]
    got = N.get_state(evaluate_at=None, pos=P)
    want = R.get_state(_oracle_env(ENVS[name][0]), N.X, N.targets, N.lengthscale, N.wall_geometry, P, O.TapeRNG())
    assert got.shape == (n, P.shape[0]) and np.all(np.abs(got - want) <= _bound(N)), float(np.abs(got - want).max())


def test_blocked_decisions_next_to_a_wall(golden):
    """Positions a hair on either side of the c2 walls and past their ends, with the target of the nearest sample point
    across the wall set far apart from the others: a wrong blocked decision on that heavily weighted point moves the
    rate by far more than the tolerance."""
    g = golden("rsn.npz")
    Ag, N = _population("c2", g, n=1)
    env = _oracle_env(ENVS["c2"][0])
    pts = []
    for x in (0.3, 0.7):
        for s in (1e-7, -1e-7, 2e-4, -2e-4):
            for y in np.linspace(0.05, 0.95, 19):
                pts.append([x + s, y])
    P = np.array(pts)
    T = np.zeros((N.X.shape[0], 1))
    j = np.argmin(np.abs(N.X[:, 0] - 0.325) + np.abs(N.X[:, 1] - 0.275))     # the point just right of wall 0
    T[j] = 1.0
    N.targets = T
    got = N.get_state(evaluate_at=None, pos=P)
    want = R.get_state(env, N.X, T, N.lengthscale, N.wall_geometry, P, O.TapeRNG())
    flip = R.get_state(env, N.X, T, N.lengthscale, "euclidean", P, O.TapeRNG())
    assert np.max(np.abs(flip - want)) > 100 * _bound(N)              # the decision matters at these positions
    assert np.all(np.abs(got - want) <= _bound(N)), float(np.abs(got - want).max())


@pytest.mark.parametrize("name", ["c2", "wall21", "periodic"])
def test_equals_normalised_place_cell_rates(golden, name):
    """Independent check: the rates equal normalise(PlaceCells over X, width l) @ targets in float64 from the existing
    place kernel's output."""
    g = golden("rsn.npz")
    Ag, N = _population(name, g)
    pc = rb.PlaceCells(Ag, {"n": N.X.shape[0], "place_cell_centres": N.X, "widths": N.lengthscale, "min_fr": 0,
                            "max_fr": 1, "wall_geometry": N.wall_geometry, "name": "PCX"})
    P = g[f"{name}_P"]
    k = pc.get_state(evaluate_at=None, pos=P).T
    want = ((k / k.sum(axis=1, keepdims=True)) @ N.targets).T
    got = N.get_state(evaluate_at=None, pos=P)
    assert np.all(np.abs(got - want) <= 2 * _bound(N)), float(np.abs(got - want).max())


def test_nan_positions_and_return_tensor(golden):
    g = golden("rsn.npz")
    Ag, N = _population("c2", g)
    P = g["c2_P"][:50].copy()
    P[[3, 17]] = np.nan
    r = N.get_state(evaluate_at=None, pos=P)
    assert np.all(r[:, [3, 17]] == 0) and np.all(np.isfinite(r))
    t = N.get_state(evaluate_at=None, pos=torch.as_tensor(P, device="cuda"), return_tensor=True)
    assert t.shape == (50, N.n) and np.array_equal(t.double().cpu().numpy().T, r)
    assert N.get_state(evaluate_at="all").shape == (N.n, Ag.Environment.flattened_discrete_coords.shape[0])


def _agent(A, noise=0.0, fused=False, rows=None):
    np.random.seed(3)
    env = _mirror_env(ENVS["c2"][0])
    Ag = rb.Agent(env, {"dt": 0.05, "n_agents": A, "seed": 7, "fused_step": fused})
    prm = {"n": 10, "lengthscale": 0.1, "noise_std": noise}
    if rows is not None:
        prm["history_bytes_limit"] = rows * A * 12 * 4
    N = rb.RandomSpatialNeurons(Ag, prm)
    return Ag, N


def _launches():
    return rb._lib.load().riab_launch_count()


@pytest.mark.parametrize("A", [1, 33, 4099])
def test_stepped_fused_and_run_are_bit_identical(A):
    T = 9
    res = {}
    for mode in ("stepped", "fused", "run", "run_fused"):
        Ag, N = _agent(A, fused=mode.endswith("fused"), rows=4)
        Ag.update()
        N.update()
        n0 = _launches()
        if mode.startswith("run"):
            Ag.run(T - 1)
        else:
            for _ in range(T - 1):
                Ag.update()
                N.update()
        pos = np.asarray(Ag.pos).reshape(A, 2).copy()                  # (reading the state runs a queued motion step)
        # per step: the motion kernel, k_rsn, and k_finish_rows for the spikes
        assert _launches() - n0 == 3 * (T - 1), (mode, _launches() - n0)
        h = N.get_history_arrays()
        assert N.history_dropped == T - 4                             # the 4-row ring wrapped
        res[mode] = (h["firingrate"], h["spikes"], pos)
        if mode == "stepped":
            fr = h["firingrate"][-1].reshape(A, N.n).astype(np.float32)
            sp = PX.expected_spikes(7, T - 1, np.arange(A), fr, 0.05, pop=N._population_id)
            assert np.array_equal(h["spikes"][-1].reshape(A, N.n), sp)
            ok = np.isfinite(pos[:, 0])
            direct = N.get_state(evaluate_at=None, pos=pos).T
            assert np.array_equal(direct[ok], h["firingrate"][-1].reshape(A, N.n)[ok])
    for mode in ("fused", "run", "run_fused"):
        for a, b in zip(res["stepped"], res[mode]):
            assert np.array_equal(a, b), mode


def test_noise_and_history_rate_maps():
    A = 64
    res = []
    for mode in ("stepped", "run"):
        Ag, N = _agent(A, noise=0.1)
        if mode == "run":
            Ag.run(5)
        else:
            for _ in range(5):
                Ag.update()
                N.update()
        res.append(N.get_history_arrays()["firingrate"])
        assert np.std(N._noise[:, : N.n].cpu().numpy()) > 0
    assert np.array_equal(res[0], res[1])
    maps = N.get_history_rate_maps(dx=0.1)
    assert maps.shape == (N.n, 10, 10) and np.all(np.isfinite(maps))
    assert N.firingrate.shape == (A, N.n)


def test_as_a_feedforward_layer_input():
    A = 257
    Ag, N = _agent(A)
    f = rb.FeedForwardLayer(Ag, {"n": 7, "input_layers": [N], "name": "F"})
    Ag.run(4)
    rows = N.get_history_arrays()["firingrate"][-1].reshape(A, N.n)
    got = f.get_history_arrays()["firingrate"][-1].reshape(A, 7)
    want = rows @ f.inputs[N.name]["w"].T + f.biases
    ok = np.isfinite(np.asarray(Ag.pos)[:, 0])
    assert np.allclose(got[ok], want[ok], rtol=0, atol=1e-5 * (np.abs(rows) @ np.abs(f.inputs[N.name]["w"]).T).max())
    assert np.all(got[~ok] == 0)


def test_matches_the_staged_live_reference(golden):
    import ref_shim
    if ref_shim.import_reference() is None:
        pytest.skip("the reference is not staged under oracle/_ref")
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import RandomSpatialNeurons
    g = golden("rsn.npz")
    Env = Environment()
    for w in ENVS["c2"][0]["walls"]:
        Env.add_wall(w)
    np.random.seed(3)
    ref = RandomSpatialNeurons(Agent(Env), {"n": 10, "lengthscale": 0.1})
    Ag, N = _population("c2", g)
    N.targets = ref.targets.copy()
    P = g["c2_P"][:128]
    orig = np.random.normal
    np.random.normal = lambda loc=0.0, scale=1.0, size=None: np.zeros(size) if scale == 1e-9 else orig(loc, scale, size)
    try:
        want = ref.get_state(evaluate_at=None, pos=P)
    finally:
        np.random.normal = orig
    assert np.all(np.abs(N.get_state(evaluate_at=None, pos=P) - want) <= _bound(N))

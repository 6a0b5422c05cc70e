"""PlaneWaveNeurons on the GPU (csrc/riab_pwn.cuh, k_step<PwnPolicy>): rates against the float64 oracle
(oracle/riab_oracle_pwn.py) within 1e-5 of |max_fr - min_fr| through update()'s history row, get_state() and the whole run,
for Rayleigh draws and hand-set wavelengths from 1 mm to 2 m at all orientations, in the unit box, at scale 10, in the
periodic box and in a polygon translated by (1000, -500) m, with both phase forms forced; bit equality of Agent.run, the
per-step loop, the stepped and the fused stepped API with pinned launch counts and wrapped rings, as a lone population,
as population 0, behind another population and under an imported trajectory; spikes against the Philox mirror; OU noise
statistics; NaN positions; edits between steps; the Neurons analytics; a FeedForwardLayer in run(); the staged live
reference."""
import numpy as np
import pytest

import philox_np as PX
import riab_oracle_pwn as W

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                                  # noqa: E402
from ratinabox_b200.contribs import PlaneWaveNeurons as PWN  # noqa: E402

WALLS2 = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
SHIFT = np.array([1000.0, -500.0])
LROOM = [[0, 0], [1, 0], [1, 0.5], [0.5, 0.5], [0.5, 1], [0, 1]]
STATE = ("pos", "velocity", "rotational_velocity", "measured_velocity", "measured_rotational_velocity",
         "head_direction", "distance_travelled", "distance_to_closest_wall")
WAYS = ("run", "run_perstep", "step", "step_fused")


def _env(kind):
    if kind == "unit":
        return rb.Environment()
    if kind == "walls":
        E = rb.Environment()
        for w in WALLS2:
            E.add_wall(w)
        return E
    if kind == "scale10":
        return rb.Environment({"scale": 10.0})
    if kind == "periodic":
        return rb.Environment({"boundary_conditions": "periodic"})
    if kind == "polygon_far":
        return rb.Environment({"boundary": (np.asarray(LROOM, dtype=float) + SHIFT).tolist()})
    raise KeyError(kind)


def _oracle(N, pos):
    return W.get_state(np.asarray(pos, dtype=float).reshape(-1, 2), N.phase_offsets, N.w, N.wavescales, N.min_fr, N.max_fr)


def _close(got, N, want, what=""):
    got = np.asarray(got, dtype=float)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    span = abs(float(N.max_fr) - float(N.min_fr))
    err = float(np.abs(got - want).max())
    assert err <= 1e-5 * span, f"{what}: max |err| {err:.3e} = {err / span:.2e} of the span"


def _points(E, rs, n=1500):
    e = E.extent
    lo, hi = np.array([e[0], e[2]]), np.array([e[1], e[3]])
    corners = np.array([[e[0], e[2]], [e[1], e[2]], [e[0], e[3]], [e[1], e[3]]])   # where |p - box centre| is largest
    return np.concatenate([lo + rs.uniform(size=(n, 2)) * (hi - lo), corners])


def _rows(Ag):
    return np.asarray(Ag.pos, dtype=float).reshape(Ag.n_agents, 2)


# ---- rates against the oracle
CASES = [(1, 1), (33, 7), (4099, 10), (257, 63), (4099, 301), (64, 1024), (4099, 1024)]


@pytest.mark.parametrize("kind", ["unit", "scale10", "periodic", "polygon_far"])
def test_rayleigh_rates_match_the_oracle(kind, capsys):
    """Rayleigh draws (the default wavescale 0.2, and 0.05): the update() history row, get_state() at the agents, at given
    positions and at "all"; min_fr > 0 and min_fr > max_fr in turn."""
    rs = np.random.RandomState(len(kind))
    for c, (A, n) in enumerate(CASES):
        Ag = rb.Agent(_env(kind), {"dt": 0.05, "n_agents": A, "seed": c})
        np.random.seed(200 + c)
        lo, hi = ((0.0, 1.0), (0.3, 2.5), (2.0, 0.5))[c % 3]
        N = PWN(Ag, {"n": n, "wavescale": (0.2, 0.05)[c % 2], "min_fr": lo, "max_fr": hi})
        for _ in range(3):
            Ag.update()
            N.update()
        want = _oracle(N, _rows(Ag))
        _close(N.get_history_arrays()["firingrate"][-1].reshape(A, n).T, N, want, f"{kind} {A}x{n} history")
        _close(N.get_state(), N, want, f"{kind} {A}x{n} get_state")
        X = _points(Ag.Environment, rs)
        _close(N.get_state(evaluate_at=None, pos=X), N, _oracle(N, X), f"{kind} {A}x{n} pos")
        if n >= 1024:
            assert N._cells().phase_turns == 1           # short Rayleigh waves: the compensated form
    all_pos = Ag.Environment.flattened_discrete_coords
    _close(N.get_state(evaluate_at="all"), N, _oracle(N, all_pos), f"{kind} all")
    printed = capsys.readouterr().out
    assert (W.PERIODIC_MESSAGE in printed) == (kind == "periodic")


@pytest.mark.parametrize("kind", ["unit", "scale10", "periodic", "polygon_far"])
@pytest.mark.parametrize("lam", [1e-3, 1e-2, 0.2, 2.0])
def test_hand_set_wavelengths_at_all_orientations(kind, lam):
    """24 orientations, offsets anywhere in the box; the pack's own choice, then each phase form forced where its error
    model keeps it within the bound (radians: |2 pi k| r_max <= 40)."""
    E = _env(kind)
    Ag = rb.Agent(E, {"dt": 0.05, "n_agents": 5})
    N = PWN(Ag, {"n": 24, "min_fr": 0.2, "max_fr": 3.0})
    ang = np.linspace(0, 2 * np.pi, 24, endpoint=False) + 0.01
    N.w = np.stack([np.cos(ang), np.sin(ang)], axis=1)
    N.wavescales = np.full(24, lam)
    rs = np.random.RandomState(int(lam * 1e4))
    e = E.extent
    N.phase_offsets = np.array([e[0], e[2]]) + rs.uniform(size=(24, 2)) * np.array([e[1] - e[0], e[3] - e[2]])
    X = _points(E, rs, 3000)
    want = _oracle(N, X)
    rmax = 0.5 * np.hypot(e[1] - e[0], e[3] - e[2])
    radians_ok = 2 * np.pi / lam * rmax <= 40
    assert N._cells().phase_turns == (0 if radians_ok else 1)
    _close(N.get_state(evaluate_at=None, pos=X), N, want, f"{kind} lam {lam} auto")
    for form in ((0, 1) if radians_ok else (1,)):
        N._phase_form = form
        assert N._cells().phase_turns == form
        _close(N.get_state(evaluate_at=None, pos=X), N, want, f"{kind} lam {lam} form {form}")


def test_non_unit_w_is_used_as_stored(golden):
    """The fixture's non-unit w, short waves and min_fr > max_fr, at its 384 positions and at "all"."""
    g = golden("pwn.npz")
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05})
    N = PWN(Ag, {"n": 24})
    for key in ("short1mm", "short1cm", "nonunit", "inverted"):
        N.phase_offsets, N.w, N.wavescales = g[f"{key}_phase_offsets"], g[f"{key}_w"], g[f"{key}_wavescales"]
        N.min_fr, N.max_fr = g[f"{key}_fr"]
        _close(N.get_state(evaluate_at=None, pos=g["pos_P"]), N, g[f"{key}_state"], key)
        if f"{key}_all" in g:
            _close(N.get_state(evaluate_at="all")[:, ::37], N, g[f"{key}_all"], key + " all")


def test_draws_equal_the_references(golden):
    g = golden("pwn.npz")
    for key in g["draw_keys"]:
        _, seed, n, ws = str(key).split("_")
        Ag = rb.Agent(rb.Environment(), {"dt": 0.05})
        np.random.seed(int(seed))
        N = PWN(Ag, {"n": int(n), "wavescale": float(ws)})
        for f in ("phase_offsets", "w", "wavescales"):
            assert np.array_equal(getattr(N, f), g[f"{key}_{f}"]), (key, f)


@pytest.mark.parametrize("kind", ["unit", "scale10", "polygon_far"])
def test_whole_run_matches_the_oracle(kind):
    """Agent.run's single launch: the last step's rates at the agents' float64 positions (the history's positions are
    float32, too coarse for short waves; earlier steps equal the stepped loop's bit for bit, test_run_and_stepped_...)."""
    from ratinabox_b200 import _lib
    lib = _lib.load()
    A, n, steps = 4099, 1024, 12
    Ag = rb.Agent(_env(kind), {"dt": 0.05, "n_agents": A, "seed": 3})
    np.random.seed(17)
    N = PWN(Ag, {"n": n, "wavescale": 0.2 * (10 if kind == "scale10" else 1), "min_fr": 0.1, "max_fr": 2.0})
    Ag.update()
    N.update()
    c0 = lib.riab_launch_count()
    Ag.run(steps)
    assert lib.riab_launch_count() - c0 == 1
    fr = N.get_history_arrays()["firingrate"]
    assert fr.shape == (1 + steps, A, n)
    _close(fr[-1].T, N, _oracle(N, _rows(Ag)), f"{kind} whole run")
    _close(N.firingrate.T, N, _oracle(N, _rows(Ag)), f"{kind} whole run firingrate")


# ---- launch paths
def _base(fused, A=257, E="walls"):
    np.random.seed(9)
    return rb.Agent(_env(E), {"dt": 0.02, "n_agents": A, "seed": 5, "fused_step": fused})


def _limit(A, n, rows=3):
    return rows * A * ((n + 3) // 4 * 4) * 4                # history rings of 3 rows: 5 steps wrap them


def lone(fused):
    Ag = _base(fused)
    PWN(Ag, {"n": 300, "max_fr": 2.0, "history_bytes_limit": _limit(257, 300)})
    return Ag


def lone_radians(fused):
    Ag = _base(fused)
    N = PWN(Ag, {"n": 260, "wavescale": 0.5, "max_fr": 2.0, "history_bytes_limit": _limit(257, 260)})
    N._phase_form = 0
    return Ag


def pwn_first(fused):
    Ag = _base(fused)
    PWN(Ag, {"n": 40, "max_fr": 5.0, "min_fr": 1.0, "history_bytes_limit": _limit(257, 40)})
    rb.PlaceCells(Ag, {"n": 64})
    return Ag


def behind_place(fused):
    Ag = _base(fused)
    rb.PlaceCells(Ag, {"n": 64, "wall_geometry": "line_of_sight"})
    PWN(Ag, {"n": 130, "max_fr": 4.0, "history_bytes_limit": _limit(257, 130)})
    PWN(Ag, {"n": 20, "noise_std": 0.05})
    return Ag


def imported(fused):
    Ag = _base(fused)
    rng = np.random.default_rng(8)
    Ag.import_trajectory(times=np.cumsum(rng.uniform(0.05, 0.2, 20)), positions=rng.uniform(0.05, 0.95, (20, 2)))
    PWN(Ag, {"n": 300, "max_fr": 3.0, "history_bytes_limit": _limit(257, 300)})
    return Ag


SETUPS = {
    # the whole run (more than 256 cells, a multiple of 4): ONE launch (MODE 3); stepped: motion + rates, or one fused launch
    "lone": (lone, lambda n: {"run": 1, "run_perstep": 1 + n, "step": 2 * n, "step_fused": n}),
    "lone_radians": (lone_radians, lambda n: {"run": 1, "run_perstep": 1 + n, "step": 2 * n, "step_fused": n}),
    # skewed: motion(0), then per step population 1 and the skewed launch of population 0
    "pwn_first": (pwn_first, lambda n: {"run": 1 + 2 * n, "run_perstep": 1 + 2 * n, "step": 3 * n, "step_fused": 2 * n}),
    "behind_place": (behind_place, lambda n: {"run": 1 + 3 * n, "run_perstep": 1 + 3 * n, "step": 4 * n,
                                              "step_fused": 3 * n}),
    # an imported trajectory: the whole run follows it in ONE launch (MODE 4); the per-step loop and the stepped API run
    # the trajectory's motion kernel, then the rates
    "imported": (imported, lambda n: {"run": 1, "run_perstep": 2 * n, "step": 2 * n, "step_fused": 2 * n}),
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
def test_run_and_stepped_are_bit_identical(name, monkeypatch):
    from ratinabox_b200 import _lib
    lib = _lib.load()
    build, launches = SETUPS[name]
    n = 5
    res, counts = {}, {}
    for way in WAYS:
        Ag = build(way == "step_fused")
        Ag.update()
        for N in Ag.Neurons:
            N.update()
        c0 = lib.riab_launch_count()
        if way.startswith("run"):
            with monkeypatch.context() as m:
                if way == "run_perstep":
                    m.setenv("RIAB_NO_WHOLE_RUN", "1")
                else:
                    m.delenv("RIAB_NO_WHOLE_RUN", raising=False)
                Ag.run(n)
        else:
            for _ in range(n):
                Ag.update()
                for N in Ag.Neurons:
                    N.update()
        res[way] = _collect(Ag)
        counts[way] = lib.riab_launch_count() - c0
        if way == "step":
            # the last step's rows against the oracle and the Philox mirror of the population's spike stream
            pos = _rows(Ag)
            for N in Ag.Neurons:
                if not isinstance(N, PWN):
                    continue
                h = N.get_history_arrays()
                fr = h["firingrate"][-1].reshape(Ag.n_agents, N.n)
                if N.noise_std == 0:
                    _close(fr.T, N, _oracle(N, pos), name)
                sp = PX.expected_spikes(5, N._upd - 1, np.arange(Ag.n_agents), fr.astype(np.float32), 0.02,
                                        pop=N._population_id)              # the dense stream (PwnPolicy::THIN = false)
                assert np.array_equal(h["spikes"][-1].reshape(Ag.n_agents, N.n), sp)
    assert counts == launches(n), counts
    ref = res["step"]
    for way in WAYS:
        for k in ref:
            x, y = np.asarray(res[way][k]), np.asarray(ref[k])
            assert x.shape == y.shape and np.array_equal(x, y, equal_nan=True), f"{name}: {way} vs step: {k}"
    assert any(np.asarray(v).any() for k, v in ref.items() if k.endswith(".spikes"))
    assert any(N._hist_rows > N._hist_cap for N in Ag.Neurons if isinstance(N, PWN) and N.noise_std == 0)


def test_ou_noise_statistics():
    """The difference to a noiseless copy has mean 0 and the stationary std of the discrete OU update."""
    Ag = rb.Agent(_env("unit"), {"dt": 0.05, "n_agents": 4096, "seed": 3})
    np.random.seed(5)
    N0 = PWN(Ag, {"n": 16, "max_fr": 2.0, "save_history": False})
    Nn = PWN(Ag, {"n": 16, "max_fr": 2.0, "noise_std": 0.3, "noise_coherence_time": 0.5, "save_history": False})
    Nn.phase_offsets, Nn.w, Nn.wavescales = N0.phase_offsets, N0.w, N0.wavescales
    Ag.run(100)
    diff = Nn.firingrate - N0.firingrate
    want = 0.3 * np.sqrt(2 / (2 - 0.05 / 0.5))
    assert abs(diff.std() / want - 1) < 0.02 and abs(diff.mean()) < 0.01, (diff.std(), want, diff.mean())


def test_nan_positions_give_zeros():
    Ag = rb.Agent(_env("walls"), {"dt": 0.05, "n_agents": 66})
    np.random.seed(6)
    N = PWN(Ag, {"n": 64, "min_fr": 0.2})
    Ag.update()
    pos = Ag.pos.copy()
    pos[[3, 40, 41]] = np.nan
    Ag.pos = pos
    N.update()
    fr = N.get_history_arrays()["firingrate"][-1]
    assert np.all(fr[[3, 40, 41]] == 0) and np.all(fr[[0, 1, 2, 4, 42]] > 0)


def test_edits_between_steps():
    """w, phase_offsets, wavescales, min_fr and max_fr are read on every call; wavescale is not."""
    Ag = rb.Agent(_env("walls"), {"dt": 0.05, "n_agents": 129})
    np.random.seed(7)
    N = PWN(Ag, {"n": 70, "max_fr": 2.0})
    Ag.update()
    N.update()
    pos = _rows(Ag)
    last = N.firingrate.copy()

    def check(changed=True):
        nonlocal last
        N.update()
        fr = N.firingrate
        _close(fr.T, N, _oracle(N, pos), "edit")
        assert (not np.array_equal(fr, last)) == changed
        last = fr.copy()

    N.wavescale = 0.01
    check(changed=False)
    N.w = N.w * 1.3
    check()
    N.phase_offsets = N.phase_offsets + 0.02
    check()
    N.wavescales = N.wavescales * 0.5
    check()
    N.wavescales[3] = 1e-3                                   # in place
    check()
    N.min_fr = 0.4
    check()
    N.max_fr = -1.0
    check()


def test_neurons_analytics():
    """get_head_direction_averaged_state is get_state (no head-direction tuning); get_history_rate_maps bins the
    history's rates by the history's positions."""
    Ag = rb.Agent(_env("unit"), {"dt": 0.05, "n_agents": 64, "seed": 2})
    np.random.seed(8)
    N = PWN(Ag, {"n": 9, "max_fr": 2.0})
    Ag.run(40)
    X = np.random.RandomState(2).uniform(0, 1, (50, 2))
    s = N.get_state(evaluate_at=None, pos=X)
    assert np.allclose(N.get_head_direction_averaged_state(evaluate_at=None, pos=X), s, rtol=0, atol=1e-6)
    maps, zero = N.get_history_rate_maps(dx=0.1, return_zero_bins=True)
    pos = Ag.get_history_arrays()["pos"].reshape(-1, 2)
    fr = N.get_history_arrays()["firingrate"].reshape(-1, 9)
    edges = np.arange(0, 1 + 0.1, 0.1)
    cnt = np.histogram2d(pos[:, 0], pos[:, 1], bins=[edges, edges])[0]
    for c in (0, 4, 8):
        ssum = np.histogram2d(pos[:, 0], pos[:, 1], bins=[edges, edges], weights=fr[:, c])[0]
        want = (ssum / np.maximum(cnt, 1)).T[::-1, :]
        assert np.allclose(maps[c], want, rtol=1e-9, atol=1e-9)


def test_feedforward_layer_reads_the_cells_in_run():
    A = 300
    res = []
    for way in ("run", "step"):
        np.random.seed(2)
        Ag = rb.Agent(_env("walls"), {"dt": 0.05, "n_agents": A, "seed": 1})
        N = PWN(Ag, {"n": 40, "max_fr": 3.0})
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


def test_matches_the_staged_live_reference():
    import ref_shim
    if ref_shim.import_reference() is None:
        pytest.skip("the reference is not staged under oracle/_ref")
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.contribs.PlaneWaveNeurons import PlaneWaveNeurons
    RE = Environment()
    for w in WALLS2:
        RE.add_wall(w)
    RA = Agent(RE, {"dt": 0.05})
    Ag = rb.Agent(_env("walls"), {"dt": 0.05, "n_agents": 16, "seed": 4})
    np.random.seed(21)
    R = PlaneWaveNeurons(RA, {"n": 30, "wavescale": 0.05, "max_fr": 10.0})
    np.random.seed(21)
    N = PWN(Ag, {"n": 30, "wavescale": 0.05, "max_fr": 10.0})
    assert all(np.array_equal(getattr(N, f), getattr(R, f)) for f in ("phase_offsets", "w", "wavescales"))
    for _ in range(20):
        Ag.update()
        N.update()
        fr = N.firingrate
        for a in (0, 7, 15):
            RA.pos = _rows(Ag)[a]
            _close(fr[a][:, None], N, R.get_state(), "live reference")

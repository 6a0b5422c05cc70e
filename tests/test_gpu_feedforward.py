"""FeedForwardLayer on the GPU (csrc/riab_ffl.cuh): the error-compensated TF32 GEMM against the float64 oracle on the
GPU's own float32 inputs, a case single-pass TF32 fails, the live reference's get_state (tests/golden/ffl.npz), bit
equality of the stepped API and Agent.run, and the edge cases of Neurons.update."""
import ctypes as C

import numpy as np
import pytest

import philox_np as PX
import riab_oracle_ffl as F

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                      # noqa: E402

BOX_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
ACTS = {"linear": {}, "sigmoid": {"max_fr": 2.0, "min_fr": 0.5, "mid_x": 0.3, "width_x": 1.5},
        "relu": {"gain": 1.5, "threshold": 0.1}, "tanh": {"gain": 0.8, "threshold": 0.2},
        "retanh": {"gain": 1.3, "threshold": -0.1}, "softmax": {"gain": 1.2, "threshold": -0.3}}


def _env():
    Env = rb.Environment()
    for w in BOX_WALLS:
        Env.add_wall(w)
    return Env


@pytest.fixture(scope="module")
def inputs():
    np.random.seed(1)
    Ag = rb.Agent(_env(), {"dt": 0.05})
    pc = rb.PlaceCells(Ag, {"n": 1024, "wall_geometry": "euclidean", "name": "PC"})
    gc = rb.GridCells(Ag, {"n": 300, "name": "GC"})       # K tail 300 % 32 != 0
    P = Ag.Environment.sample_positions(n=4096, method="random")
    Ipc = pc.get_state(evaluate_at=None, pos=P, return_tensor=True)
    Igc = gc.get_state(evaluate_at=None, pos=P, return_tensor=True)
    return Ag, pc, gc, P, Ipc, Igc


def _prime_at(ffl, rows):
    """phi'(V) over the given input tensors (riab_ffl_rates with a prime buffer), as float64 (n_rows, n)."""
    fc = type(ffl._cells()).from_buffer_copy(ffl._cells())
    n_rows = rows[0].shape[0]
    ld = ffl._ld()
    out = torch.empty((n_rows, ld), dtype=torch.float32, device="cuda")
    prime = torch.empty((n_rows, ld), dtype=torch.float32, device="cuda")
    fc.prime_dev = prime.data_ptr()
    for i, I in enumerate(rows):
        fc.inputs[i].rows_dev, fc.inputs[i].ld = I.data_ptr(), I.stride(0)
    ro = rb._lib.RatesOut()
    ro.rates_row, ro.ld = out.data_ptr(), ld
    rb._lib.check(ffl._lib.riab_ffl_rates(C.byref(fc), n_rows, None, None, C.byref(ro), None))
    torch.cuda.synchronize()
    return out[:, : ffl.n].double().cpu().numpy(), prime[:, : ffl.n].double().cpu().numpy()


@pytest.mark.parametrize("n", [1, 10, 256, 300])
@pytest.mark.parametrize("act", list(ACTS))
def test_gemm_matches_the_oracle_on_the_gpus_inputs(inputs, n, act):
    Ag, pc, gc, P, Ipc, Igc = inputs
    rs = np.random.RandomState(n)
    f = rb.FeedForwardLayer(Ag, {"n": n, "name": f"F{n}{act}", "activation_function": dict(ACTS[act], activation=act),
                                 "biases": rs.normal(0, 0.5, n)})
    f.add_input(pc, w=rs.normal(0, 1 / 32, (n, 1024)))
    f.add_input(gc, w=rs.normal(0, 1 / 17, (n, 300)))
    got = f.get_state(evaluate_at=None, pos=P)                        # (n, 4096)
    rates, prime = _prime_at(f, [Ipc, Igc])
    I1, I2 = Ipc.double().cpu().numpy().T, Igc.double().cpu().numpy().T
    W1, W2 = f.inputs["PC"]["w"], f.inputs["GC"]["w"]
    ins = [(W1, I1), (W2, I2)]
    want = F.ffl_get_state(ins, f.biases, act, ACTS[act])
    dwant = F.ffl_get_state(ins, f.biases, act, ACTS[act], deriv=True)
    scale = np.abs(W1) @ np.abs(I1) + np.abs(W2) @ np.abs(I2) + np.abs(f.biases)[:, None]
    bound = 1e-5 * scale * F.activation_lipschitz(act, ACTS[act]) + 1e-6
    assert np.all(np.abs(got - want) <= bound), np.max(np.abs(got - want) / bound)
    assert np.array_equal(rates.T, got)
    if act not in ("relu", "retanh"):                                  # derivatives of the kinks: compare off the kink
        assert np.all(np.abs(prime.T - dwant) <= bound), np.max(np.abs(prime.T - dwant) / bound)
    else:
        V = F.ffl_get_state(ins, f.biases, "linear")
        off = np.abs(V - ACTS[act]["threshold"]) > 1e-4 * scale
        assert np.all(np.abs(prime.T - dwant)[off] <= bound[off])


def test_positive_sums_are_fp32_accurate(inputs):
    """Positive weights and inputs: single-pass TF32 (10 mantissa bits, errors that cannot cancel here) is ~5e-4 off,
    the error-compensated GEMM must stay within 1e-5 relative."""
    Ag, pc, gc, P, Ipc, Igc = inputs
    rs = np.random.RandomState(5)
    f = rb.FeedForwardLayer(Ag, {"n": 256, "name": "Fpos"})
    f.add_input(pc, w=rs.uniform(0.5, 1.0, (256, 1024)))
    f.add_input(gc, w=rs.uniform(0.5, 1.0, (256, 300)))
    got = f.get_state(evaluate_at=None, pos=P)
    I1, I2 = Ipc.double().cpu().numpy().T, Igc.double().cpu().numpy().T
    want = f.inputs["PC"]["w"] @ I1 + f.inputs["GC"]["w"] @ I2
    rel = np.abs(got - want) / want
    print(f"max relative error {rel.max():.3e}")
    assert rel.max() <= 1e-5


def test_get_state_matches_the_live_reference(golden):
    g = golden("ffl.npz")
    Ag = rb.Agent(_env(), {"dt": 0.05})
    pc = rb.PlaceCells(Ag, {"n": 20, "wall_geometry": "line_of_sight", "name": "PC", "place_cell_centres": g["pc_centres"]})
    pc.place_cell_widths = g["pc_widths"].copy()
    gc = rb.GridCells(Ag, {"name": "GC", "gridscale": list(g["gc_gridscales"]), "phase_offset": g["gc_phase_offsets"],
                           "orientation": list(np.zeros(12))})
    gc.w = g["gc_w"].copy()
    mk = lambda name, n, act: rb.FeedForwardLayer(Ag, {"n": n, "name": name, "biases": g[f"{name}_biases"],  # noqa: E731
                                                       "activation_function": dict(ACTS[act], activation=act)})
    late, f1, f2, rec = mk("Late", 7, "relu"), mk("F1", 10, "sigmoid"), mk("F2", 6, "tanh"), mk("R", 5, "softmax")
    late.add_input(pc, w=g["Late_w_PC"])
    f1.add_input(pc, w=g["F1_w_PC"])
    f1.add_input(gc, w=g["F1_w_GC"])
    f2.add_input(f1, w=g["F2_w_F1"])
    rec.add_input(pc, w=g["R_w_PC"])
    rec.add_input(rec, w=g["R_w_R"], recurrent=True)
    P = g["P"]
    tol_in = 1e-5 + 0 * g["gs_PC"]
    assert np.all(np.abs(pc.get_state(evaluate_at=None, pos=P) - g["gs_PC"]) <= 1e-5)

    def bound(ws, Is, tols, b, act):
        s = sum(np.abs(w) @ (np.abs(I) + t) for w, I, t in zip(ws, Is, tols)) + np.abs(b)[:, None]
        prop = sum(np.abs(w) @ t for w, t in zip(ws, tols))
        return F.activation_lipschitz(act, ACTS[act]) * (1e-5 * s + prop) + 1e-7

    pcI, gcI = g["gs_PC"], g["gs_GC"]
    tpc, tgc = tol_in, 1e-5 + 0 * gcI
    checks = {}
    checks["Late"] = bound([g["Late_w_PC"]], [pcI], [tpc], g["Late_biases"], "relu")
    checks["F1"] = bound([g["F1_w_PC"], g["F1_w_GC"]], [pcI, gcI], [tpc, tgc], g["F1_biases"], "sigmoid")
    checks["F2"] = bound([g["F2_w_F1"]], [g["gs_F1"]], [checks["F1"]], g["F2_biases"], "tanh")
    r_in = F.ffl_get_state([(g["R_w_PC"], pcI)], g["R_biases"], "softmax", ACTS["softmax"])
    t_rin = bound([g["R_w_PC"]], [pcI], [tpc], g["R_biases"], "softmax")
    checks["R"] = bound([g["R_w_PC"], g["R_w_R"]], [pcI, r_in], [tpc, t_rin], g["R_biases"], "softmax")
    for name, layer in (("Late", late), ("F1", f1), ("F2", f2), ("R", rec)):
        got = layer.get_state(evaluate_at=None, pos=P, max_recurrence=1)
        assert got.shape == g[f"gs_{name}"].shape
        err = np.abs(got - g[f"gs_{name}"])
        assert np.all(err <= checks[name]), (name, float(np.max(err / checks[name])))


def _network(A, seed=3, noise=0.0, spikes=True):
    np.random.seed(seed)
    Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A, "seed": 7})
    small = {"history_bytes_limit": 3 * A * 12 * 4}                    # 3-row rings: they wrap
    late = rb.FeedForwardLayer(Ag, dict(small, n=7, name="Late", activation_function={"activation": "relu", "gain": 1.5},
                                        noise_std=noise, save_spikes=spikes))
    pc = rb.PlaceCells(Ag, {"n": 64, "name": "PC", "save_history": False})       # lagged input without history
    gc = rb.GridCells(Ag, {"n": 30, "name": "GC"})
    late.add_input(pc)
    f1 = rb.FeedForwardLayer(Ag, dict(small, n=10, name="F1", input_layers=[pc, gc],
                                      activation_function={"activation": "sigmoid", "max_fr": 2.0}, save_spikes=spikes))
    f2 = rb.FeedForwardLayer(Ag, dict(small, n=6, name="F2", input_layers=[f1], activation_function={"activation": "tanh"}))
    rec = rb.FeedForwardLayer(Ag, dict(small, n=5, name="R", input_layers=[pc], activation_function={"activation": "softmax"}))
    rec.add_input(rec, recurrent=True)
    return Ag, [late, f1, f2, rec]


@pytest.mark.parametrize("A", [1, 33, 4099])
def test_stepped_loop_and_run_are_bit_identical(A):
    T = 8
    Ag1, L1 = _network(A)
    Ag2, L2 = _network(A)
    for _ in range(T):
        Ag1.update()
        for N in Ag1.Neurons:
            N.update()
    Ag2.run(T)
    for a, b in zip(L1, L2):
        h1, h2 = a.get_history_arrays(), b.get_history_arrays()
        assert a.history_dropped > 0 and h1["firingrate"].shape[0] == T - a.history_dropped     # wrapped
        assert np.array_equal(h1["firingrate"], h2["firingrate"]), a.name
        assert np.array_equal(h1["spikes"], h2["spikes"]), a.name
        assert np.array_equal(a.firingrate_prime, b.firingrate_prime), a.name
        assert np.array_equal(h1["t"], h2["t"])
        want_shape = (a.n,) if A == 1 else (A, a.n)
        assert a.firingrate.shape == want_shape and a.firingrate_prime.shape == want_shape
        if a.save_spikes:                                                # the dense Philox stream of k_finish_rows
            fr = h1["firingrate"][-1].reshape(A, a.n).astype(np.float32)
            sp = PX.expected_spikes(7, T - 1, np.arange(A), fr, 0.05, pop=a._population_id)
            assert np.array_equal(h1["spikes"][-1].reshape(A, a.n), sp), a.name
    # timing: Late reads PC one step late, F1 reads PC / GC of the same step, R reads itself one step late
    late, f1, f2, rec = L1
    pcr = Ag1.Neurons[1]
    if A == 33:
        fr_pc = pcr.firingrate
        w = f1.inputs["PC"]["w"]
        gcr = f1.inputs["GC"]["layer"].firingrate
        V = fr_pc @ w.T + gcr @ f1.inputs["GC"]["w"].T + f1.biases
        assert np.allclose(f1.firingrate, F.activate(V, "sigmoid", False, {"max_fr": 2.0}), atol=1e-4)


def test_noise_and_edge_cases():
    A = 33
    Ag, (late, f1, f2, rec) = _network(A, noise=0.1)
    for _ in range(3):
        Ag.update()
        for N in Ag.Neurons:
            N.update()
    assert late._noise is not None and np.std(late._noise[:, :7].cpu().numpy()) > 0
    # NaN positions: zero rows (+ noise: none for F1) and unchanged primes
    prime0 = f1.firingrate_prime.copy()
    pos = Ag.pos.copy()
    pos[[0, 5]] = np.nan
    Ag.pos = pos
    f1.update()
    assert np.all(f1.firingrate[[0, 5]] == 0) and np.array_equal(f1.firingrate_prime[[0, 5]], prime0[[0, 5]])
    # NaN in the pad columns of an input ring never reaches an output
    gc = f1.inputs["GC"]["layer"]
    gc._hist[gc._last_slot][:, gc.n:] = float("nan")
    f2.update()
    f1.update()
    assert np.all(np.isfinite(f1.firingrate))
    # in-place edits of the weights and biases take effect on the next step
    f2.inputs["F1"]["w"][:] = 0.0
    f2.biases[:] = 0.25
    f2.update()
    ok = np.isfinite(Ag.pos[:, 0])
    assert np.allclose(f2.firingrate[ok], np.tanh(0.25), atol=1e-6) and np.all(f2.firingrate[~ok] == 0)

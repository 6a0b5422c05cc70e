"""ValueNeuron / SuccessorFeatures on the GPU (csrc/riab_td.cuh): the live reference's runs (tests/golden/td.npz) driven
along their recorded positions, the batched learning step against the float64 oracle on the device's own float32
state, replicated agents, bit equality of Agent.run and the stepped loop, the weights as host data, resets and the
reward forms."""
import numpy as np
import pytest

import riab_oracle_td as T

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                                    # noqa: E402
from ratinabox_b200.contribs import SuccessorFeatures, ValueNeuron   # noqa: E402

BOX_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
EPS32 = np.finfo(np.float32).eps


def _env():
    Env = rb.Environment()
    for w in BOX_WALLS:
        Env.add_wall(w)
    return Env


def _value_setup(g, A=1):
    Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A})
    pc = rb.PlaceCells(Ag, {"n": 20, "wall_geometry": "line_of_sight", "name": "PC", "place_cell_centres": g["v_pc_centres"]})
    pc.place_cell_widths = g["v_pc_widths"].copy()
    gc = rb.GridCells(Ag, {"name": "GC", "gridscale": list(g["v_gc_gridscales"]), "phase_offset": g["v_gc_phase_offsets"],
                           "orientation": list(np.zeros(12))})
    gc.w = g["v_gc_w"].copy()
    vn = ValueNeuron(Ag, {"tau": 1.0, "eta": 0.05, "L2": 0.01, "biases": g["v_biases"], "name": "VN",
                          "input_layers": [pc, gc]})
    vn.inputs["PC"]["w"] = g["v_W_PC"][0].copy()
    vn.inputs["GC"]["w"] = g["v_W_GC"][0].copy()
    return Ag, pc, gc, vn


def _dev(x, n):
    return x[:, :n].double().cpu().numpy()


def test_value_neuron_follows_the_live_reference(golden):
    g = golden("td.npz")
    Ag, pc, gc, vn = _value_setup(g)
    assert vn.tau_e == float(g["v_tau_e"])
    # bounds from float32 rates: V to 1e-5 of its terms' scale, dV/dt to 2 eps |V| / dt plus twice V's bound / dt, the
    # traces to 1e-5 of their size (float32 recurrence, ~eps / (dt / tau_e) relative), td to the sum of its parts; the
    # weights to 1e-5 (max|W0| + sum_t max|dW_t|)
    scale = np.abs(g["v_W_PC"][0]) @ np.abs(g["v_PC"].T) + np.abs(g["v_W_GC"][0]) @ np.abs(g["v_GC"].T) + np.abs(g["v_biases"])[:, None] + 1
    dW = sum(np.abs(np.diff(g[f"v_W_{k}"], axis=0)).max() for k in ("PC", "GC"))
    w_tol = 1e-5 * (max(np.abs(g["v_W_PC"][0]).max(), np.abs(g["v_W_GC"][0]).max()) + dW)
    for t in range(g["v_fr"].shape[0]):
        Ag.update(forced_next_position=g["v_pos"][t])
        for N in Ag.Neurons:
            N.update()
        vn.update_weights(g["v_reward"][t])
        fr_tol = 1e-5 * scale[0, t]
        assert abs(vn.firingrate[0] - g["v_fr"][t][0]) <= fr_tol, t
        assert abs(vn.firingrate_prime[0] - g["v_prime"][t][0]) <= 1e-6, t
        d_tol = (2 * EPS32 * abs(g["v_fr"][t][0]) + 2 * fr_tol) / 0.05
        assert abs(vn.firingrate_deriv[0] - g["v_deriv"][t][0]) <= d_tol, t
        for k in ("PC", "GC"):
            e = vn.inputs[k]["eligibility_trace"]
            assert np.all(np.abs(e - g[f"v_e_{k}"][t]) <= 1e-5 * (np.abs(g[f"v_e_{k}"][t]).max() + 1e-6)), (k, t)
        assert abs(vn.td_error[0] - g["v_td"][t][0]) <= d_tol + fr_tol + 1e-6, t
        if (t + 1) % 10 == 0:
            for k in ("PC", "GC"):
                assert np.all(np.abs(vn.inputs[k]["w"] - g[f"v_W_{k}"][(t + 1) // 10]) <= w_tol), (k, t)


def test_successor_features_follow_the_live_reference(golden):
    g = golden("td.npz")
    Ag = rb.Agent(_env(), {"dt": 0.05})
    feat = rb.PlaceCells(Ag, {"n": 6, "name": "Feat", "place_cell_centres": g["f_feat_centres"]})
    feat.place_cell_widths = g["f_feat_widths"].copy()
    gc = rb.GridCells(Ag, {"name": "GC", "gridscale": list(g["f_gc_gridscales"]), "phase_offset": g["f_gc_phase_offsets"],
                           "orientation": list(np.zeros(12))})
    gc.w = g["f_gc_w"].copy()
    sf = SuccessorFeatures(Ag, {"features": feat, "input_layers": [feat, gc], "eta": 0.3, "tau_e": 0.2})
    assert sf.n == 6
    sf.inputs["Feat"]["w"] = g["f_W0_Feat"].copy()
    sf.inputs["GC"]["w"] = g["f_W0_GC"].copy()
    # bounds as in the ValueNeuron test: V (relu) to 1e-5 of its terms' scale, taken with the larger of the first and last
    # recorded weights; the reward (the features' float32 rates) to 1e-5 of itself; dV/dt to 2 eps |V| / dt plus twice V's
    # bound / dt; td to the sum of its parts (tau = 2)
    Wmax = {k: np.maximum(np.abs(g[f"f_W0_{k}"]), np.abs(g[f"f_W_{k}"])) for k in ("Feat", "GC")}
    scale = Wmax["Feat"] @ np.abs(g["f_Feat"].T) + Wmax["GC"] @ np.abs(g["f_GC"].T) + 1        # (n, steps)
    for t in range(g["f_fr"].shape[0]):
        Ag.update(forced_next_position=g["f_pos"][t])
        feat.update()
        gc.update()
        sf.update()
        sf.update_weights()
        fr_tol = 1e-5 * scale[:, t]
        assert np.all(np.abs(sf.firingrate - g["f_fr"][t]) <= fr_tol), t
        d_tol = (2 * EPS32 * np.abs(g["f_fr"][t]) + 2 * fr_tol) / 0.05
        assert np.all(np.abs(sf.firingrate_deriv - g["f_deriv"][t]) <= d_tol), t
        r_tol = 1e-5 * np.abs(g["f_Feat"][t]) + 1e-7
        assert np.all(np.abs(sf.td_error - g["f_td"][t]) <= r_tol + d_tol + fr_tol / 2 + 1e-6), t
    for k in ("Feat", "GC"):
        W0 = g[f"f_W0_{k}"]
        tol = 1e-5 * (np.abs(W0).max() + 60 * np.abs(g[f"f_W_{k}"] - W0).max())
        assert np.all(np.abs(sf.inputs[k]["w"] - g[f"f_W_{k}"]) <= max(tol, 1e-6)), k


def _state(vn):
    """The device's float32 state as float64 host arrays."""
    n = vn.n
    return {"fr": _dev(vn._fr_prev, n), "deriv": _dev(vn._deriv, n), "prime": _dev(vn._prime, n),
            "td": _dev(vn._td, n), "e": {k: _dev(vn._trace[k], vn.inputs[k]["n"]) for k in vn.inputs},
            "W": {k: vn._master[k].cpu().numpy().copy() for k in vn.inputs}}


# n = 1: the CUDA-core path; 10, 300: the wgmma path with its cell (N) and input tails; A = 4093: a partial last round of
# 32 agents in every chunk's tail (the agent axis is the contraction's K)
@pytest.mark.parametrize("n,A", [(1, 4096), (10, 4096), (300, 4096), (1, 4093), (300, 4093)])
def test_batched_learning_matches_the_oracle_on_the_gpus_state(n, A):
    steps = 50
    np.random.seed(n)
    Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A, "seed": 11})
    pc = rb.PlaceCells(Ag, {"n": 100, "name": "PC", "save_history": False})
    gc = rb.GridCells(Ag, {"n": 40, "name": "GC", "save_history": False})
    rew = rb.PlaceCells(Ag, {"n": n, "name": "R", "widths": 0.3, "save_history": False})
    vn = ValueNeuron(Ag, {"n": n, "input_layers": [pc, gc], "tau": 1.0, "eta": 0.05, "L2": 0.01,
                          "biases": np.full(n, 0.3), "activation_function": {"activation": "softmax"},
                          "save_history": False})
    prev = None
    for t in range(steps):
        Ag.update()
        for N in Ag.Neurons:
            N.update()
        s = _state(vn)
        I = {"PC": _dev(pc._hist[pc._last_slot], 100), "GC": _dev(gc._hist[gc._last_slot], 40)}
        if prev is not None:                          # the trace step on the device's own rows
            for k in I:
                want = T.td_trace(prev["e"][k], I[k], 0.05, vn.tau_e)
                assert np.all(np.abs(s["e"][k] - want) <= 3 * EPS32 * (np.abs(0.05 * I[k]) + np.abs(prev["e"][k]))), k
            want_d = T.td_derivative(s["fr"], prev["fr"], 0.05)
            assert np.all(np.abs(s["deriv"] - want_d) <= 2 * EPS32 * np.abs(want_d) + 1e-30)
        r = _dev(rew._hist[rew._last_slot], n)
        vn.update_weights(rew)
        after = _state(vn)
        W = {k: s["W"][k].copy() for k in vn.inputs}
        td = T.td_learn([W[k] for k in vn.inputs], [s["e"][k] for k in vn.inputs], r, s["fr"], s["deriv"], s["prime"],
                        0.05, 1.0, 0.05, 0.01)
        assert np.all(np.abs(after["td"] - td) <= 4 * EPS32 * (np.abs(r) + np.abs(s["deriv"]) + np.abs(s["fr"]))), t
        bounds = T.td_learn_bound([s["e"][k] for k in vn.inputs], r, s["fr"], s["deriv"], s["prime"], 1.0)
        for (k, b) in zip(vn.inputs, bounds):
            err = np.abs((after["W"][k] - s["W"][k]) - (W[k] - s["W"][k]))
            tol = 0.05 * 0.05 * 1e-5 * b + 1e-15 * np.abs(s["W"][k])
            assert np.all(err <= tol), (k, t, np.max(err / np.maximum(tol, 1e-300)))
        prev = after


def test_replicated_agents_learn_the_single_agent_weights(golden):
    g = golden("td.npz")
    Ag1, _, _, v1 = _value_setup(g, 1)
    Ag2, _, _, v2 = _value_setup(g, 256)
    for t in range(100):
        Ag1.update(forced_next_position=g["v_pos"][t])
        Ag2.update(forced_next_position=np.tile(g["v_pos"][t], (256, 1)))
        for Ag, v in ((Ag1, v1), (Ag2, v2)):
            for N in Ag.Neurons:
                N.update()
            v.update_weights(g["v_reward"][t])
    for k in ("PC", "GC"):
        W1, W2 = v1.inputs[k]["w"], v2.inputs[k]["w"]
        assert np.all(np.abs(W2 - W1) <= 1e-6 * np.abs(W1).max()), k
    assert np.array_equal(v2.firingrate, np.tile(v1.firingrate, (256, 1)))


def _net(A, seed=5):
    np.random.seed(seed)
    Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A, "seed": 9})
    small = {"history_bytes_limit": 3 * A * 12 * 4}                   # 3-row rings: they wrap
    pc = rb.PlaceCells(Ag, dict(small, n=12, name="PC"))
    gc = rb.GridCells(Ag, dict(small, n=9, name="GC"))
    vn = ValueNeuron(Ag, dict(small, n=10, name="VN", input_layers=[pc, gc], noise_std=0.05,
                              activation_function={"activation": "tanh", "gain": 0.7}))
    vn.add_input(vn, recurrent=True, w_init_scale=0.3)
    vn.inputs["VN"]["eligibility_trace"] = np.zeros(10)
    rew = rb.PlaceCells(Ag, dict(small, n=10, name="R", widths=0.3))
    return Ag, vn, rew


def test_run_and_stepped_loop_are_bit_identical():
    A, steps = 777, 7
    Ag1, v1, r1 = _net(A)
    Ag2, v2, r2 = _net(A)
    for _ in range(steps):
        Ag1.update()
        for N in Ag1.Neurons:
            N.update()
    Ag2.run(steps)
    for a, b in ((v1, v2), (r1, r2)):                                  # the real columns (pads are never written)
        assert a._hist_cap == b._hist_cap == 3 and a._hist_rows == b._hist_rows == steps      # wrapped
        assert torch.equal(a._hist[:, :, : a.n], b._hist[:, :, : b.n])
    for k in v1.inputs:
        assert torch.equal(v1._trace[k], v2._trace[k])
    for x, y in ((v1._deriv, v2._deriv), (v1._fr_prev, v2._fr_prev), (v1._prime, v2._prime)):
        assert torch.equal(x, y)
    for _ in range(3):
        v1.update_weights(r1)
        v2.update_weights(r2)
    for k in v1.inputs:
        assert torch.equal(v1._master[k], v2._master[k]) and torch.equal(v1._w_pack[k], v2._w_pack[k])
    # learning in the stepped loop, twice from the same start: the same bits
    for _ in range(5):
        for Ag, v, r in ((Ag1, v1, r1), (Ag2, v2, r2)):
            Ag.update()
            for N in Ag.Neurons:
                N.update()
            v.update_weights(r)
    for k in v1.inputs:
        assert torch.equal(v1._master[k], v2._master[k])


def test_weights_are_host_data_and_edits_take_effect():
    lib = rb._lib.load()
    Ag, vn, rew = _net(64)
    for _ in range(3):
        Ag.update()
        for N in Ag.Neurons:
            N.update()
        vn.update_weights(rew)
    for k in vn.inputs:
        w = vn.inputs[k]["w"]
        assert np.array_equal(w, vn._master[k].cpu().numpy())
        host = np.zeros(lib.riab_ffl_pack_floats(vn.n, w.shape[1]), dtype=np.float32)
        meta = rb._lib.FflInput()
        rb._lib.check(lib.riab_ffl_pack(w.ctypes.data_as(rb._lib.c_double_p), vn.n, w.shape[1], __import__("ctypes").byref(meta),
                                        host.ctypes.data_as(rb._lib.c_float_p)))
        assert np.array_equal(host, vn._w_pack[k].cpu().numpy())
    # in-place scaling, an element write and an assignment all reach the device before the next use
    vn.inputs["PC"]["w"] *= 0.1
    w = vn.inputs["GC"]["w"]
    w[0, 0] = 1.25
    vn.inputs["VN"]["w"] = np.zeros((10, 10))
    want_pc = vn.inputs["PC"]["w"].copy()
    Ag.update()
    for N in Ag.Neurons:
        N.update()
    assert np.array_equal(vn._master["PC"].cpu().numpy(), want_pc)
    assert vn._master["GC"][0, 0].item() == 1.25
    assert not vn._master["VN"].any()
    for k in vn.inputs:                   # the operands the next update's GEMM read
        w = vn._master[k].cpu().numpy()
        host = np.zeros(lib.riab_ffl_pack_floats(vn.n, w.shape[1]), dtype=np.float32)
        rb._lib.check(lib.riab_ffl_pack(w.ctypes.data_as(rb._lib.c_double_p), vn.n, w.shape[1],
                                        __import__("ctypes").byref(rb._lib.FflInput()), host.ctypes.data_as(rb._lib.c_float_p)))
        assert np.array_equal(host, vn._w_pack[k].cpu().numpy()), k


def test_resets_and_reward_forms():
    A = 32
    Ag, vn, rew = _net(A)
    for _ in range(3):
        Ag.update()
        for N in Ag.Neurons:
            N.update()
    mask = np.zeros(A, dtype=bool)
    mask[[1, 5, 7]] = True
    e0 = vn.inputs["PC"]["eligibility_trace"]
    fr0 = vn.firingrate
    vn.reset(agents=mask)
    e1, fr1 = vn.inputs["PC"]["eligibility_trace"], vn.firingrate
    assert not e1[mask].any() and not fr1[mask].any() and not vn.firingrate_deriv[mask].any()
    assert np.array_equal(e1[~mask], e0[~mask]) and np.array_equal(fr1[~mask], fr0[~mask])
    vn.reset(agents=[0, 2])
    assert not vn.firingrate[[0, 2]].any() and vn.firingrate[3].any()
    vn.reset()
    assert not vn.firingrate.any() and not vn.td_error.any() and not vn.inputs["GC"]["eligibility_trace"].any()
    for _ in range(2):
        Ag.update()
        for N in Ag.Neurons:
            N.update()
    n = vn.n
    W0 = {k: vn._master[k].clone() for k in vn.inputs}
    # 0.25 is exact in float32, so the per-agent (float32) and shared (float64) forms give the same update
    forms = [np.full(n, 0.25), [0.25] * n, np.full((A, n), 0.25), torch.full((A, n), 0.25, device="cuda"),
             torch.full((n,), 0.25, device="cuda", dtype=torch.float64)]
    results = []
    for r in forms:
        for k in vn.inputs:
            vn._master[k].copy_(W0[k])
        vn.update_weights(r)
        results.append({k: vn._master[k].clone() for k in vn.inputs})
    for res in results[1:]:
        for k in vn.inputs:
            assert torch.equal(res[k], results[0][k]), k
    vn.update_weights(rew)
    for bad in (np.zeros(3), np.zeros((A, n + 1)), torch.zeros(5, device="cuda")):
        with pytest.raises(AssertionError):
            vn.update_weights(bad)
    with pytest.raises(ValueError):
        vn.update_weights(rb.PlaceCells(Ag, {"n": 3, "name": "R3"}))
    # n == 1: an (A,) reward is per agent
    v1 = ValueNeuron(Ag, {"n": 1, "input_layers": [vn.inputs["PC"]["layer"]], "name": "V1"})
    Ag.update()
    for N in Ag.Neurons:
        N.update()
    W0 = v1._master["PC"].clone()
    v1.update_weights(np.linspace(0, 1, A, dtype=np.float32).astype(np.float64))
    W1 = v1._master["PC"].clone()
    v1._master["PC"].copy_(W0)
    v1.update_weights(torch.linspace(0, 1, A, device="cuda"))
    assert torch.equal(v1._master["PC"], W1) and not torch.equal(W0, W1)
    v1.update_weights(0.25)
    v1.update_weights(torch.tensor(0.25, device="cuda"))


def test_construction_errors_match_the_reference(golden):
    import json
    errs = json.loads(str(golden("td.npz")["errors_json"]))
    Ag = rb.Agent(_env(), {"dt": 0.05})
    pc = rb.PlaceCells(Ag, {"n": 5, "name": "PC"})
    with pytest.raises(Exception) as ei:
        SuccessorFeatures(Ag, {"input_layers": [pc]})
    assert str(ei.value) == errs["sf_no_features"][1]
    vz = ValueNeuron(Ag, {"input_layers": [pc], "tau_e": 0, "name": "VZ"})
    Ag.update()
    pc.update()
    with pytest.raises(AttributeError, match="no attribute 'firingrate'"):
        vz.update()
    vl = ValueNeuron(Ag, {"input_layers": [pc], "name": "VL"})
    vl.add_input(rb.PlaceCells(Ag, {"n": 3, "name": "Late"}))
    with pytest.raises(KeyError):
        vl.update()
    with pytest.raises(KeyError):
        vl.inputs["Late"]["eligibility_trace"]
    vr = ValueNeuron(Ag, {"n": 2, "input_layers": [pc], "name": "VR"})
    import contextlib
    import io
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf), pytest.raises(AssertionError):
        vr.update_weights(np.zeros(3))
    assert buf.getvalue() == errs["reward_length"][2]

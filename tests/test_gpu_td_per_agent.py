"""ValueNeuron / SuccessorFeatures with per_agent_weights on the GPU (csrc/riab_td.cuh, k_td_forward_pa and
k_td_learn_pa): one batch tracking K independent live-reference runs (tests/golden/td_pa.npz), the learning step and
the forward pass against the float64 per-agent oracle on the device's own float32 state, independence of the agents,
agreement with the shared path for one agent, shards, Agent.run against the stepped loop, and the weights as host
data."""
import numpy as np
import pytest

import riab_oracle_ffl as F
import riab_oracle_td as T
import riab_oracle_td_pa as P

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                                    # noqa: E402
from ratinabox_b200.contribs import SuccessorFeatures, ValueNeuron   # noqa: E402

BOX_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
EPS32 = np.finfo(np.float32).eps
EPS64 = np.finfo(np.float64).eps


def _env():
    Env = rb.Environment()
    for w in BOX_WALLS:
        Env.add_wall(w)
    return Env


def _dev(x, n):
    return x[:, :n].double().cpu().numpy()


def _step(Ag, pos=None):
    Ag.update() if pos is None else Ag.update(forced_next_position=pos)
    for N in Ag.Neurons:
        N.update()


def _golden_setup(g, A):
    Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A})
    pc = rb.PlaceCells(Ag, {"n": 20, "wall_geometry": "line_of_sight", "name": "PC", "place_cell_centres": g["pc_centres"]})
    pc.place_cell_widths = g["pc_widths"].copy()
    gc = rb.GridCells(Ag, {"name": "GC", "gridscale": list(g["gc_gridscales"]), "phase_offset": g["gc_phase_offsets"],
                           "orientation": list(np.zeros(12))})
    gc.w = g["gc_w"].copy()
    return Ag, pc, gc


def test_each_agent_follows_its_own_live_reference_run(golden):
    g = golden("td_pa.npz")
    K = g["fr"].shape[0]
    Ag, pc, gc = _golden_setup(g, K)
    vn = ValueNeuron(Ag, {"tau": 1.0, "eta": 0.05, "L2": 0.01, "biases": g["biases"][0], "name": "VN",
                          "input_layers": [pc, gc], "per_agent_weights": True})
    assert vn.tau_e == float(g["tau_e"])
    vn.inputs["PC"]["w"] = g["W_PC"][:, 0].copy()                      # (K, 1, 20): each run's own initial weights
    vn.inputs["GC"]["w"] = g["W_GC"][:, 0].copy()
    # the bounds of the shared path's golden test (tests/test_gpu_td.py), per run
    for k in range(K):
        assert np.array_equal(g["biases"][k], g["biases"][0])
    scale = np.stack([np.abs(g["W_PC"][k, 0]) @ np.abs(g["PC"][k].T) + np.abs(g["W_GC"][k, 0]) @ np.abs(g["GC"][k].T)
                      + np.abs(g["biases"][k])[:, None] + 1 for k in range(K)])[:, 0]      # (K, steps)
    for t in range(g["fr"].shape[1]):
        _step(Ag, np.tile(g["pos"][t], (K, 1)))
        vn.update_weights(g["reward"][:, t, 0])                            # (A,) with n == 1: one reward per agent
        fr, prime, td = vn.firingrate[:, 0], vn.firingrate_prime[:, 0], vn.td_error[:, 0]
        fr_tol = 1e-5 * scale[:, t]
        assert np.all(np.abs(fr - g["fr"][:, t, 0]) <= fr_tol), t
        assert np.all(np.abs(prime - g["prime"][:, t, 0]) <= 1e-6), t
        d_tol = (2 * EPS32 * np.abs(g["fr"][:, t, 0]) + 2 * fr_tol) / 0.05
        assert np.all(np.abs(td - g["td"][:, t, 0]) <= d_tol + fr_tol + 1e-6), t
        for key in ("PC", "GC"):
            e, want = vn.inputs[key]["eligibility_trace"], g[f"e_{key}"][:, t]
            assert np.all(np.abs(e - want) <= 1e-5 * (np.abs(want).max() + 1e-6)), (key, t)
        if (t + 1) % 10 == 0:
            for key in ("PC", "GC"):
                W = g[f"W_{key}"]
                dW = sum(np.abs(np.diff(g[f"W_{k2}"], axis=1)).max() for k2 in ("PC", "GC"))
                w_tol = 1e-5 * (max(np.abs(g["W_PC"][:, 0]).max(), np.abs(g["W_GC"][:, 0]).max()) + dW)
                assert np.all(np.abs(vn.inputs[key]["w"] - W[:, (t + 1) // 10]) <= w_tol), (key, t)


def _state(vn):
    n = vn.n
    return {"fr": _dev(vn._fr_prev, n), "deriv": _dev(vn._deriv, n), "prime": _dev(vn._prime, n),
            "td": _dev(vn._td, n), "e": {k: _dev(vn._trace[k], vn.inputs[k]["n"]) for k in vn.inputs},
            "W": {k: vn._master[k].cpu().numpy().copy() for k in vn.inputs}}


def _check_learning_step(vn, reward, steps_state):
    """One update_weights against the oracle's per-agent update on the device's own float32 td, phi' and traces."""
    s = steps_state
    vn.update_weights() if reward is None else vn.update_weights(reward)
    after = _state(vn)
    W = {k: s["W"][k].copy() for k in vn.inputs}
    P.td_apply_pa([W[k] for k in vn.inputs], [s["e"][k] for k in vn.inputs], after["td"], s["prime"],
                  vn.Agent.dt, vn.eta, vn.L2)
    for k in vn.inputs:
        g = np.abs(after["td"] * s["prime"])
        bound = np.abs(s["W"][k]) + vn.Agent.dt * vn.eta * g[:, :, None] * np.abs(s["e"][k])[:, None, :]
        err = np.abs(after["W"][k] - W[k])
        assert np.all(err <= 4 * EPS64 * bound), (k, np.max(err / np.maximum(bound, 1e-300)))
    return after


@pytest.mark.parametrize("n,A", [(1, 4096), (3, 1000), (70, 300)])
def test_learning_step_matches_the_oracle_on_the_gpus_state(n, A):
    np.random.seed(n)
    Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A, "seed": 11})
    pc = rb.PlaceCells(Ag, {"n": 100, "name": "PC", "save_history": False})
    gc = rb.GridCells(Ag, {"n": 40, "name": "GC", "save_history": False})
    rew = rb.PlaceCells(Ag, {"n": n, "name": "R", "widths": 0.3, "save_history": False})
    vn = ValueNeuron(Ag, {"n": n, "input_layers": [pc, gc], "tau": 1.0, "eta": 0.05, "L2": 0.01,
                          "biases": np.full(n, 0.3), "activation_function": {"activation": "softmax"},
                          "save_history": False, "per_agent_weights": True})
    vn.inputs["PC"]["w"] = np.random.normal(size=(A, n, 100)) * 0.1
    vn.inputs["GC"]["w"] = np.random.normal(size=(A, n, 40)) * 0.1
    for t in range(20):
        _step(Ag)
        s = _state(vn)
        I = {"PC": _dev(pc._hist[pc._last_slot], 100), "GC": _dev(gc._hist[gc._last_slot], 40)}
        # forward: the float64 per-agent contraction, rounded once to float32 before the activation
        V = sum(np.einsum("anj,aj->an", s["W"][k], I[k]) for k in I) + 0.3
        want_fr = F.activate(V, "softmax")
        assert np.all(np.abs(s["fr"] - want_fr) <= 4 * EPS32 * (np.abs(want_fr) + np.abs(V) + 1e-30)), t
        _check_learning_step(vn, rew, s)


def test_get_state_shapes_and_values():
    A, n = 6, 2
    np.random.seed(2)
    Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A})
    pc = rb.PlaceCells(Ag, {"n": 30, "name": "PC"})
    gc = rb.GridCells(Ag, {"n": 10, "name": "GC"})
    vn = ValueNeuron(Ag, {"n": n, "input_layers": [pc, gc], "activation_function": {"activation": "linear"},
                          "biases": np.array([0.1, -0.2]), "per_agent_weights": True})
    Wpc, Wgc = np.random.normal(size=(A, n, 30)), np.random.normal(size=(A, n, 10))
    vn.inputs["PC"]["w"], vn.inputs["GC"]["w"] = Wpc, Wgc
    n_all = Ag.Environment.flattened_discrete_coords.shape[0]
    full = vn.get_state("all")
    assert full.shape == (A, n, n_all)
    Ipc, Igc = pc.get_state("all"), gc.get_state("all")                    # (n_in, n_pos)
    want = np.einsum("anj,jp->anp", Wpc, Ipc) + np.einsum("anj,jp->anp", Wgc, Igc) + np.array([0.1, -0.2])[:, None]
    assert np.all(np.abs(full - want) <= 4 * EPS32 * (np.abs(np.einsum("anj,jp->anp", np.abs(Wpc), Ipc))
                                                       + np.einsum("anj,jp->anp", np.abs(Wgc), np.abs(Igc)) + 0.2))
    pos = np.array([[0.1, 0.2], [0.5, 0.9], [0.8, 0.3]])
    some = vn.get_state(evaluate_at=None, pos=pos, agents=[4, 1])
    assert some.shape == (2, n, 3)
    every = vn.get_state(evaluate_at=None, pos=pos)
    assert every.shape == (A, n, 3) and np.array_equal(some, every[[4, 1]])
    _step(Ag)
    last = vn.get_state("last")
    assert last.shape == (n, A) and np.array_equal(last, vn.firingrate.T)
    assert np.allclose(vn.get_state("agent"), last, rtol=1e-5, atol=1e-6)


def test_agents_are_independent_and_replicas_identical():
    A, n = 8, 3
    nets = []
    for _ in range(2):
        np.random.seed(1)
        Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A, "seed": 3})
        pc = rb.PlaceCells(Ag, {"n": 25, "name": "PC"})
        vn = ValueNeuron(Ag, {"n": n, "input_layers": [pc], "per_agent_weights": True, "eta": 0.5})
        nets.append((Ag, vn))
    pos = np.tile([[0.2, 0.2]], (A, 1))
    for t in range(10):
        r = np.full((A, n), 0.5)
        for i, (Ag, vn) in enumerate(nets):
            _step(Ag, pos + 0.01 * t)
            rr = r.copy()
            if i == 1:
                rr[3] = 2.0                                                    # only agent 3's reward differs
            vn.update_weights(rr)
    W1, W2 = nets[0][1]._master["PC"], nets[1][1]._master["PC"]
    others = [a for a in range(A) if a != 3]
    assert torch.equal(W1[others], W2[others]) and not torch.equal(W1[3], W2[3])
    # every agent of net 0 saw the same inputs, weights and rewards: identical rows
    fr = nets[0][1].firingrate
    assert np.array_equal(fr, np.tile(fr[0], (A, 1)))
    assert all(torch.equal(W1[a], W1[0]) for a in range(A))


def test_one_agent_agrees_with_the_shared_path(golden):
    g = golden("td_pa.npz")
    nets = []
    for pa in (False, True):
        Ag, pc, gc = _golden_setup(g, 1)
        vn = ValueNeuron(Ag, {"tau": 1.0, "eta": 0.05, "L2": 0.01, "biases": g["biases"][0], "name": "VN",
                              "input_layers": [pc, gc], "per_agent_weights": pa})
        vn.inputs["PC"]["w"] = g["W_PC"][1, 0].copy()
        vn.inputs["GC"]["w"] = g["W_GC"][1, 0].copy()
        nets.append((Ag, vn))
    for t in range(100):
        for Ag, vn in nets:
            _step(Ag, g["pos"][t])
            vn.update_weights(g["reward"][1, t])
    (_, v0), (_, v1) = nets
    for k in ("PC", "GC"):
        assert v1.inputs[k]["w"].shape == v0.inputs[k]["w"].shape
        assert np.all(np.abs(v1.inputs[k]["w"] - v0.inputs[k]["w"]) <= 1e-6 * np.abs(v0.inputs[k]["w"]).max()), k
    assert abs(v1.firingrate[0] - v0.firingrate[0]) <= 1e-5 * (abs(v0.firingrate[0]) + 1)


def test_a_shard_gives_its_rows_of_the_full_batch():
    A, lo, hi, n = 64, 16, 40, 4
    rs = np.random.RandomState(0)
    W = rs.normal(size=(A, n, 30))
    pos = rs.uniform(0.05, 0.95, (12, A, 2))
    rewards = rs.uniform(0, 1, (12, A, n))

    def net(n_agents, off):
        Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": n_agents, "id_offset": off, "seed": 5})
        np.random.seed(6)                                               # the same cells in both batches
        pc = rb.PlaceCells(Ag, {"n": 30, "name": "PC"})
        vn = ValueNeuron(Ag, {"n": n, "input_layers": [pc], "per_agent_weights": True, "eta": 0.2})
        vn.inputs["PC"]["w"] = W[off:off + n_agents].copy()
        return Ag, vn
    Ag_f, v_f = net(A, 0)
    Ag_s, v_s = net(hi - lo, lo)
    for t in range(12):
        _step(Ag_f, pos[t])
        _step(Ag_s, pos[t, lo:hi])
        v_f.update_weights(rewards[t])
        v_s.update_weights(rewards[t, lo:hi])
        assert np.array_equal(v_s.firingrate, v_f.firingrate[lo:hi]), t
    assert torch.equal(v_s._master["PC"], v_f._master["PC"][lo:hi])


def _net(A, seed=5):
    np.random.seed(seed)
    Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A, "seed": 9})
    small = {"history_bytes_limit": 3 * A * 12 * 4}                   # 3-row rings: they wrap
    pc = rb.PlaceCells(Ag, dict(small, n=12, name="PC"))
    gc = rb.GridCells(Ag, dict(small, n=9, name="GC"))
    vn = ValueNeuron(Ag, dict(small, n=10, name="VN", input_layers=[pc, gc], noise_std=0.05, per_agent_weights=True,
                              activation_function={"activation": "tanh", "gain": 0.7}))
    vn.add_input(vn, recurrent=True, w_init_scale=0.3)
    vn.inputs["VN"]["eligibility_trace"] = np.zeros(10)
    vn.inputs["PC"]["w"] = np.random.normal(size=(A, 10, 12)) * 0.3
    rew = rb.PlaceCells(Ag, dict(small, n=10, name="R", widths=0.3))
    return Ag, vn, rew


def test_run_and_stepped_loop_are_bit_identical():
    A, steps = 777, 7
    Ag1, v1, r1 = _net(A)
    Ag2, v2, r2 = _net(A)
    for _ in range(steps):
        _step(Ag1)
    Ag2.run(steps)
    for a, b in ((v1, v2), (r1, r2)):
        assert a._hist_cap == b._hist_cap == 3 and a._hist_rows == b._hist_rows == steps      # wrapped
        assert torch.equal(a._hist[:, :, : a.n], b._hist[:, :, : b.n])
    for k in v1.inputs:
        assert torch.equal(v1._trace[k], v2._trace[k]) and torch.equal(v1._master[k], v2._master[k])
    for x, y in ((v1._deriv, v2._deriv), (v1._fr_prev, v2._fr_prev), (v1._prime, v2._prime)):
        assert torch.equal(x, y)
    for _ in range(3):
        for Ag, v, r in ((Ag1, v1, r1), (Ag2, v2, r2)):
            _step(Ag)
            v.update_weights(r)
    for k in v1.inputs:
        assert torch.equal(v1._master[k], v2._master[k])


def test_weights_are_host_data_resets_and_reward_forms():
    A = 16
    Ag, vn, rew = _net(A)
    n = vn.n
    assert vn.inputs["PC"]["w"].shape == (A, n, 12) and vn.inputs["VN"]["w"].shape == (A, n, n)
    # construction: the reference's (n, n_in) draw, given to every agent
    W = vn.inputs["GC"]["w"]
    assert all(np.array_equal(W[a], W[0]) for a in range(A))
    for _ in range(3):
        _step(Ag)
        vn.update_weights(rew)
    # in-place edits, a broadcast and a per-agent assignment reach the device before the next use
    vn.inputs["PC"]["w"][2] *= 0.5
    vn.inputs["GC"]["w"] = np.full((n, 9), 0.125)
    per = np.random.normal(size=(A, n, n))
    vn.inputs["VN"]["w"] = per
    want_pc = vn.inputs["PC"]["w"].copy()
    _step(Ag)
    assert np.array_equal(vn._master["PC"].cpu().numpy(), want_pc)
    assert np.all(vn._master["GC"].cpu().numpy() == 0.125) and vn.inputs["GC"]["w"].shape == (A, n, 9)
    assert np.array_equal(vn._master["VN"].cpu().numpy(), per)
    with pytest.raises(ValueError):
        vn.inputs["GC"]["w"] = np.zeros((A + 1, n, 9))
        _step(Ag)
    vn.inputs["GC"]["w"] = np.full((n, 9), 0.125)
    # reset leaves the weights alone
    W0 = {k: vn._master[k].clone() for k in vn.inputs}
    vn.reset(agents=[1, 3])
    vn.reset()
    assert all(torch.equal(W0[k], vn._master[k]) for k in vn.inputs)
    assert not vn.firingrate.any()
    _step(Ag)
    _step(Ag)
    W0 = {k: vn._master[k].clone() for k in vn.inputs}
    forms = [0.25 if n == 1 else np.full(n, 0.25), [0.25] * n, np.full((A, n), 0.25),
             torch.full((A, n), 0.25, device="cuda"), torch.full((n,), 0.25, device="cuda", dtype=torch.float64)]
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
    # n == 1: (A,) is one reward per agent; one agent reads (n, n_in)
    v1 = ValueNeuron(Ag, {"n": 1, "input_layers": [vn.inputs["PC"]["layer"]], "name": "V1", "per_agent_weights": True})
    _step(Ag)
    W0 = v1._master["PC"].clone()
    v1.update_weights(np.linspace(0, 1, A, dtype=np.float32).astype(np.float64))
    W1 = v1._master["PC"].clone()
    v1._master["PC"].copy_(W0)
    v1.update_weights(torch.linspace(0, 1, A, device="cuda"))
    assert torch.equal(v1._master["PC"], W1) and not torch.equal(W1[0], W1[-1])
    v1.update_weights(0.25)
    Ag1 = rb.Agent(_env(), {"dt": 0.05})
    p1 = rb.PlaceCells(Ag1, {"n": 7, "name": "P"})
    u = ValueNeuron(Ag1, {"input_layers": [p1], "per_agent_weights": True})
    _step(Ag1)
    assert u.inputs["P"]["w"].shape == (1, 7) and u.get_state("all").shape[0] == 1


def test_memory_error_names_the_bytes():
    A = 65536
    Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A})
    pc = rb.PlaceCells(Ag, {"n": 1024, "name": "PC", "save_history": False})
    n_before = len(Ag.Neurons)
    need = 8 * A * 1024 * 1024
    with pytest.raises(MemoryError, match=f"{need} bytes"):
        SuccessorFeatures(Ag, {"features": pc, "input_layers": [pc], "per_agent_weights": True})
    assert len(Ag.Neurons) == n_before


def test_successor_features_per_agent_against_the_oracle():
    A, n = 128, 64
    np.random.seed(8)
    Ag = rb.Agent(_env(), {"dt": 0.05, "n_agents": A, "seed": 2})
    feat = rb.PlaceCells(Ag, {"n": n, "name": "Feat", "widths": 0.2})
    sf = SuccessorFeatures(Ag, {"features": feat, "input_layers": [feat], "eta": 0.3, "tau_e": 0.2,
                                "per_agent_weights": True})
    assert sf.inputs["Feat"]["w"].shape == (A, n, n)
    sf.inputs["Feat"]["w"] *= 0.1
    for t in range(15):
        _step(Ag)
        s = _state(sf)
        I = _dev(feat._hist[feat._last_slot], n)
        V = np.einsum("anj,aj->an", s["W"]["Feat"], I)
        want = np.maximum(V, 0)
        assert np.all(np.abs(s["fr"] - want) <= 4 * EPS32 * (np.einsum("anj,aj->an", np.abs(s["W"]["Feat"]), I) + 1e-30)), t
        after = _check_learning_step(sf, None, s)
        td = T.td_error(I, s["fr"], s["deriv"], sf.tau)
        assert np.all(np.abs(after["td"] - td) <= 4 * EPS32 * (np.abs(I) + np.abs(s["deriv"]) + np.abs(s["fr"]))), t

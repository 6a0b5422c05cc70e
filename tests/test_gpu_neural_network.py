"""NeuralNetworkNeurons on the GPU (csrc/riab_nnn.cuh, k_nnn): the fused forward against the float64 oracle
(oracle/riab_oracle_nnn.py) next to torch's own float32 forward, the live reference's run and get_state
(tests/golden/nnn.npz), Agent.run against the stepped loop (wrapped rings, an input read one step late), the generic path,
training through firingrate_torch, and noise, spikes, NaN positions and a FeedForwardLayer reading the network."""
import numpy as np
import pytest

import philox_np as PX
import riab_oracle_ffl as F
import riab_oracle_nnn as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import torch.nn as nn                                                  # noqa: E402

import ratinabox_b200 as rb                                            # noqa: E402
from ratinabox_b200.contribs import MultiLayerPerceptron, NeuralNetworkNeurons as NNN   # noqa: E402

ACT = {nn.ReLU: "relu", nn.Sigmoid: "sigmoid", nn.Tanh: "tanh", nn.Identity: "identity"}


def _chain(module):
    """The oracle's chain of a Sequential / MultiLayerPerceptron."""
    mods = [m for m in module.modules() if type(m) in (nn.Linear,) + tuple(ACT)]
    out = []
    for m in mods:
        if type(m) is nn.Linear:
            out.append([m.weight.detach().double().cpu().numpy(),
                        None if m.bias is None else m.bias.detach().double().cpu().numpy(), "identity"])
        elif type(m) is not nn.Identity:
            out[-1][2] = ACT[type(m)]
    return [tuple(c) for c in out]


def _X(N):
    """The rows the network read at its last update: the inputs' firing-rate rows concatenated (float32, device)."""
    return N._gather(N._input_rows(), N.Agent.n_agents)


def _accuracy(N):
    """(max |kernel - oracle|, max |torch float32 - oracle|) on the population's last update."""
    X = _X(N)
    got = N._hist[N._last_slot][:, : N.n].double().cpu().numpy()
    want = O.forward(X.double().cpu().numpy(), _chain(N.NeuralNetworkModule))
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            ref = N.NeuralNetworkModule(X).double().cpu().numpy()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return float(np.abs(got - want).max()), float(np.abs(ref - want).max())


def _net(A, n_pc, n_gc, module=None, n=None, seed=0, **kw):
    np.random.seed(seed)
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05, "n_agents": A, "seed": seed})
    pc = rb.PlaceCells(Ag, {"n": n_pc, "save_history": False})
    ins = [pc]
    if n_gc:
        ins.append(rb.GridCells(Ag, {"n": n_gc, "save_history": False}))
    torch.manual_seed(seed)
    p = dict(kw, input_layers=ins)
    p.update({"NeuralNetworkModule": module} if module is not None else {"n": n})
    with pytest.warns(UserWarning) if module is None else _nullcontext():
        N = NNN(Ag, p)
    return Ag, ins, N


class _nullcontext:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def _step(Ag, k=1):
    for _ in range(k):
        Ag.update()
        for ns in Ag.Neurons:
            ns.update()


def _check_accuracy(N, what):
    err, err_torch = _accuracy(N)
    print(f"{what}: kernel {err:.3e}, torch float32 {err_torch:.3e}")
    assert err <= max(2 * err_torch, 1e-7), (what, err, err_torch)


# ---- accuracy against the oracle, next to torch's float32 forward
@pytest.mark.parametrize("A", [1, 37, 65536])
def test_default_mlp_accuracy(A):
    Ag, _, N = _net(A, 256, 128, n=10)
    assert N.fused and type(N.NeuralNetworkModule) is MultiLayerPerceptron
    _step(Ag, 2)
    _check_accuracy(N, f"default MLP, {A} agents")


@pytest.mark.parametrize("act", [nn.ReLU, nn.Sigmoid, nn.Tanh, nn.Identity])
def test_three_hidden_layers_of_each_activation(act):
    torch.manual_seed(1)
    m = nn.Sequential(nn.Linear(300, 64), act(), nn.Linear(64, 48), act(), nn.Linear(48, 33), act(), nn.Linear(33, 7))
    Ag, _, N = _net(37, 200, 100, module=m)
    assert N.fused and N.n == 7
    _step(Ag, 2)
    _check_accuracy(N, act.__name__)


@pytest.mark.parametrize("n_in", [1, 31, 32, 100, 385, 1000, 2048])
def test_input_widths(n_in):
    torch.manual_seed(n_in)
    m = nn.Sequential(nn.Linear(n_in, 96), nn.ReLU(), nn.Linear(96, 20), nn.Tanh(), nn.Linear(20, 3))
    Ag, _, N = _net(37, n_in, 0, module=m)
    _step(Ag)
    _check_accuracy(N, f"n_in {n_in}")


def test_wide_and_single_layer_networks():
    """Hidden width 256 (layer 1 in 4 column chunks), a single Linear with 200 outputs, and 65 536 agents."""
    torch.manual_seed(5)
    wide = nn.Sequential(nn.Linear(384, 256), nn.ReLU(), nn.Linear(256, 256), nn.ReLU(), nn.Linear(256, 5))
    Ag, _, N = _net(65536, 256, 128, module=wide)
    assert N.fused
    _step(Ag)
    _check_accuracy(N, "256 wide, 65536 agents")
    torch.manual_seed(6)
    Ag, _, N = _net(37, 256, 128, module=nn.Sequential(nn.Linear(384, 200), nn.Sigmoid()))
    assert N.fused
    _step(Ag)
    _check_accuracy(N, "single Linear")


# ---- the live reference
def _golden_net(g, Ag):
    pc = rb.PlaceCells(Ag, {"n": 30, "place_cell_centres": g["run_pc_centres"]})
    pc.place_cell_widths = g["run_pc_widths"].copy()
    gc = rb.GridCells(Ag, {"n": 12, "gridscale": list(g["run_gc_gridscales"]), "phase_offset": g["run_gc_phase_offsets"],
                           "orientation": list(np.zeros(12))})
    gc.w = g["run_gc_w"].copy()
    torch.manual_seed(0)
    with pytest.warns(UserWarning) as ws:
        N = NNN(Ag, {"input_layers": [pc, gc], "n": 5})
    assert str(g["default_warning"]) in [str(w.message) for w in ws]
    return pc, gc, N


def test_golden_native_run_and_get_state(golden):
    g = golden("nnn.npz")
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05})
    pc, gc, N = _golden_net(g, Ag)
    sd = N.NeuralNetworkModule.state_dict()                      # the reference's initial weights under the same seed
    for k in g["mlp_keys"]:
        assert np.array_equal(sd[str(k)].cpu().numpy(), g[f"mlp_sd_{k}"]), k
    for s in range(len(g["run_pos"])):
        Ag.update(forced_next_position=g["run_pos"][s])
        pc.update()
        gc.update()
        N.update()
        assert np.abs(pc.firingrate - g["run_pc"][s]).max() <= 1e-5 and np.abs(gc.firingrate - g["run_gc"][s]).max() <= 1e-5
        assert np.abs(N.firingrate - g["run_fr"][s]).max() <= 1e-5, s
        assert N.firingrate_torch.shape == (1, 5)
        assert np.abs(N.firingrate_torch.detach().cpu().numpy()[0] - g["run_fr_torch"][s]).max() <= 1e-5
    assert N.get_state().shape == (5, 1)
    assert np.abs(N.get_state(evaluate_at=None, pos=g["pos_P"]) - g["pos_state"]).max() <= 1e-5
    assert np.abs(N.get_state(evaluate_at="all")[:, ::37] - g["all_state"]).max() <= 1e-5
    for key, module in (("seq", nn.Sequential(nn.Linear(42, 16), nn.Tanh(), nn.Linear(16, 3), nn.Sigmoid())),
                        ("nobias", nn.Sequential(nn.Linear(42, 8, bias=False), nn.ReLU(), nn.Linear(8, 4)))):
        module.load_state_dict({str(k): torch.as_tensor(g[f"{key}_sd_{k}"]) for k in g[f"{key}_keys"]})
        S = NNN(Ag, {"input_layers": [pc, gc], "NeuralNetworkModule": module})
        assert S.fused
        assert np.abs(S.get_state(evaluate_at=None, pos=g["pos_P"]) - g[f"{key}_state"]).max() <= 1e-5, key


def test_construction_errors(golden):
    g = golden("nnn.npz")
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05})
    pc = rb.PlaceCells(Ag, {"n": 30})
    with pytest.raises(ValueError) as e:
        NNN(Ag, {"input_layers": [pc], "n": 3, "NeuralNetworkModule": nn.Linear(30, 3)})
    assert str(e.value) == str(g["err_both"])
    with pytest.raises(ValueError) as e:
        NNN(Ag, {"input_layers": [pc]})
    assert str(e.value) == str(g["err_neither"])
    with pytest.raises(ValueError) as e:
        NNN(Ag, {"input_layers": [pc], "NeuralNetworkModule": nn.Linear(31, 2)})
    assert str(e.value) == str(g["err_probe"])
    with pytest.raises(AssertionError):
        NNN(Ag, {"input_layers": [], "n": 2})
    other = rb.PlaceCells(rb.Agent(rb.Environment()), {"n": 4})
    with pytest.raises(ValueError):
        NNN(Ag, {"input_layers": [other], "n": 2})


# ---- Agent.run against the stepped loop
def _run_net(A, late):
    np.random.seed(4)
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05, "n_agents": A, "seed": 9})
    pc = rb.PlaceCells(Ag, {"n": 64})
    gc = rb.GridCells(Ag, {"n": 40})
    torch.manual_seed(3)
    m = MultiLayerPerceptron(104, 6, [32, 20])
    N = NNN(Ag, {"input_layers": [pc, gc], "NeuralNetworkModule": m, "history_bytes_limit": 3 * A * 8 * 4})   # wraps
    if late:                                            # an input registered after the network: read one step late
        gc2 = rb.GridCells(Ag, {"n": 40, "save_history": False})
        N.input_layers = [pc, gc2]
    return Ag, N


@pytest.mark.parametrize("A", [1, 33, 4099])
@pytest.mark.parametrize("late", [False, True])
def test_run_equals_the_stepped_loop(A, late):
    T = 7
    Ag1, N1 = _run_net(A, late)
    Ag2, N2 = _run_net(A, late)
    _step(Ag1, 2)
    _step(Ag2, 2)
    _step(Ag1, T)
    Ag2.run(T)
    h1, h2 = N1.get_history_arrays(), N2.get_history_arrays()
    assert N1.history_dropped > 0                           # the ring wrapped
    assert np.array_equal(h1["firingrate"], h2["firingrate"])
    assert np.array_equal(h1["spikes"], h2["spikes"])
    assert np.array_equal(N1.firingrate, N2.firingrate)
    for a, b in zip(Ag1.Neurons, Ag2.Neurons):
        assert np.array_equal(a.firingrate, b.firingrate), a.name
    if late:
        assert N1._cells().inputs[1].lag == 1


# ---- generic path
def test_generic_module():
    torch.manual_seed(2)
    m = nn.Sequential(nn.Linear(50, 16), nn.LayerNorm(16), nn.Linear(16, 4))
    Ag, _, N = _net(33, 50, 0, module=m)
    assert not N.fused
    _step(Ag, 2)
    X = _X(N)
    with torch.no_grad():
        want = m(X).cpu().numpy()
    assert np.array_equal(N.firingrate, want.astype(np.float64))
    assert N.firingrate_torch.requires_grad and N.firingrate_torch.shape == (33, 4)
    P = np.random.RandomState(0).uniform(size=(100, 2))
    Ipc = N.input_layers[0].get_state(evaluate_at=None, pos=P, return_tensor=True)
    with torch.no_grad():
        assert np.array_equal(N.get_state(evaluate_at=None, pos=P), m(Ipc.contiguous()).T.double().cpu().numpy())
    with pytest.raises(NotImplementedError, match="LayerNorm"):
        Ag.run(3)
    wide = nn.Sequential(nn.Linear(50, 300), nn.ReLU(), nn.Linear(300, 2))
    Ag, _, N = _net(5, 50, 0, module=wide)
    assert not N.fused
    with pytest.raises(NotImplementedError, match="width 300"):
        Ag.run(2)


# ---- training
def test_gradients_equal_torch_autograd():
    Ag, _, N = _net(64, 80, 40, n=3)
    _step(Ag, 2)
    X = _X(N)
    target = torch.randn(64, 3, device=X.device)
    params = list(N.NeuralNetworkModule.parameters())
    # a loss linear in the rates: both graphs receive the same upstream gradient
    g1 = torch.autograd.grad((N.firingrate_torch * target).sum(), params)
    g2 = torch.autograd.grad((N.NeuralNetworkModule(X) * target).sum(), params)
    for a, b in zip(g1, g2):
        assert torch.equal(a, b)


def test_adam_reduces_a_regression_loss_and_repacks_on_edits():
    Ag, (pc, gc), N = _net(256, 64, 32, n=2, seed=8)
    _step(Ag)
    opt = torch.optim.Adam(N.NeuralNetworkModule.parameters(), lr=3e-3)
    losses = []
    for it in range(200):
        Ag.update()
        pc.update()
        gc.update()
        packs = N._n_packs
        N.update()
        assert N._n_packs == packs + (1 if it > 0 else 0)       # one re-pack after each opt.step(), none otherwise
        N.update()
        assert N._n_packs == packs + (1 if it > 0 else 0)
        pos = torch.as_tensor(Ag.pos, dtype=torch.float32, device=N.firingrate_torch.device)
        loss = ((N.firingrate_torch - pos) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert np.mean(losses[-20:]) < 0.5 * np.mean(losses[:20]), (losses[:3], losses[-3:])
    # the next update uses the new weights: its rates equal the module's on the same rows
    N.update()
    with torch.no_grad():
        want = N.NeuralNetworkModule(_X(N)).cpu().numpy()
    assert np.abs(N.firingrate - want).max() <= 1e-5


# ---- composition
def test_noise_spikes_nan_and_a_feedforward_reader():
    A = 33
    Ag, (pc, gc), N = _net(A, 64, 32, n=5, noise_std=0.1)
    ffl = rb.FeedForwardLayer(Ag, {"n": 4, "input_layers": [N], "activation_function": {"activation": "tanh"}})
    _step(Ag, 3)
    assert N._noise is not None and np.std(N._noise[:, :5].cpu().numpy()) > 0
    with torch.no_grad():
        clean = N.NeuralNetworkModule(_X(N)).cpu().numpy()
    assert np.abs(N.firingrate_torch.detach().cpu().numpy() - clean).max() <= 1e-5      # firingrate_torch: no noise
    noisy = N.firingrate
    assert np.abs(noisy - clean - N._noise[:, :5].cpu().numpy()).max() <= 1e-5
    # the FeedForwardLayer reading the network's row of this step
    want = F.ffl_get_state([(ffl.inputs[N.name]["w"], noisy.T)], ffl.biases, "tanh").T
    assert np.abs(ffl.firingrate - want).max() <= 1e-5
    # spikes: the dense Philox stream of k_finish_rows
    Ag2, _, M = _net(A, 64, 32, n=5, seed=4)
    _step(Ag2, 2)
    fr = M._hist[M._last_slot][:, :5].cpu().numpy()
    sp = PX.expected_spikes(int(Ag2.seed), M._upd - 1, np.arange(A), fr, 0.05, pop=M._population_id)
    assert np.array_equal(M.get_history_arrays()["spikes"][-1], sp)
    # NaN positions: zero rows
    pos = Ag2.pos.copy()
    pos[[0, 5]] = np.nan
    Ag2.pos = pos
    M.update()
    assert np.all(M.firingrate[[0, 5]] == 0) and np.all(M.firingrate[[1, 2]] != 0)


def test_spike_statistics():
    """Spike counts of a constant-rate network follow rate * dt (the FeedForwardLayer's statistical check)."""
    A, T = 4096, 20
    torch.manual_seed(0)
    m = nn.Sequential(nn.Linear(8, 4))
    with torch.no_grad():
        m[0].weight.zero_()
        m[0].bias.copy_(torch.tensor([2.0, 5.0, 10.0, 0.0]))
    Ag, _, N = _net(A, 8, 0, module=m)
    counts = np.zeros(4)
    for _ in range(T):
        _step(Ag)
        counts += N.get_history_arrays()["spikes"][-1].sum(axis=0)
    p = np.array([2.0, 5.0, 10.0, 0.0]) * 0.05
    expect = p * A * T
    sd = np.sqrt(A * T * p * (1 - p))
    assert counts[3] == 0 and np.all(np.abs(counts[:3] - expect[:3]) <= 5 * sd[:3]), (counts, expect)

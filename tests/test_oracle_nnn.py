"""CPU checks of NeuralNetworkNeurons: the float64 oracle (oracle/riab_oracle_nnn.py) against the live reference's fixture
(tests/golden/nnn.npz, oracle/gen_nnn_golden.py), MultiLayerPerceptron's initial weights, the reference's messages, the
riab_nnn_cells layout and riab_nnn_pack's block.  No CUDA calls."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

import riab_oracle_nnn as O

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _state(g, key):
    return {str(k): g[f"{key}_sd_{k}"] for k in g[f"{key}_keys"]}


ACTS = {"mlp": ["relu", "relu", "identity"], "seq": ["tanh", "sigmoid"], "nobias": ["relu", "identity"]}


def _f32_close(want64, got32):
    """got32 (the reference's float32 forward) equals the float64 forward within float32 rounding of the terms."""
    err = np.abs(np.asarray(got32, dtype=np.float64) - want64)
    assert err.max() <= 1e-6 * max(1.0, np.abs(want64).max()), err.max()


def test_oracle_reproduces_the_native_run(golden):
    g = golden("nnn.npz")
    chain = O.chain_from_state_dict(_state(g, "mlp"), ACTS["mlp"])
    X = np.concatenate([g["run_pc"], g["run_gc"]], axis=1).astype(np.float32)
    want = O.forward(X, chain)
    _f32_close(want, g["run_fr"])
    _f32_close(want, g["run_fr_torch"])


@pytest.mark.parametrize("key", ["mlp", "seq", "nobias"])
def test_oracle_reproduces_get_state(golden, key):
    g = golden("nnn.npz")
    chain = O.chain_from_state_dict(_state(g, key), ACTS[key])
    pos = O.get_state([g["pos_pc"].astype(np.float32), g["pos_gc"].astype(np.float32)], chain)
    _f32_close(pos, g["pos_state" if key == "mlp" else f"{key}_state"])
    if key == "mlp":
        _f32_close(O.get_state([g["all_pc"].astype(np.float32), g["all_gc"].astype(np.float32)], chain), g["all_state"])
    if key == "nobias":
        assert not any(k.startswith("0.") and k.endswith("bias") for k in _state(g, key))


def test_multilayer_perceptron_initial_weights_are_the_references(golden):
    from ratinabox_b200.contribs.NeuralNetworkNeurons import MultiLayerPerceptron
    g = golden("nnn.npz")
    torch.manual_seed(0)
    m = MultiLayerPerceptron(n_in=int(g["mlp_n_in"]), n_out=5, n_hidden=[20, 20])
    sd = m.state_dict()
    want = _state(g, "mlp")
    assert list(sd.keys()) == list(want.keys())
    for k, v in sd.items():
        assert v.dtype == torch.float32 and np.array_equal(v.numpy(), want[k]), k


def test_messages_and_defaults_are_the_references(golden):
    import sys
    from ratinabox_b200.contribs import MultiLayerPerceptron, NeuralNetworkNeurons
    M = sys.modules["ratinabox_b200.contribs.NeuralNetworkNeurons"]
    assert M.NeuralNetworkNeurons is NeuralNetworkNeurons and M.MultiLayerPerceptron is MultiLayerPerceptron
    g = golden("nnn.npz")
    assert json.loads(str(g["default_params_json"])) == NeuralNetworkNeurons.default_params
    assert M.DEFAULT_MLP_WARNING.format(n_in=int(g["mlp_n_in"]), n=5) == str(g["default_warning"])
    assert M.BOTH_ERROR == str(g["err_both"]) and M.NEITHER_ERROR == str(g["err_neither"])
    assert M.PROBE_ERROR.format(n_in=30) == str(g["err_probe"])


def test_fused_chains_and_their_limits():
    import torch.nn as nn
    from ratinabox_b200.contribs.NeuralNetworkNeurons import MultiLayerPerceptron, _linear_chain
    ok = [MultiLayerPerceptron(10, 3), nn.Sequential(nn.Linear(4, 5), nn.Sequential(nn.Tanh(), nn.Identity()), nn.Linear(5, 2)),
          nn.Sequential(nn.Linear(4, 256), nn.Sigmoid(), nn.Linear(256, 1000)), nn.Linear(3, 2),
          nn.Sequential(*[nn.Linear(4, 4) for _ in range(8)])]
    for m in ok:
        chain, reason = _linear_chain(m)
        assert chain is not None and reason is None, m
    bad = {"LayerNorm": nn.Sequential(nn.Linear(4, 5), nn.LayerNorm(5)),
           "width 257": nn.Sequential(nn.Linear(4, 257), nn.ReLU(), nn.Linear(257, 1)),
           "9 Linear": nn.Sequential(*[nn.Linear(4, 4) for _ in range(9)]),
           "after another activation": nn.Sequential(nn.Linear(4, 4), nn.ReLU(), nn.Tanh()),
           "before the first Linear": nn.Sequential(nn.ReLU(), nn.Linear(4, 4)),
           "float64": nn.Linear(4, 4).double()}
    for what, m in bad.items():
        chain, reason = _linear_chain(m)
        assert chain is None and what in reason, (what, reason)
    hooked = nn.Linear(4, 4)
    hooked.register_forward_hook(lambda *a: None)
    assert _linear_chain(hooked)[0] is None


def test_nnn_cells_layout_matches_the_header(tmp_path):
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "riab_b200.h")).read()
    assert re.search(r"RIAB_CELLS_NNN = 11\b", hdr) and _lib.CELLS_NNN == 11
    assert re.search(r"#define RIAB_NNN_MAX_LAYERS %d\b" % _lib.NNN_MAX_LAYERS, hdr)
    assert re.search(r"#define RIAB_NNN_MAX_HIDDEN %d\b" % _lib.NNN_MAX_HIDDEN, hdr)
    for name in ("riab_nnn_pack_floats", "riab_nnn_pack", "riab_nnn_rates"):
        assert name in hdr and name in _lib.SYMBOLS
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    c = tmp_path / "nnn.c"
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "riab_b200.h"\nint main(void) {\n'
                 '  printf("%zu %zu %zu %zu\\n", sizeof(riab_nnn_cells), offsetof(riab_nnn_cells, act),\n'
                 '         offsetof(riab_nnn_cells, packed_dev), offsetof(riab_nnn_cells, inputs));\n  return 0;\n}\n')
    exe = tmp_path / "nnn"
    subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    size, act, packed, inputs = map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    S = _lib.NnnCells
    assert (C.sizeof(S), S.act.offset, S.packed_dev.offset, S.inputs.offset) == (size, act, packed, inputs)


def test_pack_block_layout():
    """riab_nnn_pack: layer 1 as riab_ffl_pack blocks per input (W_hi + W_lo ~ float32(W)), then b_1 and W_l^T | b_l."""
    from ratinabox_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(0)
    n_ins, widths = [7, 40], [47, 20, 20, 3]
    Ws = [rs.normal(size=(widths[l + 1], widths[l])) for l in range(3)]
    bs = [rs.normal(size=widths[l + 1]) for l in range(3)]
    params = np.concatenate([np.concatenate([W.ravel(), b]) for W, b in zip(Ws, bs)])
    c = _lib.NnnCells()
    c.n_layers, c.n_inputs = 3, 2
    for l, w in enumerate(widths):
        c.widths[l] = w
    for l, a in enumerate(("relu", "tanh", "identity")):
        c.act[l] = _lib.NNN_ACTIVATIONS[a]
    for i, n in enumerate(n_ins):
        c.inputs[i].n_in = n
    host = np.zeros(lib.riab_nnn_pack_floats(C.byref(c)), dtype=np.float32)
    _lib.check(lib.riab_nnn_pack(params.ctypes.data_as(_lib.c_double_p), C.byref(c), host.ctypes.data_as(_lib.c_float_p)))
    assert c.n_cells == 3 and [c.inputs[i].k_pad for i in range(2)] == [32, 64]
    o, col = 0, 0
    for i, n in enumerate(n_ins):
        kp = c.inputs[i].k_pad
        hi = host[o: o + 24 * kp].reshape(24, kp)
        lo = host[o + 24 * kp: o + 48 * kp].reshape(24, kp)
        w32 = Ws[0][:, col: col + n].astype(np.float32)
        assert np.abs(hi[:20, :n].astype(np.float64) + lo[:20, :n] - w32).max() <= 2.0 ** -20 * np.abs(w32).max()
        assert not hi[20:].any() and not hi[:, n:].any()
        o, col = o + 48 * kp, col + n
    assert np.array_equal(host[o: o + 20], bs[0].astype(np.float32)) and not host[o + 20: o + 24].any()
    o += 24
    for l in (1, 2):
        ni, no, no8 = widths[l], widths[l + 1], (widths[l + 1] + 7) // 8 * 8
        Wt = host[o: o + ni * no8].reshape(ni, no8)
        assert np.array_equal(Wt[:, :no], Ws[l].T.astype(np.float32)) and not Wt[:, no:].any()
        o += ni * no8
        assert np.array_equal(host[o: o + no], bs[l].astype(np.float32))
        o += no8
    assert o == host.size
    c.widths[1] = 257                                       # a hidden width over the kernel's limit
    assert lib.riab_nnn_pack(params.ctypes.data_as(_lib.c_double_p), C.byref(c), host.ctypes.data_as(_lib.c_float_p)) != 0

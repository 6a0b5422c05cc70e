"""CPU checks of FeedForwardLayer (ratinabox/Neurons.py:2654-2847): the float64 oracle (oracle/riab_oracle_ffl.py)
against the live reference's fixture (tests/golden/ffl.npz, oracle/gen_ffl_golden.py), the host mirror's set-up,
the operand packing of riab_ffl_pack, and the resources of the compiled kernel.  No CUDA calls."""
import ctypes as C
import json
import os
import re
import types

import numpy as np
import pytest

import riab_oracle_ffl as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ACTS = {"linear": {}, "sigmoid": {"max_fr": 2.0, "min_fr": 0.5, "mid_x": 0.3, "width_x": 1.5},
        "relu": {"gain": 1.5, "threshold": 0.1}, "tanh": {"gain": 0.8, "threshold": 0.2},
        "retanh": {"gain": 1.3, "threshold": -0.1}, "softmax": {"gain": 1.2, "threshold": -0.3}}
LAYERS = {"Late": ("relu", [("PC", 1)]), "F1": ("sigmoid", [("PC", 0), ("GC", 0)]), "F2": ("tanh", [("F1", 0)]),
          "R": ("softmax", [("PC", 0), ("R", 1)])}     # (activation, [(input, lag)]): the reference's update order


def test_activations_match_the_reference(golden):
    g = golden("ffl.npz")
    for name, args in ACTS.items():
        for deriv in (False, True):
            got = F.activate(g["act_x"], name, deriv, dict(args, activation=name))
            want = g[f"act_{name}" + ("_deriv" if deriv else "")]
            assert np.array_equal(got, want), (name, deriv)


def test_oracle_reproduces_the_native_run_bit_for_bit(golden):
    """Every step's rates and primes of the four layers from their inputs' rates, with the reference's timing: an input
    registered before the layer gives this step's row, one registered at or after it (the self-recurrent input, and
    PlaceCells for the layer created before them) the previous step's, zeros before its first update."""
    g = golden("ffl.npz")
    T = g["run_PC"].shape[0]
    for name, (act, ins) in LAYERS.items():
        args = dict(ACTS[act], activation=act)
        for t in range(T):
            inputs = []
            for src, lag in ins:
                I = g[f"run_{src}"][t - lag] if t - lag >= 0 else np.zeros(g[f"run_{src}"].shape[1])
                inputs.append((g[f"{name}_w_{src}"], I))
            assert np.array_equal(F.ffl_get_state(inputs, g[f"{name}_biases"], act, args), g[f"run_{name}"][t]), (name, t)
            assert np.array_equal(F.ffl_get_state(inputs, g[f"{name}_biases"], act, args, deriv=True),
                                  g[f"run_{name}_prime"][t]), (name, t)


def test_oracle_reproduces_get_state_at_positions(golden):
    g = golden("ffl.npz")
    pc, gc = g["gs_PC"], g["gs_GC"]
    late = F.ffl_get_state([(g["Late_w_PC"], pc)], g["Late_biases"], "relu", ACTS["relu"])
    assert np.array_equal(late, g["gs_Late"])
    r_inner = F.ffl_get_state([(g["R_w_PC"], pc)], g["R_biases"], "softmax", ACTS["softmax"])      # recurrence cut
    r = F.ffl_get_state([(g["R_w_PC"], pc), (g["R_w_R"], r_inner)], g["R_biases"], "softmax", ACTS["softmax"])
    assert np.array_equal(r, g["gs_R"])
    assert g["gs_F1"].shape == (10, 384) and g["gs_F2"].shape == (6, 384)


def _stub(n, pop, agent):
    return types.SimpleNamespace(n=n, name=f"L{pop}", Agent=agent, _population_id=pop, _ring_min=1, inputs={})


def test_host_mirror_set_up_matches_the_reference(golden):
    """add_input's weight draw under the same np.random seed, default_params, the lag bookkeeping, and the refusal of
    bespoke activations -- without a GPU (the methods run on stand-ins)."""
    import ratinabox_b200 as rb
    g = golden("ffl.npz")
    ag = object()
    layer, src = _stub(int(g["draw_n"]), 3, ag), _stub(int(g["draw_n_in"]), 1, ag)
    np.random.seed(int(g["draw_seed"]))
    rb.FeedForwardLayer.add_input(layer, src, w_init_scale=float(g["draw_scale"]), tag=1)
    e = layer.inputs["L1"]
    assert np.array_equal(e["w"], g["draw_w"]) and np.array_equal(e["w_init"], g["draw_w"])
    assert set(dict.keys(e)) == {"layer", "w", "w_init", "I", "n", "recurrent", "tag"} and e["n"] == src.n
    assert src._ring_min == 1                              # registered before the layer: read in the same step
    rb.FeedForwardLayer.add_input(layer, layer)
    assert layer._ring_min == 2                            # self-recurrent: its previous row must survive
    with pytest.raises(ValueError):
        rb.FeedForwardLayer.add_input(layer, _stub(4, 0, object()))
    ref = json.loads(str(g["default_params_json"]))
    have = rb.FeedForwardLayer.default_params
    assert set(ref) == set(have)
    for k, v in ref.items():
        assert (have[k] == v) or (have[k] is None and v is None), k
    for af in (lambda x, deriv=False: x, {"activation": "relu", "function": lambda x, deriv=False: x}):
        with pytest.raises(NotImplementedError):
            rb.FeedForwardLayer._activation(types.SimpleNamespace(activation_function=af))
    act, prm = rb.FeedForwardLayer._activation(types.SimpleNamespace(activation_function=dict(ACTS["sigmoid"], activation="sigmoid")))
    assert act == 1 and np.isclose(prm[3], np.log(19) / 0.75)


@pytest.mark.parametrize("n,n_in", [(1, 1), (10, 300), (257, 33)])
def test_ffl_pack_splits_exactly(n, n_in):
    from ratinabox_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(n + n_in)
    w = rs.normal(0, 1, (n, n_in)) * 10.0 ** rs.uniform(-3, 3, (n, n_in))
    meta = _lib.FflInput()
    out = np.full(lib.riab_ffl_pack_floats(n, n_in), np.nan, dtype=np.float32)
    assert lib.riab_ffl_pack(np.ascontiguousarray(w).ctypes.data_as(_lib.c_double_p), n, n_in, C.byref(meta),
                             out.ctypes.data_as(_lib.c_float_p)) == 0
    npad, kpad = (n + 7) // 8 * 8, (n_in + 31) // 32 * 32
    assert (meta.n_in, meta.k_pad) == (n_in, kpad) and out.size == 2 * npad * kpad
    hi, lo = out[: npad * kpad].reshape(npad, kpad), out[npad * kpad:].reshape(npad, kpad)
    for part in (hi, lo):
        assert np.all(part.view(np.uint32) & 0x1FFF == 0)          # tf32: the 13 low mantissa bits are clear
    assert np.all(hi[n:] == 0) and np.all(hi[:, n_in:] == 0) and np.all(lo[n:] == 0) and np.all(lo[:, n_in:] == 0)
    w32 = w.astype(np.float32).astype(np.float64)
    s = hi[:n, :n_in].astype(np.float64) + lo[:n, :n_in].astype(np.float64)
    assert np.all(np.abs(s - w32) <= 2.0 ** -22 * np.abs(w32))
    assert lib.riab_ffl_pack(None, n, n_in, C.byref(meta), out.ctypes.data_as(_lib.c_float_p)) < 0


def test_ffl_kernel_resources():
    """The FeedForwardLayer kernel (one instantiation per N tile: 8, 32, 64) has no local-memory spills, fits its 288
    threads in the register file at one CTA per SM, and keeps only its mbarriers in static shared memory (the 4-stage
    operand ring is dynamic: 4 x (16 KB + 2 x BN x 128 B) + 1 KB, at most 132 KB)."""
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([tool, "--dump-resource-usage", _lib.lib_path()], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*5k_fflILi(\d+)E\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", txt)
    assert sorted(int(f[1]) for f in found) == [8, 32, 64], found
    for name, bn, reg, stack, shared, local in found:
        assert int(stack) == 0 and int(local) == 0, (bn, stack, local)
        assert int(reg) * 288 <= 65536, (bn, reg)
        assert int(shared) <= 1024 + 256, (bn, shared)   # + the 1 KB the driver reserves per CTA


def test_ffl_structs_have_the_headers_layout(tmp_path):
    """ctypes mirrors of riab_ffl_input / riab_ffl_cells against the C compiler's layout of include/riab_b200.h."""
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "riab_b200.h"', "int main(void) {",
           '  printf("%zu %zu %zu %zu %d\\n", sizeof(riab_ffl_input), offsetof(riab_ffl_input, lag), sizeof(riab_ffl_cells),'
           ' offsetof(riab_ffl_cells, inputs), RIAB_CELLS_FFL);', "  return 0;", "}"]
    c = tmp_path / "ffl.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "ffl"
    subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(_lib.FflInput), _lib.FflInput.lag.offset, C.sizeof(_lib.FflCells), _lib.FflCells.inputs.offset,
                   _lib.CELLS_FFL]

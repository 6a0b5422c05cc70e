"""The per-agent TD oracle (oracle/riab_oracle_td_pa.py) against K live-reference ValueNeuron runs along one shared
trajectory (tests/golden/td_pa.npz, oracle/gen_td_pa_golden.py): as one batch of K agents with per-agent weights it
replays every run bit for bit.  Also: with one agent it is riab_oracle_td, the riab_td_cells layout with its
per_agent_weights field, the new entry point's export and its argument checks, none of which needs a device."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import riab_oracle_td as T        # noqa: E402
import riab_oracle_td_pa as P     # noqa: E402

DT = 0.05


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "td_pa.npz"))


def test_one_batch_replays_every_reference_run_bit_for_bit(g):
    K, steps = g["fr"].shape[:2]
    assert K == 3 and steps == 200
    tau_e = float(g["tau_e"])
    W = [g["W_PC"][:, 0].copy(), g["W_GC"][:, 0].copy()]                 # (K, 1, n_in): each run's own weights
    assert not np.array_equal(W[0][0], W[0][1])
    fr_last = np.zeros((K, 1))
    e = [np.zeros((K, 20)), np.zeros((K, 12))]
    for t in range(steps):
        I = [g["PC"][:, t], g["GC"][:, t]]
        assert np.array_equal(I[0][0], I[0][1])                          # one trajectory, shared inputs
        fr = np.stack([P.td_rates_pa(W, I, g["biases"][k], "relu")[k] for k in range(K)])
        prime = np.stack([P.td_rates_pa(W, I, g["biases"][k], "relu", deriv=True)[k] for k in range(K)])
        np.testing.assert_array_equal(fr, g["fr"][:, t])
        np.testing.assert_array_equal(prime, g["prime"][:, t])
        deriv = T.td_derivative(fr, fr_last, DT)
        e = [T.td_trace(e[l], I[l], DT, tau_e) for l in range(2)]
        np.testing.assert_array_equal(e[0], g["e_PC"][:, t])
        np.testing.assert_array_equal(e[1], g["e_GC"][:, t])
        td = P.td_learn_pa(W, e, g["reward"][:, t], fr, deriv, prime, DT, 1.0, 0.05, 0.01)
        np.testing.assert_array_equal(td, g["td"][:, t])
        fr_last = fr
        if (t + 1) % 10 == 0:
            np.testing.assert_array_equal(W[0], g["W_PC"][:, (t + 1) // 10])
            np.testing.assert_array_equal(W[1], g["W_GC"][:, (t + 1) // 10])
    # the runs learned different things
    assert not np.allclose(W[0][0] - g["W_PC"][0, 0], W[0][1] - g["W_PC"][1, 0])


def test_one_agent_is_the_shared_oracle():
    rs = np.random.RandomState(3)
    n, n_in = 3, 7
    W0 = rs.normal(size=(n, n_in))
    fr, deriv, prime = rs.rand(1, n), rs.normal(size=(1, n)), rs.rand(1, n)
    e, r = rs.rand(1, n_in), rs.rand(n)
    Ws = W0.copy()
    td_s = T.td_learn([Ws], [e], r, fr, deriv, prime, DT, 2.0, 0.1, 0.01)
    Wp = W0[None].copy()
    td_p = P.td_learn_pa([Wp], [e], r, fr, deriv, prime, DT, 2.0, 0.1, 0.01)
    np.testing.assert_array_equal(Wp[0], Ws)
    np.testing.assert_array_equal(td_p, td_s)


def test_agents_learn_independently_and_apply_matches_learn():
    rs = np.random.RandomState(4)
    A, n, n_in = 5, 2, 6
    W0 = rs.normal(size=(A, n, n_in))
    fr, deriv, prime = rs.rand(A, n), rs.normal(size=(A, n)), rs.rand(A, n)
    e, r = rs.rand(A, n_in), rs.rand(A, n)
    W = W0.copy()
    td = P.td_learn_pa([W], [e], r, fr, deriv, prime, DT, 2.0, 0.1, 0.01)
    for a in range(A):
        Wa = W0[a].copy()
        T.td_learn([Wa], [e[a]], r[a], fr[a], deriv[a], prime[a], DT, 2.0, 0.1, 0.01)
        np.testing.assert_array_equal(W[a], Wa)
    W2 = W0.copy()
    P.td_apply_pa([W2], [e], td, prime, DT, 0.1, 0.01)
    np.testing.assert_array_equal(W2, W)


def test_td_cells_per_agent_field_has_the_headers_layout(tmp_path):
    from ratinabox_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = ["#include <stdio.h>", "#include <stddef.h>", '#include "riab_b200.h"', "int main(void) {",
           '  printf("%zu %zu %zu\\n", sizeof(riab_td_cells), offsetof(riab_td_cells, per_agent_weights),'
           ' offsetof(riab_td_cells, reserved));',
           "  return 0;", "}"]
    c = tmp_path / "td_pa_layout.c"
    c.write_text("\n".join(src) + "\n")
    exe = tmp_path / "td_pa_layout"
    subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    size, off, off_old = (int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True,
                                                         text=True).stdout.split())
    assert size == C.sizeof(_lib.TdCells)
    assert off == off_old == _lib.TdCells.per_agent_weights.offset == _lib.TdCells.reserved.offset
    t = _lib.TdCells()
    t.per_agent_weights = 1
    assert t.reserved == 1


def test_rates_pa_is_exported_and_validates_without_a_device():
    from ratinabox_b200 import _lib
    lib = _lib.load()
    assert hasattr(lib, "riab_td_rates_pa") and "riab_td_rates_pa" in _lib.SYMBOLS
    assert lib.riab_td_rates_pa(None, 1, None, None, None, 4, None) == -1
    assert b"bad argument" in lib.riab_last_error()
    c = _lib.TdCells()
    c.ffl.n_cells = 1
    c.ffl.bias_dev = 16
    assert lib.riab_td_rates_pa(C.byref(c), 1, None, None, C.c_void_p(16), 4, None) == -1
    assert b"shared" in lib.riab_last_error()
    c.per_agent_weights = 2
    assert lib.riab_td_reset(C.byref(c), 1, None, None) == -1
    # per-agent learning needs no scratch
    c.per_agent_weights = 1
    c.ffl.n_inputs = 1
    c.ffl.inputs[0].n_in = 1024
    assert lib.riab_td_scratch_bytes(C.byref(c), 65536) == 0
    c.per_agent_weights = 0
    assert lib.riab_td_scratch_bytes(C.byref(c), 65536) > 0


def test_per_agent_param_is_collected_beside_the_reference_defaults():
    """``per_agent_weights`` defaults to False through the engine's base class; ValueNeuron.default_params stay the
    reference's."""
    from ratinabox_b200.contribs.ValueNeuron import ValueNeuron
    collected = {}
    for cls in reversed(ValueNeuron.__mro__):
        collected.update(getattr(cls, "default_params", {}))
    assert collected["per_agent_weights"] is False
    assert "per_agent_weights" not in ValueNeuron.default_params

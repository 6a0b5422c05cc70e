"""The float64 TD oracle (oracle/riab_oracle_td.py) against the live reference's ValueNeuron / SuccessorFeatures
(tests/golden/td.npz, oracle/gen_td_golden.py): replayed on the recorded input rates, it reproduces every recorded
quantity bit for bit.  Also the mirror's default params and error texts, the riab_td_cells layout, and the argument
validation of the riab_td_* entry points, none of which needs a device."""
import ctypes as C
import io
import json
import os
import contextlib
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import riab_oracle_ffl as F  # noqa: E402
import riab_oracle_td as T   # noqa: E402

DT = 0.05


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "td.npz"))


def _replay(g, p, inputs, W, biases, act, act_args, tau, tau_e, eta, L2, reward_of, self_name=None, reset_after=None,
            checkpoints=None):
    """Replay a recorded run: rates from the FFL oracle with the oracle's own weights, then the derivative, the
    traces and the learning step, each compared exactly with the recording."""
    n = g[f"{p}_fr"].shape[1]
    fr_last = np.zeros(n)
    e = {k: np.zeros(W[k].shape[1]) for k in W}
    steps = g[f"{p}_fr"].shape[0]
    for t in range(steps):
        ins = [(W[k], fr_last if k == self_name else g[f"{p}_{k}"][t]) for k in inputs]
        fr = F.ffl_get_state(ins, biases, act, act_args)
        np.testing.assert_array_equal(fr, g[f"{p}_fr"][t])
        np.testing.assert_array_equal(F.ffl_get_state(ins, biases, act, act_args, deriv=True), g[f"{p}_prime"][t])
        deriv = T.td_derivative(fr, fr_last, DT)
        np.testing.assert_array_equal(deriv, g[f"{p}_deriv"][t])
        for k in inputs:
            e[k] = T.td_trace(e[k], fr if k == self_name else g[f"{p}_{k}"][t], DT, tau_e)
            np.testing.assert_array_equal(e[k], g[f"{p}_e_{k}"][t])
        td = T.td_learn([W[k] for k in inputs], [e[k] for k in inputs], reward_of(t), fr, deriv, g[f"{p}_prime"][t],
                        DT, tau, eta, L2)
        np.testing.assert_array_equal(td[0], g[f"{p}_td"][t])
        fr_last = fr
        if checkpoints is not None and (t + 1) % 10 == 0:
            for k in inputs:
                np.testing.assert_array_equal(W[k], g[f"{p}_W_{k}"][(t + 1) // 10])
        if reset_after is not None and t == reset_after:
            fr_last = np.zeros(n)
            e = {k: np.zeros_like(v) for k, v in e.items()}
    return W


def test_value_neuron_run_replays_bit_for_bit(g):
    W = {"PC": g["v_W_PC"][0].copy(), "GC": g["v_W_GC"][0].copy()}
    assert float(g["v_tau_e"]) == 0.25
    _replay(g, "v", ["PC", "GC"], W, g["v_biases"], "relu", {}, 1.0, 0.25, 0.05, 0.01,
            lambda t: g["v_reward"][t], checkpoints=True)


def test_recurrent_sigmoid_with_reset_replays_bit_for_bit(g):
    W = {"PC": g["s_W0_PC"].copy(), "VN": g["s_W0_VN"].copy()}
    act = {"max_fr": 2.0, "min_fr": 0.5, "mid_x": 0.3, "width_x": 1.5}
    _replay(g, "s", ["PC", "VN"], W, np.zeros(2), "sigmoid", act, 0.8, 0.3, 0.2, 0.05, lambda t: g["s_reward"][t],
            self_name="VN", reset_after=29)
    np.testing.assert_array_equal(W["PC"], g["s_W_PC"])
    np.testing.assert_array_equal(W["VN"], g["s_W_VN"])


def test_successor_features_replay_bit_for_bit(g):
    W = {"Feat": g["f_W0_Feat"].copy(), "GC": g["f_W0_GC"].copy()}
    assert int(g["f_n"]) == 6
    _replay(g, "f", ["Feat", "GC"], W, np.zeros(6), "relu", {}, 2, 0.2, 0.3, 0.001, lambda t: g["f_Feat"][t])
    np.testing.assert_array_equal(W["Feat"], g["f_W_Feat"])
    np.testing.assert_array_equal(W["GC"], g["f_W_GC"])


def test_batched_learning_is_the_mean_of_single_agent_updates():
    rs = np.random.RandomState(0)
    A, n, n_in = 5, 3, 7
    W0 = rs.normal(size=(n, n_in))
    fr, deriv, prime = rs.rand(A, n), rs.normal(size=(A, n)), rs.rand(A, n)
    e, r = rs.rand(A, n_in), rs.rand(A, n)
    Wb = W0.copy()
    T.td_learn([Wb], [e], r, fr, deriv, prime, DT, 2.0, 0.1, 0.01)
    dws = []
    for a in range(A):
        Wa = W0.copy()
        T.td_learn([Wa], [e[a]], r[a], fr[a], deriv[a], prime[a], DT, 2.0, 0.1, 0.01)
        dws.append(Wa - W0)
    np.testing.assert_allclose(Wb - W0, np.mean(dws, axis=0), rtol=1e-12, atol=1e-15)


def test_mirror_default_params_and_error_texts_match_the_reference(g):
    from ratinabox_b200.contribs import SuccessorFeatures, ValueNeuron
    from ratinabox_b200.contribs.ValueNeuron import ValueNeuron as VN2
    from ratinabox_b200.contribs.SuccessorFeatures import SuccessorFeatures as SF2
    assert VN2 is ValueNeuron and SF2 is SuccessorFeatures
    want = json.loads(str(g["default_params_json"]))
    assert {k: v for k, v in ValueNeuron.default_params.items()} == want["ValueNeuron"]
    assert {k: v for k, v in SuccessorFeatures.default_params.items()} == want["SuccessorFeatures"]
    errs = json.loads(str(g["errors_json"]))
    with pytest.raises(Exception) as ei:
        SuccessorFeatures(None, {"input_layers": []})
    assert type(ei.value).__name__ == errs["sf_no_features"][0] and str(ei.value) == errs["sf_no_features"][1]


class _Stub:
    """Just enough of a ValueNeuron for its host-side checks (no device)."""
    n = 2
    tau_e = 0.0


def test_host_side_errors_match_the_reference_without_a_device(g):
    from ratinabox_b200.contribs.ValueNeuron import ValueNeuron, _TdInput
    errs = json.loads(str(g["errors_json"]))
    s = _Stub()
    s.inputs = {}
    with pytest.raises(AttributeError) as ei:
        ValueNeuron._check_update(s)
    assert str(ei.value) == errs["tau_e_zero"][1]
    s.tau_e = 0.5
    s.inputs = {"Late": _TdInput(None, "Late", {"n": 3})}
    with pytest.raises(KeyError) as ei:
        ValueNeuron._check_update(s)
    assert str(ei.value) == errs["late_input"][1]


def test_td_cells_have_the_headers_layout(tmp_path):
    """The same method as the layout test of the other structs: a C program compiled against the header prints sizeof /
    offsetof, compared with the ctypes mirror."""
    from ratinabox_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    fields = ["ffl", "fr_prev_dev", "deriv_dev", "td_error_dev", "ld", "trace_dev", "trace_ld", "w_master_dev", "dt",
              "tau", "tau_e", "eta", "L2", "self_input", "reserved"]
    src = ["#include <stdio.h>", "#include <stddef.h>", '#include "riab_b200.h"', "int main(void) {",
           '  printf("%zu\\n", sizeof(riab_td_cells));']
    src += [f'  printf("%zu\\n", offsetof(riab_td_cells, {f}));' for f in fields]
    src += ['  printf("%d %d %d\\n", (int)RIAB_CELLS_TD, (int)RIAB_TD_REWARD_SHARED, (int)RIAB_TD_REWARD_ROWS);',
            "  return 0;", "}"]
    c = tmp_path / "td_layout.c"
    c.write_text("\n".join(src) + "\n")
    exe = tmp_path / "td_layout"
    subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    assert int(got[0]) == C.sizeof(_lib.TdCells)
    for f, off in zip(fields, got[1:]):
        assert int(off) == getattr(_lib.TdCells, f).offset, f
    assert got[len(fields) + 1].split() == [str(_lib.CELLS_TD), str(_lib.TD_REWARD_SHARED), str(_lib.TD_REWARD_ROWS)]


def test_td_entry_points_validate_their_arguments_without_a_device():
    """Every refusal below happens before any CUDA call."""
    from ratinabox_b200 import _lib
    lib = _lib.load()
    assert lib.riab_td_learn(None, 1, None, 0, None, None, None) == -1
    assert b"bad argument" in lib.riab_last_error()
    assert lib.riab_td_reset(None, 1, None, None) == -1
    assert lib.riab_td_scratch_bytes(None, 1) == -1
    c = _lib.TdCells()
    c.ffl.n_cells = 1
    assert lib.riab_td_learn(C.byref(c), 1, C.c_void_p(16), 7, C.c_void_p(16), C.c_void_p(16), None) == -1
    assert lib.riab_td_learn(C.byref(c), 1, C.c_void_p(16), 0, C.c_void_p(16), C.c_void_p(8), None) == -1
    assert b"16-byte" in lib.riab_last_error()
    # no TD state
    assert lib.riab_td_learn(C.byref(c), 1, C.c_void_p(16), 0, C.c_void_p(16), C.c_void_p(16), None) == -1
    assert b"fr_prev" in lib.riab_last_error()
    c.fr_prev_dev = c.deriv_dev = c.td_error_dev = 16
    c.ld = 4
    c.dt, c.tau_e = 0.05, 0.0
    assert lib.riab_td_reset(C.byref(c), 1, None, None) == -1
    assert b"tau_e" in lib.riab_last_error()
    c.tau_e = 0.5
    c.ffl.n_inputs = 1
    c.ffl.inputs[0].n_in = 5
    assert lib.riab_td_reset(C.byref(c), 1, None, None) == -1
    assert b"td input 0" in lib.riab_last_error()
    c.ld = 6
    assert lib.riab_td_reset(C.byref(c), 1, None, None) == -1
    assert b"ld" in lib.riab_last_error()
    c.ld, c.self_input = 4, 3
    assert lib.riab_td_reset(C.byref(c), 1, None, None) == -1
    assert b"self_input" in lib.riab_last_error()
    c.ffl.n_inputs = 0
    c.self_input = -1
    assert lib.riab_td_scratch_bytes(C.byref(c), 1000) > 0

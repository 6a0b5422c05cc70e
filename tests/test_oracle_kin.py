"""CPU checks of the kinematic cells (HeadDirectionCells, VelocityCells, SpeedCell): the float64 oracle
(oracle/riab_oracle_kin.py) against the live reference's fixture (tests/golden/kin.npz, oracle/gen_kin_golden.py), the
host mirror's default_params, riab_kin_pack against a NumPy packing, the riab_kin_cells layout and the resources of the
k_step<KinPolicy> instantiations.  No CUDA calls."""
import ctypes as C
import json
import os
import re
import warnings

import numpy as np
import pytest

import riab_oracle_kin as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _eq(a, b):
    """Bit equality, or within 1e-12 relative where libm's exp / arctan2 may differ between machines."""
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    assert a.shape == b.shape, (a.shape, b.shape)
    if np.array_equal(a, b, equal_nan=True):
        return
    assert np.array_equal(np.isnan(a), np.isnan(b))
    ok = ~np.isnan(a)
    assert np.all(np.abs(a[ok] - b[ok]) <= 1e-12 * np.maximum(1.0, np.abs(b[ok]))), float(np.abs(a[ok] - b[ok]).max())


def test_oracle_reproduces_the_defaults_and_the_native_run(golden):
    g = golden("kin.npz")
    pref, tun = K.default_tuning(10, 45)
    assert np.array_equal(pref, g["hdc_preferred_angles"]) and np.array_equal(tun, g["hdc_angular_tunings"])
    assert np.array_equal(pref, g["vel_preferred_angles"]) and np.array_equal(tun, g["vel_angular_tunings"])
    oss = float(g["vel_one_sigma_speed"])
    assert oss == 0.08 + 0.08
    for t in range(g["run_hd"].shape[0]):
        hd, vel = g["run_hd"][t], g["run_vel"][t]
        _eq(K.head_direction_rates(hd, pref, tun), g["run_hdc"][t])
        _eq(K.head_direction_rates(vel, pref, tun, use_velocity=True), g["run_hdc_usevel"][t])
        _eq(K.velocity_rates(vel, vel, oss, pref, tun), g["run_velc"][t])
    _eq(K.head_direction_rates(g["run_hd"][-1], pref, tun)[:, 0], g["run_hdc_firingrate"])


def test_oracle_reproduces_the_kwargs(golden):
    g = golden("kin.npz")
    pref, tun = K.default_tuning(10, 45)
    hd, P = g["kw_hd"], g["kw_P"]
    _eq(K.head_direction_rates(hd, pref, tun), g["kw_head_direction"])
    _eq(K.head_direction_rates(hd, pref, tun, n_pos=10000), g["kw_head_direction_all"])
    _eq(K.head_direction_rates(hd, pref, tun, n_pos=len(P)), g["kw_head_direction_pos"])
    _eq(K.head_direction_rates(hd, pref, tun), g["kw_vel"])
    assert list(g["kw_vel_warnings"]) == ["'vel' kwarg deprecated in favour of 'head_direction'"]
    _eq(K.head_direction_rates([1, 0], pref, tun), g["kw_none"])
    assert str(g["kw_none_printed"]) == ("HeadDirection cells need a head direction but you didn't pass one. Taking [1,0] as "
                                         "defaultRecommended to pass one in the 'head_direction' argument of get_state()\n")
    _eq(K.head_direction_rates([1, 0], pref, tun, use_velocity=True), g["kw_none_usevel"])
    assert str(g["kw_none_usevel_printed"]) == ("HeadDirection cells need a velocity but you didn't pass one. Taking [1,0] as "
                                                "defaultRecommended to pass one in the 'velocity' argument of get_state()\n")
    _eq(K.head_direction_rates(hd, pref, tun, use_velocity=True), g["kw_velocity_usevel"])
    av = g["kw_agent_velocity"]
    _eq(K.velocity_rates(hd, av, 0.16, pref, tun), g["kw_velc_velocity"])
    _eq(K.velocity_rates(hd, av, 0.16, pref, tun, n_pos=len(P)), g["kw_velc_velocity_pos"])


@pytest.mark.parametrize("case", ["lo", "inv"])
def test_oracle_reproduces_the_firing_rate_ranges(golden, case):
    g = golden("kin.npz")
    prm = json.loads(str(g[f"fr_{case}_params"]))
    lo, hi = prm["min_fr"], prm["max_fr"]
    pref, tun = K.default_tuning(13, 30)
    hd, av, mv, vel = g["fr_agent_hd"], g["fr_agent_vel"], g["fr_agent_mvel"], g["fr_vel"]
    _eq(K.velocity_rates(av, av, 0.16, pref, tun, lo, hi), g[f"fr_{case}_velc"])
    _eq(K.velocity_rates(vel, av, 0.16, pref, tun, lo, hi), g[f"fr_{case}_velc_kw"])
    _eq(K.head_direction_rates(hd, pref, tun, lo, hi), g[f"fr_{case}_hdc"])
    _eq(K.speed_rate(mv, 0.16, lo, hi), g[f"fr_{case}_speed_agent"])
    _eq(K.speed_rate(vel, 0.16, lo, hi), g[f"fr_{case}_speed_kw"])


def test_oracle_reproduces_the_narrow_spread_and_the_zero_velocity(golden):
    g = golden("kin.npz")
    pref, tun = K.default_tuning(36, float(g["narrow_deg"]))
    assert np.all(1 / tun ** 2 <= 700 * (1 + 1e-12))
    cols = [K.head_direction_rates([np.cos(t), np.sin(t)], pref, tun)[:, 0] for t in g["narrow_theta"]]
    _eq(np.stack(cols, axis=1), g["narrow"])
    assert np.all(np.isfinite(g["narrow"])) and g["narrow"].max() > 0.99
    pref, tun = K.default_tuning(10, 45)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _eq(K.velocity_rates([0.0, 0.0], [0.0, 0.0], 0.16, pref, tun), g["zero_velc"])
        _eq(K.head_direction_rates([0.0, 0.0], pref, tun, use_velocity=True), g["zero_hdc_usevel"])
    assert np.all(np.isnan(g["zero_velc"])) and np.all(np.isnan(g["zero_hdc_usevel"]))


def test_speed_cell_quirk_is_on_record(golden):
    """The reference sizes a SpeedCell's noise for its default n = 10 before it sets n = 1: its firing rate and history
    rows are 10 wide (one value broadcast).  A {"n": 1} population is one wide, like the mirror's SpeedCell."""
    g = golden("kin.npz")
    assert int(g["speed_default_n"]) == 1 and int(g["speed_default_history_width"]) == 10
    s10, s1, mv = g["speed_run_s10"], g["speed_run_s1"], g["speed_run_mvel"]
    assert s10.shape == (5, 10) and s1.shape == (5, 1)
    for t in range(5):
        want = K.speed_rate(mv[t], float(g["speed_one_sigma_speed"]))
        _eq(s1[t], want)
        _eq(s10[t], np.repeat(want, 10))
    assert list(g["speed_n4_warnings"]) == ["Ignoring 'n' parameter value (4) that was passed for SpeedCell. Only 1 speed "
                                            "cell is needed."]


def test_oracle_reproduces_the_head_direction_average(golden):
    g = golden("kin.npz")
    pref, tun = K.default_tuning(8, 30)
    for key, res in (("avg_hdc_all", 10), ("avg_hdc_all_res30", 30)):
        n_angles = int(360 / res)
        fr = np.zeros((8, 10000, n_angles))
        for i, a in enumerate(np.linspace(0, 2 * np.pi, n_angles)):
            fr[:, :, i] = K.head_direction_rates(np.array([np.cos(a), np.sin(a)]), pref, tun, 0.1, 1.7, n_pos=10000)
        _eq(np.mean(fr, axis=2), g[key])
    # at the agent the head_direction kwarg is ignored: the average is the agent's own rates
    _eq(K.head_direction_rates(g["avg_agent_hd"], pref, tun, 0.1, 1.7), g["avg_hdc_agent"])


def test_mirror_default_params_match_the_reference(golden):
    import ratinabox_b200 as rb
    ref = json.loads(str(golden("kin.npz")["default_params_json"]))
    for name, want in ref.items():
        have = {}
        for c in reversed(getattr(rb, name).__mro__):
            have.update(getattr(c, "default_params", {}))
        for k, v in want.items():
            assert k in have and have[k] == v, (name, k)
        extra = set(have) - set(want) - {"color"}
        assert extra <= {"save_spikes", "history_bytes_limit", "noise_std", "noise_coherence_time", "save_history", "n"} | \
            set(ref["HeadDirectionCells"]), (name, sorted(extra))


def test_kin_pack_matches_numpy():
    from ratinabox_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(2)
    n = 37
    pref, tun = rs.uniform(0, 2 * np.pi, n), rs.uniform(0.04, 1.5, n)
    meta = _lib.KinCells()
    out = np.zeros(lib.riab_kin_pack_floats(n), dtype=np.float32)
    f = lambda a: a.ctypes.data_as(_lib.c_double_p)
    assert lib.riab_kin_pack(f(pref), f(tun), n, _lib.KIN_VELOCITY, 0, 0.5, 2.0, 0.16, C.byref(meta),
                             out.ctypes.data_as(_lib.c_float_p)) == 0
    npad = meta.n_pad
    assert npad == 128 and len(out) == 3 * npad
    assert (meta.n_cells, meta.variant, meta.use_velocity, meta.min_fr, meta.max_fr) == (n, _lib.KIN_VELOCITY, 1, 0.5, 2.0)
    assert meta.inv_one_sigma_speed == 1 / 0.16
    want = np.zeros(3 * npad, dtype=np.float32)
    want[:npad] = 1.0
    want[:n] = np.cos(0.5 * pref).astype(np.float32)
    want[npad:npad + n] = np.sin(0.5 * pref).astype(np.float32)
    want[2 * npad:2 * npad + n] = np.sqrt(2.0 * (1 / tun ** 2) * np.log2(np.e)).astype(np.float32)
    assert np.array_equal(out[:2 * npad], want[:2 * npad])
    assert np.all(np.abs(out[2 * npad:] - want[2 * npad:]) <= np.spacing(want[2 * npad:]))
    # a speed cell packs no tuning: every cell is a pad (1, 0, 0)
    s = np.zeros(lib.riab_kin_pack_floats(1), dtype=np.float32)
    assert lib.riab_kin_pack(None, None, 1, _lib.KIN_SPEED, 0, 0.0, 1.0, 0.16, C.byref(meta), s.ctypes.data_as(_lib.c_float_p)) == 0
    assert np.array_equal(s, np.concatenate([np.ones(128), np.zeros(256)]).astype(np.float32))
    # bad arguments are refused with a message
    assert lib.riab_kin_pack(None, f(tun), n, _lib.KIN_HEAD_DIRECTION, 0, 0.0, 1.0, 1.0, C.byref(meta),
                             out.ctypes.data_as(_lib.c_float_p)) < 0
    assert b"riab_kin_pack" in lib.riab_last_error()
    assert lib.riab_kin_pack(f(pref), f(tun), n, 7, 0, 0.0, 1.0, 1.0, C.byref(meta), out.ctypes.data_as(_lib.c_float_p)) < 0


def test_kin_cells_struct_has_the_headers_layout(tmp_path):
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    fields = [f[0] for f in _lib.KinCells._fields_]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "riab_b200.h"', "int main(void) {",
           '  printf("%zu\\n", sizeof(riab_kin_cells));']
    src += [f'  printf("%zu\\n", offsetof(riab_kin_cells, {f}));' for f in fields]
    src += [f'  printf("%d %d %d %d\\n", RIAB_CELLS_KIN, RIAB_KIN_HEAD_DIRECTION, RIAB_KIN_VELOCITY, RIAB_KIN_SPEED);',
            "  return 0;", "}"]
    c = tmp_path / "kin.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "kin"
    subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    assert int(lines[0]) == C.sizeof(_lib.KinCells)
    for f, off in zip(fields, lines[1:]):
        assert getattr(_lib.KinCells, f).offset == int(off), f
    assert lines[1 + len(fields)].split() == [str(x) for x in (_lib.CELLS_KIN, _lib.KIN_HEAD_DIRECTION, _lib.KIN_VELOCITY,
                                                               _lib.KIN_SPEED)]


def test_kin_step_kernels_are_built_with_the_launch_registers():
    """The k_step<KinPolicy, MODE 0/1/2> instantiations exist, with their configuration's launch registers (the test in
    test_cabi_cpu.py holds every k_step to that) and no local memory in the consumers' static shared-memory budget."""
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([tool, "--dump-resource-usage", _lib.lib_path()], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*6k_stepIN\S*9KinPolicyELi(\d)E\S*7StepCfgILi(\d+)E\S*):\s*\n\s*REG:(\d+) STACK:\d+ "
                       r"SHARED:(\d+)", txt)
    modes = {m for _, m, _, _, _ in found}
    assert modes == {"0", "1", "2"}, modes
    want = {"4": 96, "8": 80, "12": 80}
    for name, mode, cfg, reg, shared in found:
        assert int(reg) == want[cfg] and int(shared) <= 48 * 1024, (name[:100], reg, shared)

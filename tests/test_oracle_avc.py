"""CPU checks of AgentVectorCells / FieldOfViewAVCs: the float64 oracle (oracle/riab_oracle_avc.py) against the live
reference's fixture (tests/golden/avc.npz, oracle/gen_avc_golden.py), the host mirror's default_params, riab_avc_pack
against a NumPy packing, the riab_avc_cells layout and the k_step<AvcPolicy> resources.  No CUDA calls."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

import riab_oracle as O
import riab_oracle_avc as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
POPS = ("allo", "eucl", "fov")


def _tuning(g, k):
    return tuple(g[f"{k}_tuning"])


def _state(g, k, env, partner, pos, rng, hd=None):
    lo, hi = g[f"{k}_fr_range"]
    return V.avc_get_state(env, partner, _tuning(g, k), pos, rng, str(g[f"{k}_geom"]), head_direction=hd, min_fr=lo, max_fr=hi)


def test_oracle_reproduces_the_two_agent_native_run(golden):
    """Two Agents in ovc.npz's box, ``Ag1.update(); Ag2.update()`` then AVC populations both ways, replayed on the global
    RNG (motion, line-of-sight jitter and spike draws in the reference's order): every row bit for bit."""
    g = golden("avc.npz")
    env = O.OracleEnvironment(walls=WALLS)
    ag1 = O.OracleAgent(env, g["pos0_1"], g["vel0_1"], {"dt": 0.02})
    ag2 = O.OracleAgent(env, g["pos0_2"], g["vel0_2"], {"dt": 0.02, "speed_mean": 0.15})
    rng = O.GlobalRNG()

    def pop(k, me, other):
        ego = str(g[f"{k}_frame"]) == "egocentric"
        return O.OracleNeurons(me, len(g[f"{k}_tuning"][0]), lambda p, r: _state(
            g, k, env, other.pos, p, r, me.head_direction if ego else None))

    pops = {}
    for tag, (me, other) in (("1", (ag1, ag2)), ("2", (ag2, ag1))):
        for k in POPS:
            pops[k + tag] = pop(k + tag, me, other)
    np.random.set_state(("MT19937", g["rng_keys"], int(g["rng_pos"]), int(g["rng_has_gauss"]), float(g["rng_cached"])))
    for _ in range(200):
        ag1.update(rng)
        ag2.update(rng)
        for P in pops.values():
            P.update(rng)
    assert np.array_equal(np.array(ag1.history["pos"]), g["pos_1"])
    assert np.array_equal(np.array(ag2.history["pos"]), g["pos_2"])
    for k, P in pops.items():
        assert np.array_equal(np.array(P.history["firingrate"]), g[f"{k}_fr"]), k
        assert np.array_equal(np.array(P.history["spikes"]), g[f"{k}_spikes"]), k
    assert int(g["fov_default_n"]) == 58
    assert (g["allo1_fr"] > 0.05).mean() > 0.005 and (g["fov2_fr"] > 0.05).mean() > 0.001


def test_oracle_reproduces_mode_a_against_placed_partners(golden):
    """get_state at 384 positions, one placed partner each (random, wall ends, on wall lines, the position itself,
    behind a wall, beyond a wall end), allocentric, Euclidean and egocentric with per-position head directions."""
    g = golden("avc.npz")
    env = O.OracleEnvironment(walls=WALLS)
    for k in POPS:
        hd = g["A_hd"] if k == "fov" else None
        assert np.array_equal(_state(g, k + "1", env, g["A_partner"], g["A_pos"], O.TapeRNG(), hd), g[f"A_{k}"]), k
    assert np.array_equal(_state(g, "allo1", env, g["B_partner"], g["A_pos"], O.TapeRNG()), g["B_allo"])
    assert np.array_equal(_state(g, "fov1", env, g["B_partner"], g["A_pos"][:16], O.TapeRNG(), np.array([1, 0])),
                          g["B_fov_default_hd"])
    assert list(g["B_fov_warnings"]) == ["OVCs in egocentric plane require a head direction vector but none was passed. "
                                         "Using [1,0]"]
    # the line-of-sight decisions of the placed cases are all present: blocked and clear, at distance 0 too
    d = O.distances_accounting_for_environment(env, g["A_pos"], g["A_partner"], "line_of_sight", O.TapeRNG()).diagonal()
    kind = g["A_kind"]
    assert (d[kind == 4] == 1000).any() and (d[kind == 4] < 1000).any()
    assert np.all(d[kind == 3] == 0)


def test_oracle_reproduces_the_special_cases(golden):
    g = golden("avc.npz")
    env = O.OracleEnvironment(walls=WALLS)
    # the Agent as its own partner: distance 0, bearing get_angle of a -0 vector
    self_pos, self_hd = g["self_pos"], g["self_hd"]
    want = V.avc_get_state(env, self_pos, tuple(g["self_tuning"]), self_pos, O.TapeRNG(), "line_of_sight", min_fr=0.1)
    assert np.array_equal(want, g["self_rates"])
    want = V.avc_get_state(env, self_pos, tuple(g["self_fov_tuning"]), self_pos, O.TapeRNG(), "line_of_sight",
                           head_direction=self_hd)
    assert np.array_equal(want, g["self_fov_rates"])
    # a NaN partner: NaN rates, and through update() NaN firing rates with no spikes
    assert np.all(np.isnan(g["nan_rates"])) and np.all(np.isnan(g["nan_fov_rates"]))
    assert np.all(np.isnan(g["nan_update_fr"])) and not g["nan_update_spikes"].any()
    nan_partner = np.array([np.nan, np.nan])
    assert np.all(np.isnan(_state(g, "allo1", env, nan_partner, g["pos_1"][-1], O.TapeRNG())))
    # no partner: zeros (the reference's are (n,); the oracle gives one column per position)
    assert np.array_equal(g["none_rates"], np.zeros(6)) and np.array_equal(g["none_rates_pos"], np.zeros(6))
    assert np.array_equal(V.avc_get_state(env, None, _tuning(g, "eucl1"), g["A_pos"][:5], O.TapeRNG()), np.zeros((6, 5)))
    # construction with Other_Agent = None fails on its agent_idx; FieldOfViewAVCs ignores an n it was given
    assert str(g["none_init_error"]) == "AttributeError"
    assert int(g["fov_n7_n"]) == 58
    assert list(g["fov_n7_warnings"]) == ["Ignoring 'n' parameter value (7) that was passed, and setting number of "
                                          "AgentVectorCell neurons to 58, inferred from the cell arrangement parameter."]
    assert len(g["avc_n7_warnings"]) == 0
    # get_head_direction_averaged_state of a FieldOfViewAVCs population: the mean over np.linspace(0, 2 pi, 12)
    acc = 0
    for ang in np.linspace(0, 2 * np.pi, 12):
        acc = acc + _state(g, "fov1", env, g["avg_partner"], g["avg_P"], O.TapeRNG(), np.array([np.cos(ang), np.sin(ang)]))
    assert np.allclose(acc / 12, g["avg_fov"], rtol=1e-12, atol=1e-15)


def test_mirror_default_params_match_the_reference(golden):
    import ratinabox_b200 as rb
    ref = json.loads(str(golden("avc.npz")["default_params_json"]))
    for name, want in ref.items():
        have = {}
        for c in reversed(getattr(rb, name).__mro__):
            have.update(getattr(c, "default_params", {}))
        for k, v in want.items():
            if k == "color":
                continue                                   # plotting only
            assert k in have, (name, k)
            assert np.array_equal(np.asarray(have[k], dtype=object), np.asarray(v, dtype=object)), (name, k, have[k], v)
        extra = set(have) - set(want) - {"color"}
        assert extra <= {"save_spikes", "history_bytes_limit"}, (name, sorted(extra))


def test_avc_pack_matches_numpy():
    from ratinabox_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(3)
    n = 37
    td, ta = rs.uniform(0.05, 0.3, n), rs.uniform(0, 2 * np.pi, n)
    sd, sa = rs.uniform(0.01, 0.2, n), rs.uniform(0.05, 1.0, n)
    meta = _lib.AvcCells()
    out = np.zeros(lib.riab_avc_pack_floats(n), dtype=np.float32)
    f = lambda a: a.ctypes.data_as(_lib.c_double_p)
    assert lib.riab_avc_pack(f(td), f(ta), f(sd), f(sa), n, C.byref(meta), out.ctypes.data_as(_lib.c_float_p)) == 0
    npad = meta.n_pad
    assert (meta.n_cells, npad, len(out)) == (n, 128, 5 * 128)
    log2e = np.log2(np.e)
    want = np.zeros((5, npad))
    want[2] = 1.0
    want[:, :n] = (td, np.sqrt(0.5 * log2e) / sd, np.cos(0.5 * ta), np.sin(0.5 * ta), np.sqrt(2.0 * (1 / sa ** 2) * log2e))
    want = want.astype(np.float32).reshape(-1)
    assert np.all(np.abs(out - want) <= np.spacing(np.abs(want))), np.abs(out - want).max()
    # the ObjectVectorCells block without its type column
    ovc = _lib.OvcCells()
    blk = np.zeros(lib.riab_ovc_pack_floats(n), dtype=np.float32)
    types = np.zeros(n, dtype=np.int32)
    assert lib.riab_ovc_pack(f(td), f(ta), f(sd), f(sa), types.ctypes.data_as(C.POINTER(C.c_int32)), n, C.byref(ovc),
                             blk.ctypes.data_as(_lib.c_float_p)) == 0
    assert np.array_equal(out, blk[: 5 * npad])
    assert lib.riab_avc_pack(None, f(ta), f(sd), f(sa), n, C.byref(meta), out.ctypes.data_as(_lib.c_float_p)) < 0
    assert b"riab_avc_pack" in lib.riab_last_error()


def test_avc_cells_struct_has_the_headers_layout(tmp_path):
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    fields = [f[0] for f in _lib.AvcCells._fields_]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "riab_b200.h"', "int main(void) {",
           '  printf("%zu\\n", sizeof(riab_avc_cells));']
    src += [f'  printf("%zu\\n", offsetof(riab_avc_cells, {f}));' for f in fields]
    src += ['  printf("%d\\n", RIAB_CELLS_AVC);', "  return 0;", "}"]
    c = tmp_path / "avc.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "avc"
    subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    assert int(lines[0]) == C.sizeof(_lib.AvcCells)
    for f, off in zip(fields, lines[1:]):
        assert getattr(_lib.AvcCells, f).offset == int(off), f
    assert int(lines[1 + len(fields)]) == _lib.CELLS_AVC == 7


def test_avc_step_kernels_are_built_with_the_launch_registers():
    """The k_step<AvcPolicy, MODE 0/1/2> instantiations exist with their configuration's launch registers."""
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([tool, "--dump-resource-usage", _lib.lib_path()], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*6k_stepIN\S*9AvcPolicyELi(\d)E\S*7StepCfgILi(\d+)E\S*):\s*\n\s*REG:(\d+) STACK:\d+ "
                       r"SHARED:(\d+)", txt)
    assert {m for _, m, _, _, _ in found} == {"0", "1", "2"}
    want = {"4": 96, "8": 80, "12": 80}
    for name, mode, cfg, reg, shared in found:
        assert int(reg) == want[cfg] and int(shared) <= 48 * 1024, (name[:100], reg, shared)

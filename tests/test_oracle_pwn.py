"""CPU checks of PlaneWaveNeurons: the float64 oracle (oracle/riab_oracle_pwn.py) against the live reference's fixture
(tests/golden/pwn.npz, oracle/gen_pwn_golden.py) bit for bit, the host class's defaults, and the riab_pwn_cells layout.
No CUDA calls."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

import riab_oracle_pwn as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _state(g, key, pos):
    lo, hi = g[f"{key}_fr"]
    return W.get_state(pos, g[f"{key}_phase_offsets"], g[f"{key}_w"], g[f"{key}_wavescales"], lo, hi)


def test_defaults_and_instance_params(golden):
    g = golden("pwn.npz")
    assert json.loads(str(g["default_params_json"])) == W.DEFAULTS
    inst = json.loads(str(g["instance_params_json"]))
    assert {k: inst[k] for k in W.DEFAULTS} == W.DEFAULTS


def test_draws_are_the_references(golden):
    g = golden("pwn.npz")
    for key in g["draw_keys"]:
        _, seed, n, ws = str(key).split("_")
        np.random.seed(int(seed))
        po, w, lam = W.draw(int(n), float(ws))
        assert np.array_equal(po, g[f"{key}_phase_offsets"]) and np.array_equal(w, g[f"{key}_w"])
        assert np.array_equal(lam, g[f"{key}_wavescales"]), key


@pytest.mark.parametrize("key", ["open", "walls"])
def test_oracle_reproduces_the_native_runs(golden, key):
    g = golden("pwn.npz")
    for s in range(len(g[f"{key}_pos"])):
        want = _state(g, key, g[f"{key}_pos"][s])[:, 0]
        assert np.array_equal(want, g[f"{key}_state"][s]) and np.array_equal(want, g[f"{key}_firingrate"][s]), (key, s)


@pytest.mark.parametrize("key", ["pos", "short1mm", "short1cm", "nonunit", "inverted"])
def test_oracle_reproduces_get_state(golden, key):
    g = golden("pwn.npz")
    assert np.array_equal(_state(g, key, g["pos_P"]), g[f"{key}_state"])
    if key in ("pos", "short1mm", "short1cm"):
        assert np.array_equal(_state(g, key, g["all_coords"]), g[f"{key}_all"])


def test_fixture_covers_what_it_says(golden):
    g = golden("pwn.npz")
    assert g["short1mm_wavescales"].max() == 1e-3 and g["short1cm_wavescales"].max() == 1e-2
    assert not np.allclose(np.linalg.norm(g["nonunit_w"], axis=1), 1.0)
    lo, hi = g["inverted_fr"]
    assert lo > hi and np.all(g["inverted_state"] <= lo) and np.all(g["inverted_state"] >= hi)
    assert str(g["periodic_printed"]) == W.PERIODIC_MESSAGE + "\n"


def test_host_class_defaults_match():
    from ratinabox_b200.contribs.PlaneWaveNeurons import PlaneWaveNeurons
    assert PlaneWaveNeurons.default_params == W.DEFAULTS


def test_pwn_cells_layout_matches_the_header():
    from ratinabox_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "riab_b200.h")).read()
    assert re.search(r"RIAB_CELLS_PWN = 10\b", hdr) and _lib.CELLS_PWN == 10
    assert C.sizeof(_lib.PwnCells) == 32
    assert [f[0] for f in _lib.PwnCells._fields_] == ["n_cells", "n_pad", "min_fr", "max_fr", "packed_dev", "phase_turns",
                                                      "reserved"]
    for name in ("riab_pwn_pack_floats", "riab_pwn_pack", "riab_pwn_rates"):
        assert name in hdr and name in _lib.SYMBOLS

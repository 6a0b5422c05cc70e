"""CPU checks of PhasePrecessingPlaceCells: the float64 oracle (oracle/riab_oracle_pppc.py) against the live reference's
fixture (tests/golden/pppc.npz, oracle/gen_pppc_golden.py) bit for bit (mode A: geometry jitter off), the host mirror's
defaults and constructor, and the riab_pppc_cells layout.  No CUDA calls."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

import riab_oracle as O
import riab_oracle_pppc as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNS = ("desc_gaussian", "desc_gaussian_threshold", "desc_diff_of_gaussians", "desc_top_hat", "los2", "geo1", "example")


def _env(g, k):
    return O.OracleEnvironment(walls=[w for w in g[f"{k}_walls"][4:]])


def _state(g, k, pos, vel, t, prm=None):
    prm = prm or json.loads(str(g[f"{k}_params"]))
    return P.get_state_agent(_env(g, k), pos, vel, t, g[f"{k}_centres"], g[f"{k}_widths"], O.TapeRNG(), prm["description"],
                             prm["wall_geometry"], prm["min_fr"], prm["max_fr"], prm["theta_freq"], prm["sigma"],
                             prm["precess_fraction"], scalar_width=prm["widths"])[:, 0]


@pytest.mark.parametrize("k", RUNS)
def test_oracle_reproduces_the_native_runs(golden, k):
    """Every step of the seeded runs: get_state(), firingrate and theta_modulation_factors() bit for bit."""
    g = golden("pppc.npz")
    prm = json.loads(str(g[f"{k}_params"]))
    for s in range(len(g[f"{k}_t"])):
        pos, vel, t = g[f"{k}_pos"][s], g[f"{k}_vel"][s], float(g[f"{k}_t"][s])
        want = _state(g, k, pos, vel, t)
        assert np.array_equal(want, g[f"{k}_state"][s]), (k, s)
        assert np.array_equal(want, g[f"{k}_firingrate"][s]), (k, s)
        f = P.theta_modulation_factors(pos, vel, t, g[f"{k}_centres"], g[f"{k}_widths"], prm["description"],
                                       prm["theta_freq"], prm["sigma"], prm["precess_fraction"])[:, 0]
        assert np.array_equal(f, g[f"{k}_factors"][s]), (k, s)


def test_oracle_reproduces_clocks_zero_velocity_and_edits(golden):
    g = golden("pppc.npz")
    k = "example"
    for t, want in zip(g["clock_t"], g["clock_state"]):
        assert np.array_equal(_state(g, k, g["clock_pos"], g["clock_vel"], float(t)), want), t
    assert np.array_equal(_state(g, k, g["zero_pos"], np.zeros(2), float(g["zero_t"])), g["zero_state"])
    assert np.all(np.isfinite(g["zero_state"]))
    prm = json.loads(str(g[f"{k}_params"]))
    before = _state(g, k, g["zero_pos"], g["edit_vel"], float(g["zero_t"]), prm)
    assert np.array_equal(before, g["edit_before"]) and np.array_equal(before, g["edit_kappa"])   # kappa is not read
    prm["sigma"] = float(g["edit_sigma_value"])
    assert np.array_equal(_state(g, k, g["zero_pos"], g["edit_vel"], float(g["zero_t"]), prm), g["edit_sigma"])
    assert not np.array_equal(g["edit_sigma"], g["edit_before"])


def test_away_from_the_agent_is_placecells_and_prints(golden):
    g = golden("pppc.npz")
    k = "example"
    prm = json.loads(str(g[f"{k}_params"]))
    for pts, key in ((g["away_P"], "away_pos"), (g["away_all_coords"], "away_all")):
        want = O.place_cells_get_state(_env(g, k), g[f"{k}_centres"], g[f"{k}_widths"], pts, O.TapeRNG(), prm["description"],
                                       prm["wall_geometry"], prm["min_fr"], prm["max_fr"], scalar_width=prm["widths"])
        assert np.array_equal(want, g[key]), key
        assert str(g[f"{key}_printed"]) == P.MESSAGE + "\n"


def test_defaults_constructor_and_quirks(golden):
    """The mirror's default_params, its merged params and sigma, the one_hot assert; the peak factor bound."""
    g = golden("pppc.npz")
    from ratinabox_b200.contribs import PhasePrecessingPlaceCells as Cls
    from ratinabox_b200 import PlaceCells
    assert json.loads(str(g["default_params_json"])) == Cls.default_params == P.DEFAULTS
    assert issubclass(Cls, PlaceCells)
    inst = json.loads(str(g["instance_params_json"]))
    assert inst["description"] == "gaussian_threshold" and inst["wall_geometry"] == "geodesic" and inst["widths"] == 0.2
    assert inst["sigma"] == float(np.sqrt(1 / 1))
    assert str(g["one_hot_raises"]) == "AssertionError:"
    assert str(g["top_hat_int_raises"]) == "UFuncTypeError"      # numpy: the in-place *= on an int64 array
    merged = {}
    for c in reversed(Cls.__mro__):
        merged.update(getattr(c, "default_params", {}))
    for key in ("description", "wall_geometry", "widths", "min_fr", "max_fr", "theta_freq", "kappa", "precess_fraction", "n",
                "name"):
        assert merged[key] == inst[key], key
    assert abs(P.peak_factor(1.0) - 2.14703) < 1e-5 and abs(P.peak_factor(np.sqrt(0.5)) - 3.24140) < 1e-5


def test_pppc_struct_has_the_headers_layout(tmp_path):
    from ratinabox_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "riab_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %d\\n", sizeof(riab_pppc_cells), offsetof(riab_pppc_cells, theta_freq), '
                   'offsetof(riab_pppc_cells, t), (int)RIAB_CELLS_PPPC);\n  return 0;\n}\n')
    exe = tmp_path / "s"
    subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    size, off_tf, off_t, kind = map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    assert C.sizeof(_lib.PppcCells) == size
    assert _lib.PppcCells.theta_freq.offset == off_tf and _lib.PppcCells.t.offset == off_t
    assert kind == _lib.CELLS_PPPC == 9

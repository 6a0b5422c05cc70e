"""CPU checks of imported / forced trajectories (Agent.import_trajectory, Agent.update(forced_next_position=...);
ratinabox/Agent.py:202-259, :543-659): the float64 oracle (oracle/riab_oracle_traj.py) against the live reference's
fixture (tests/golden/traj.npz, oracle/gen_traj_golden.py), the NumPy mirror of the device spline (tests/spline_np.py)
against scipy, the host mirror's validation, the new structs' layouts and the new kernels' resources.  No CUDA calls."""
import ctypes as C
import os
import re
import types

import numpy as np
import pytest
from scipy.interpolate import interp1d

import riab_oracle as O
import riab_oracle_traj as OT
import spline_np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATE = ("pos", "velocity", "rotational_velocity", "measured_velocity", "measured_rotational_velocity",
         "head_direction", "distance_travelled")


def _oracle_agent(g, case, env, dt):
    ag = OT.OracleTrajAgent(env, g[f"{case}_s0_pos"], g[f"{case}_s0_velocity"], {"dt": dt})
    for k in STATE:
        setattr(ag, k, np.array(g[f"{case}_s0_{k}"]) if g[f"{case}_s0_{k}"].ndim else float(g[f"{case}_s0_{k}"]))
    ag.t = float(g[f"{case}_s0_t"])
    return ag


def _check_run(g, case, ag, steps_kw):
    n = g[f"{case}_t"].shape[0]
    for i in range(n):
        ag.update(**steps_kw(i))
        for k in STATE + ("t",):
            assert np.array_equal(np.asarray(getattr(ag, k), dtype=np.float64), g[f"{case}_{k}"][i], equal_nan=True), \
                (case, i, k, getattr(ag, k), g[f"{case}_{k}"][i])
    assert np.array_equal(np.array(ag.history["pos"]), g[f"{case}_hist_pos"], equal_nan=True)
    assert np.array_equal(np.array(ag.history["vel"]), g[f"{case}_hist_vel"], equal_nan=True)


@pytest.mark.parametrize("case,dt", [("syn", 0.05), ("sar", 0.1), ("prec", 0.05)])
def test_oracle_reproduces_imported_runs_bit_for_bit(golden, case, dt):
    """Imported trajectories: an irregular one run past t_max (the wrap), and a sargolini slice imported at t != 0."""
    g = golden("traj.npz")
    src = "sar" if case == "sar" else "syn"
    env = O.OracleEnvironment(walls=g["box_walls"] if case == "syn" else ())
    ag = _oracle_agent(g, case, env, dt)
    ag.import_trajectory(g[f"{src}_times"], g[f"{src}_positions"])
    assert np.array_equal(ag.pos, g[f"{case}_s0_pos"])
    if case == "syn":
        assert g["syn_t"][-1] > g["syn_times"][-1] - g["syn_times"][0]           # the run wraps past t_max
    if case == "sar":
        assert float(g["sar_s0_t"]) > 0
    _check_run(g, case, ag, lambda i: {})


@pytest.mark.parametrize("case", ["frc", "per"])
def test_oracle_reproduces_forced_runs_bit_for_bit(golden, case):
    """Forced positions: a NaN sample (velocities NaN, distance unchanged), a zero displacement (the fall-back draw is
    an input), and a crossing of a periodic boundary (wrapped displacement)."""
    g = golden("traj.npz")
    env = O.OracleEnvironment(walls=g["box_walls"]) if case == "frc" else O.OracleEnvironment(boundary_conditions="periodic")
    ag = _oracle_agent(g, case, env, 0.05)
    F = g[f"{case}_forced"]
    fb = g["frc_fallback"] if case == "frc" else np.zeros(2)
    _check_run(g, case, ag, lambda i: {"forced_next_position": F[i].copy(), "fallback": fb})
    if case == "frc":
        assert np.isnan(g["frc_measured_velocity"][15]).all() and g["frc_distance_travelled"][15] == g["frc_distance_travelled"][14]
        assert 0 < np.linalg.norm(g["frc_fallback"]) <= 1.5e-7 and g["frc_rates_pc"][15].max() == 0.0
    else:
        d = np.abs(np.diff(g["per_pos"], axis=0)).max()
        assert d > 0.5 and np.abs(g["per_measured_velocity"] * 0.05).max() < 0.5    # wrapped, not across the box


def test_reference_error_cases(golden):
    g = golden("traj.npz")
    assert str(g["err_short"]) == "ValueError" and str(g["err_duplicate"]) == "ValueError"
    assert str(g["err_periodic"]) == "AssertionError"
    assert str(g["err_interpolate_false"]) == "AttributeError"     # the reference's own failure at Agent.py:657
    assert str(g["err_precedence"]) == "TypeError"                 # Agent.py:230 passes kwargs to a method without them


def _spline_err(x, y, q):
    return np.abs(spline_np.evaluate(x, y, spline_np.build(x, y), q) - interp1d(x, y, axis=0, kind="cubic")(q)).max()


def test_spline_mirror_matches_scipy(golden):
    g = golden("traj.npz")
    t = g["sar_times"] - g["sar_times"].min()
    q = np.random.default_rng(0).uniform(0, t.max(), 20000)
    assert _spline_err(t, g["sar_positions"], q) <= 1e-12                     # sargolini slice (0.02-0.36 s spacing)
    x = np.sort(np.random.default_rng(1).uniform(0, 20, 400))
    x -= x[0]
    y = np.stack([np.sin(x), np.cos(0.7 * x)], axis=1)
    assert _spline_err(x, y, np.linspace(0, x[-1], 5000)) <= 1e-12          # smooth
    rng = np.random.default_rng(2)
    x = np.concatenate([[0.0], np.cumsum(rng.uniform(0.001, 0.5, 999))])
    y = rng.uniform(-3, 3, (1000, 5, 2))                                       # rough, spacing ratios up to 500
    assert _spline_err(x, y, rng.uniform(0, x[-1], 5000)) <= 1e-12 * 6.0
    x = np.array([0.0, 0.3, 0.5, 1.2])                                         # T = 4, the smallest system
    y = rng.normal(size=(4, 2))
    assert _spline_err(x, y, np.linspace(0, 1.2, 50)) <= 1e-12


def _stub_agent(rb, env, n_agents=1):
    a = types.SimpleNamespace(Environment=env, n_agents=n_agents, _pending=None, use_imported_trajectory=False,
                              _src=types.SimpleNamespace())
    a._flush_pending = lambda: None
    return a


def test_host_mirror_validation_matches_the_reference(golden, capsys, tmp_path):
    """import_trajectory's and forced_next_position's checks raise what the reference raises (interp1d's exceptions
    for too few / duplicate times), before any device work -- the methods run on stand-ins."""
    import ratinabox_b200 as rb
    g = golden("traj.npz")
    times, pos = g["syn_times"], g["syn_positions"]
    imp = rb.Agent.import_trajectory
    a = _stub_agent(rb, rb.Environment())
    with pytest.raises(NotImplementedError, match="Agent.py:657"):
        imp(a, times=times, positions=pos, interpolate=False)
    assert not a.use_imported_trajectory
    with pytest.raises(AssertionError, match="Only solid boundary conditions are supported"):
        imp(_stub_agent(rb, rb.Environment({"boundary_conditions": "periodic"})), times=times, positions=pos)
    with pytest.raises(ValueError):
        imp(a, times=times[:3], positions=pos[:3])
    tdup = times.copy()
    tdup[5] = tdup[4]
    with pytest.raises(ValueError):
        imp(a, times=tdup, positions=pos)
    with pytest.raises(AssertionError, match="time and position arrays must have same length"):
        imp(a, times=times[:-1], positions=pos)
    with pytest.raises(NotImplementedError, match="per-agent time bases"):
        imp(_stub_agent(rb, rb.Environment(), 2), times=np.stack([times, times]), positions=np.stack([pos, pos]))
    capsys.readouterr()
    assert imp(a, dataset=str(tmp_path / "missing")) is None
    out = capsys.readouterr().out
    assert "IMPORT FAILED. No datafile found at" in out and not a.use_imported_trajectory
    stage = rb.Agent._stage_source
    with pytest.raises(AssertionError, match="forced_next_position must be an np.array$"):
        stage(a, [0.1, 0.2])
    with pytest.raises(AssertionError, match="forced_next_position must be an np.array of shape Env.D"):
        stage(a, np.zeros(3))


def test_structs_have_the_headers_layout(tmp_path):
    """ctypes mirrors of riab_trajectory / riab_motion_source against the C compiler's layout of include/riab_b200.h."""
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "riab_b200.h"', "int main(void) {",
           '  printf("%zu %zu %zu %zu %zu %zu %d %d %d %d\\n", sizeof(riab_trajectory), offsetof(riab_trajectory, t_max),'
           ' sizeof(riab_motion_source), offsetof(riab_motion_source, t), offsetof(riab_motion_source, traj),'
           ' offsetof(riab_motion_source, forced_dev), RIAB_MOTION_RANDOM, RIAB_MOTION_IMPORTED, RIAB_MOTION_FORCED,'
           ' RIAB_ABI_VERSION);', "  return 0;", "}"]
    c = tmp_path / "traj.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "traj"
    subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(_lib.Trajectory), _lib.Trajectory.t_max.offset, C.sizeof(_lib.MotionSource),
                   _lib.MotionSource.t.offset, _lib.MotionSource.traj.offset, _lib.MotionSource.forced_dev.offset,
                   _lib.MOTION_RANDOM, _lib.MOTION_IMPORTED, _lib.MOTION_FORCED, 3]


def test_trajectory_kernels_do_not_spill():
    """The spline build and the stand-alone imported / forced motion kernel keep everything in registers."""
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([tool, "--dump-resource-usage", _lib.lib_path()], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*(?:k_traj_build|k_agent_update_src)\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", txt)
    assert len(found) == 2, found
    for name, reg, stack, shared, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        assert int(reg) <= 128, (name, reg)

"""CPU: the NumPy restatement of DumbAgent, ShiftAgent and ReplayAgent (oracle/riab_oracle_subagents.py) against
tests/golden/subagents.npz, written from the live reference by oracle/gen_subagents_golden.py; the lazy replay rollout
against the eager one; and the layout of riab_subagent against its ctypes mirror."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import riab_oracle as O  # noqa: E402
from riab_oracle_subagents import OracleDumb, OracleReplay, shift_position  # noqa: E402

G = np.load(os.path.join(ROOT, "tests", "golden", "subagents.npz"))
CASES = json.loads(str(G["cases_json"]))
WALLS2 = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
HOLED = {"boundary": [[0, 0], [1.2, 0], [1.2, 0.4], [0.8, 1.0], [0, 1.0]],
         "holes": [[[0.4, 0.4], [0.6, 0.4], [0.6, 0.6], [0.4, 0.6]]]}


def meta(case):
    return json.loads(str(G[f"{case}_meta"]))


def subs_of(kind):
    return [(c, n) for c in CASES for n, (cls, _) in meta(c)["subs"].items() if cls == kind]


def oracle_env(kind):
    if kind == "periodic":
        return O.OracleEnvironment(boundary_conditions="periodic")
    if kind == "holed":
        return O.OracleEnvironment(boundary=HOLED["boundary"], holes=HOLED["holes"])
    return O.OracleEnvironment(walls=WALLS2 if kind == "walls" else ())


def replay_run(case, name, mode, xi=None):
    """(positions, flags, (speed, duration, start, end), oracle) of the recorded lead through OracleReplay."""
    m = meta(case)
    k = f"{case}_{name}"
    init = m["init"][name]
    o = OracleReplay(oracle_env(m["env"]), m["subs"][name][1], m["lead_params"]["dt"],
                     (init["sham_mv"], init["sham_hd"], init["sham_dist"]), mode=mode)
    starts = list(G[f"{k}_replay_start"])
    xi = G[f"{k}_replay_xi"] if xi is None else xi
    pos, flags, times = [], [], []
    r = -1
    for s in range(len(G[f"{case}_lead_t"])):
        if s in starts:
            r = starts.index(s)
        normals = np.nan_to_num(xi[r]) if r >= 0 else np.zeros((1, 2))
        pos.append(o.step(G[f"{case}_lead_pos"][s], G[f"{case}_lead_t"][s], G[f"{k}_draws"][s], normals))
        flags.append(o.is_undergoing_replay)
        times.append((o.replay_speed, o.replay_duration, o.replay_start_time, o.replay_end_time))
    return np.array(pos), np.array(flags), np.array(times), o


@pytest.mark.parametrize("case,name", subs_of("DumbAgent"))
def test_dumb_agent_bit_for_bit(case, name):
    m = meta(case)
    k = f"{case}_{name}"
    o = OracleDumb(oracle_env(m["env"]), m["subs"][name][1])
    init = m["init"][name]
    assert (o.tau_v, o.sigma, o.acceleration_scale) == (init["tau_v"], init["sigma"], init["acceleration_scale"])
    for s in range(len(G[f"{case}_lead_t"])):
        pos = o.step(G[f"{case}_lead_pos"][s], m["lead_params"]["dt"], G[f"{k}_xi"][s], G[f"{k}_resample"][s])
        assert np.array_equal(pos, G[f"{k}_pos"][s]), (k, s)
        assert np.array_equal(o.displacement, G[f"{k}_disp"][s]), (k, s)
    if case == "walls":
        # wall cuts happened, and no segment from the lead to the DumbAgent strictly crosses a wall
        assert o.cuts > 0
        walls = oracle_env("walls").walls
        for s in range(len(G[f"{case}_lead_t"])):
            seg = np.array([G[f"{case}_lead_pos"][s], G[f"{k}_pos"][s]])
            assert not O.vector_intercepts(walls, seg, O.TapeRNG(), return_collisions=True).any()


@pytest.mark.parametrize("case,name", subs_of("ShiftAgent"))
def test_shift_agent_bit_for_bit(case, name):
    m = meta(case)
    k = f"{case}_{name}"
    shift = m["subs"][name][1].get("shift_m", 0.01)
    for s in range(len(G[f"{case}_lead_t"])):
        pos = shift_position(G[f"{case}_lead_pos"][s], G[f"{case}_lead_hd"][s], shift)
        assert np.array_equal(pos, G[f"{k}_pos"][s]), (k, s)


@pytest.mark.parametrize("case,name", subs_of("ReplayAgent"))
def test_replay_agent_bit_for_bit(case, name):
    """Positions, flags and replay times of the lazy oracle equal the reference's bit for bit, and so do the eager
    oracle's."""
    k = f"{case}_{name}"
    lazy = replay_run(case, name, "lazy")
    eager = replay_run(case, name, "eager")
    for pos, flags, times, _ in (lazy, eager):
        assert np.array_equal(pos, G[f"{k}_pos"], equal_nan=True), k
        assert np.array_equal(flags, G[f"{k}_flag"]), k
        want = np.stack([G[f"{k}_speed"], G[f"{k}_duration"], G[f"{k}_start"], G[f"{k}_end"]], axis=1)
        assert np.array_equal(times, want, equal_nan=True), k
    assert G[f"{k}_flag"].any() and not G[f"{k}_flag"].all()
    assert np.array_equal(lazy[3].t, G[f"{k}_t"][-1])


def test_lazy_rollout_equals_eager_on_long_fresh_replays():
    """Fresh normals, replays of more than 500 rollout steps (replay_speed 5, duration 0.2 s): identical positions."""
    rs = np.random.RandomState(4)
    env = O.OracleEnvironment(walls=WALLS2)
    dt, T = 0.01, 120
    lead = np.stack([0.5 + 0.1 * np.cos(np.arange(T) * 0.05), 0.5 + 0.1 * np.sin(np.arange(T) * 0.05)], axis=1)
    longest = 0
    for trial in range(3):
        xi = rs.normal(size=(3000, 2))
        runs = []
        for mode in ("lazy", "eager"):
            o = OracleReplay(env, {"replay_freq": 5.0, "replay_speed": 5.0, "replay_duration": 0.2}, dt,
                             ([0.08, 0.0], [1.0, 0.0], 0.0), mode=mode)
            out = []
            for s in range(T):
                draws = (0.0 if s in (3, 60) else 1.0, 5.0, 0.2, 0.2 + 0.1 * trial, 0.8, 1.0 + trial)
                out.append(o.step(lead[s], (s + 1) * dt, draws, xi))
            runs.append(np.array(out))
            if mode == "eager":
                longest = max(longest, o.max_rollout)
        assert np.array_equal(runs[0], runs[1], equal_nan=True)
        assert np.isfinite(runs[0]).all()
    assert longest >= 500


def test_defaults_derived_and_warning():
    d = json.loads(str(G["default_params_json"]))
    assert d == {"DumbAgent": {"drift_distance": 0.05, "drift_timescale": 3.0},
                 "ReplayAgent": {"replay_freq": 0.3, "replay_duration": 0.1, "replay_speed": 1.0},
                 "ShiftAgent": {"shift_m": 0.01}, "UnrelatedAgent": {}}
    o = OracleDumb(None, {"drift_distance": 0.1, "drift_timescale": 2.0})
    assert json.loads(str(G["derived_json"])) == {"tau_v": o.tau_v, "sigma": o.sigma,
                                                  "acceleration_scale": o.acceleration_scale}
    assert "overwritten to match dt of the LeadAgent" in str(G["dt_warning"])


def test_subagent_struct_has_the_headers_layout(tmp_path):
    """gcc against include/riab_b200.h: sizeof and every offsetof of riab_subagent equal the ctypes mirror's."""
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    cls = _lib.SubAgentStep
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "riab_b200.h"', "int main(void) {",
           '  printf("sizeof %zu\\n", sizeof(riab_subagent));']
    for f, _ in cls._fields_:
        src.append(f'  printf("{f} %zu\\n", offsetof(riab_subagent, {f}));')
    src += ['  printf("fields %d\\n", RIAB_REPLAY_FIELDS);', "  return 0;", "}"]
    c = tmp_path / "sub.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "sub"
    subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True,
                                                        text=True).stdout.strip().splitlines())
    assert C.sizeof(cls) == int(out.pop("sizeof"))
    assert _lib.REPLAY_FIELDS == int(out.pop("fields"))
    for f, off in out.items():
        assert getattr(cls, f).offset == int(off), f

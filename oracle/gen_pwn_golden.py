"""TEST INFRASTRUCTURE -- write tests/golden/pwn.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): ratinabox/contribs/PlaneWaveNeurons.py.

    python oracle/gen_pwn_golden.py

Records: the class's default_params (JSON) and the params an instance ends up with; the drawn phase_offsets / w /
wavescales for a few seeds, sizes and wavescales; seeded native runs (Agent + cells, dt 0.05 s) in the open box and in a
box with two walls (walls do not enter the rates), with the agent's position, get_state() and firingrate per step;
get_state at 384 positions and at "all" for drawn cells, for hand-set short waves (wavescale 1e-3 and 1e-2 m) at all
orientations, and for a non-unit w; min_fr > max_fr; and the text printed in a periodic box.  Each record keeps the
inputs the oracle needs.
"""
import contextlib
import io
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
WALLS2 = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]


def printed(fn):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        r = fn()
    return r, buf.getvalue()


def cells(out, key, N):
    out[f"{key}_phase_offsets"] = np.array(N.phase_offsets, dtype=float)
    out[f"{key}_w"] = np.array(N.w, dtype=float)
    out[f"{key}_wavescales"] = np.array(N.wavescales, dtype=float)
    out[f"{key}_fr"] = np.array([float(N.min_fr), float(N.max_fr)])


def native_run(out, key, walls, params, n_steps=30, seed=0):
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.contribs.PlaneWaveNeurons import PlaneWaveNeurons
    np.random.seed(seed)
    Env = Environment()
    for w in walls:
        Env.add_wall(w)
    Ag = Agent(Env, {"dt": 0.05})
    N = PlaneWaveNeurons(Ag, params)
    rec = {k: [] for k in ("pos", "state", "firingrate")}
    for _ in range(n_steps):
        Ag.update()
        N.update()
        rec["pos"].append(np.array(Ag.pos, dtype=float))
        rec["state"].append(N.get_state()[:, 0])
        rec["firingrate"].append(np.array(N.firingrate, dtype=float))
    for k, v in rec.items():
        out[f"{key}_{k}"] = np.array(v)
    cells(out, key, N)
    return Ag, N


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.contribs.PlaneWaveNeurons import PlaneWaveNeurons
    out = {}
    out["default_params_json"] = np.array(json.dumps(PlaneWaveNeurons.default_params, sort_keys=True))
    np.random.seed(1)
    N0 = PlaneWaveNeurons(Agent(Environment()))
    inst = {k: (v if not isinstance(v, np.ndarray) else None) for k, v in N0.params.items()}
    out["instance_params_json"] = np.array(json.dumps(inst, sort_keys=True, default=float))

    # ---- the draws: seeds x sizes x wavescales, seeded after the Agent is built (its own draws do not enter)
    draws = []
    for seed in (0, 1, 7):
        for n in (1, 10, 37, 1024):
            for ws in (0.2, 0.05):
                Ag = Agent(Environment())
                np.random.seed(seed)
                N = PlaneWaveNeurons(Ag, {"n": n, "wavescale": ws})
                key = f"draw_{seed}_{n}_{ws}"
                cells(out, key, N)
                draws.append(key)
    out["draw_keys"] = np.array(draws)

    # ---- native runs (walls do not enter the rates)
    native_run(out, "open", [], {"n": 40}, seed=10)
    native_run(out, "walls", WALLS2, {"n": 33, "wavescale": 0.1, "min_fr": 0.5, "max_fr": 3.0}, seed=11)

    # ---- get_state at 384 positions and at "all"
    np.random.seed(12)
    Ag = Agent(Environment())
    N = PlaneWaveNeurons(Ag, {"n": 64})
    X = np.random.RandomState(3).uniform(0.0, 1.0, size=(384, 2))
    out["pos_P"] = X
    cells(out, "pos", N)
    out["pos_state"] = N.get_state(evaluate_at=None, pos=X)
    out["pos_all"] = N.get_state(evaluate_at="all")[:, ::37]                     # every 37th point (fixture size)
    out["all_coords"] = np.array(Ag.Environment.flattened_discrete_coords, dtype=float)[::37]
    # hand-set short waves at all orientations, and a non-unit w (used as stored)
    ang = np.linspace(0, 2 * np.pi, 24, endpoint=False)
    for key, lam in (("short1mm", 1e-3), ("short1cm", 1e-2)):
        N.w = np.stack([np.cos(ang), np.sin(ang)], axis=1)
        N.wavescales = np.full(24, lam)
        N.phase_offsets = np.random.RandomState(4).uniform(0, lam, size=(24, 2))
        N.n = 24
        cells(out, key, N)
        out[f"{key}_state"] = N.get_state(evaluate_at=None, pos=X)
        out[f"{key}_all"] = N.get_state(evaluate_at="all")[:, ::37]
    N.w = np.random.RandomState(5).normal(size=(24, 2)) * 1.7
    N.wavescales = np.random.RandomState(6).uniform(0.05, 0.5, 24)
    cells(out, "nonunit", N)
    out["nonunit_state"] = N.get_state(evaluate_at=None, pos=X)
    # min_fr > max_fr
    N.min_fr, N.max_fr = 2.0, 0.5
    cells(out, "inverted", N)
    out["inverted_state"] = N.get_state(evaluate_at=None, pos=X)

    # ---- the periodic box's message
    np.random.seed(13)
    _, txt = printed(lambda: PlaneWaveNeurons(Agent(Environment({"boundary_conditions": "periodic"})), {"n": 5}))
    out["periodic_printed"] = np.array(txt)
    np.savez_compressed(os.path.join(GOLD, "pwn.npz"), **out)
    print("pwn.npz", os.path.getsize(os.path.join(GOLD, "pwn.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()

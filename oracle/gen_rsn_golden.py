"""TEST INFRASTRUCTURE -- write tests/golden/rsn.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): RandomSpatialNeurons (ratinabox/Neurons.py:2865-2954).

    python oracle/gen_rsn_golden.py

Per environment (ENVS), under a fixed seed: X, the SHA-256 of Q's bytes and three of its rows, targets, the NumPy RNG
state after construction, and get_state(evaluate_at=None, pos=P) at 384 positions with the geometry jitter off (mode A:
np.random.normal of scale 1e-9 returns zeros), P including positions on and next to the inner walls' lines and ends.
Also: a native seeded run (Agent + RandomSpatialNeurons, euclidean box, 200 steps: positions and rates),
default_params (JSON), the lengthscale assertion, the printed geodesic -> line_of_sight message and the assertion of
walls in a periodic environment.
"""
import contextlib
import hashlib
import io
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
C2_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
HOLE = [[0.4, 0.4], [0.6, 0.4], [0.6, 0.6], [0.4, 0.6]]
# name: (Environment params, add_wall list, RandomSpatialNeurons params, seed)
ENVS = {
    "box": ({}, [], {"n": 10, "lengthscale": 0.1, "wall_geometry": "euclidean"}, 1),
    "wall21": ({"aspect": 2}, [[[1.0, 0.0], [1.0, 0.6]]], {"n": 12, "lengthscale": 0.1}, 2),
    "c2": ({}, C2_WALLS, {"n": 10, "lengthscale": 0.1}, 3),
    "periodic": ({"boundary_conditions": "periodic"}, [], {"n": 9, "lengthscale": 0.15, "wall_geometry": "euclidean"}, 4),
    "holed": ({"boundary": [[0, 0], [1, 0], [1, 1], [0, 1]], "walls": [[[0.8, 0.0], [0.8, 0.35]]], "holes": [HOLE]}, [],
              {"n": 8, "lengthscale": 0.08, "wall_geometry": "line_of_sight", "min_fr": 0.5, "max_fr": 3.0}, 5),
    "long": ({}, [], {"n": 10, "lengthscale": 0.02, "wall_geometry": "euclidean"}, 6),
}
N_POS = 384


@contextlib.contextmanager
def no_jitter():
    orig = np.random.normal

    def patched(loc=0.0, scale=1.0, size=None):
        if scale == 1e-9:
            return np.zeros(size)
        return orig(loc=loc, scale=scale, size=size)

    np.random.normal = patched
    try:
        yield
    finally:
        np.random.normal = orig


def special_positions(walls):
    """Points on and next to each inner wall's line and ends (at 0, +-1e-7, +-1e-3 across the line)."""
    pts = []
    for w in walls:
        a, b = np.asarray(w[0], float), np.asarray(w[1], float)
        t = b - a
        nrm = np.array([-t[1], t[0]]) / np.linalg.norm(t)
        for s in (0.0, 1e-7, -1e-7, 1e-3, -1e-3):
            for u in (0.0, 0.3, 1.0, 1.0 + 1e-3, 1.02):
                pts.append(a + u * t + s * nrm)
    return np.array(pts)


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import RandomSpatialNeurons
    out = {}
    for name, (eprm, walls, nprm, seed) in ENVS.items():
        Env = Environment(eprm)
        for w in walls:
            Env.add_wall(w)
        Ag = Agent(Env)
        np.random.seed(seed)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            N = RandomSpatialNeurons(Ag, dict(nprm, name=name))
        st = np.random.get_state()
        out[f"{name}_printed"] = np.array(buf.getvalue())
        out[f"{name}_walls"] = np.asarray(Env.walls, dtype=float)
        out[f"{name}_geometry"] = np.array(N.wall_geometry)
        out[f"{name}_X"] = N.X
        out[f"{name}_Q_sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(N.Q).tobytes()).hexdigest())
        rows = [0, N.Q.shape[0] // 2, N.Q.shape[0] - 1]
        out[f"{name}_Q_rows_idx"] = np.array(rows)
        out[f"{name}_Q_rows"] = N.Q[rows]
        out[f"{name}_targets"] = N.targets
        out[f"{name}_rng_keys"], out[f"{name}_rng_pos"] = st[1], np.array(st[2])
        out[f"{name}_rng_has_gauss"], out[f"{name}_rng_cached"] = np.array(st[3]), np.array(st[4])
        np.random.seed(100 + seed)
        inner = np.asarray(Env.walls, float)[4:] if N.wall_geometry != "euclidean" else np.zeros((0, 2, 2))
        sp = special_positions(inner)
        sp = sp[[bool(Env.check_if_position_is_in_environment(p)) for p in sp]] if len(sp) else sp.reshape(0, 2)
        P = np.vstack((Env.sample_positions(n=N_POS - len(sp), method="random"), sp))[:N_POS]
        out[f"{name}_P"] = P
        with no_jitter():
            out[f"{name}_gs"] = N.get_state(evaluate_at=None, pos=P)
        out[f"{name}_params"] = np.array(json.dumps({k: N.params[k] for k in ("n", "lengthscale", "min_fr", "max_fr")}))
        print(name, N.X.shape, N.wall_geometry, repr(buf.getvalue()[:60]))
    # native seeded run: euclidean box, jitter-free rates at the Agent's positions
    np.random.seed(7)
    Env = Environment()
    Ag = Agent(Env, {"dt": 0.05})
    N = RandomSpatialNeurons(Ag, {"n": 6, "lengthscale": 0.1, "wall_geometry": "euclidean", "name": "run"})
    pos, rates = [], []
    for _ in range(200):
        Ag.update()
        N.update()
        pos.append(Ag.pos.copy())
        rates.append(N.firingrate.copy())
    out["run_targets"], out["run_pos"], out["run_rates"] = N.targets, np.array(pos), np.array(rates)
    # messages
    try:
        RandomSpatialNeurons(Agent(Environment()), {"lengthscale": 0.01})
        raise RuntimeError("no assertion")
    except AssertionError as e:
        out["msg_lengthscale"] = np.array(str(e))
    try:
        RandomSpatialNeurons(Agent(Environment({"boundary_conditions": "periodic"})), {"n": 2})
        raise RuntimeError("no assertion")
    except AssertionError as e:
        out["msg_periodic_geodesic"] = np.array(str(e))
    d = {}
    for k, v in RandomSpatialNeurons.default_params.items():
        d[k] = v
    out["default_params_json"] = np.array(json.dumps(d, sort_keys=True))
    np.savez_compressed(os.path.join(GOLD, "rsn.npz"), **out)
    print("rsn.npz", os.path.getsize(os.path.join(GOLD, "rsn.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()

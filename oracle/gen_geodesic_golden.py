"""TEST INFRASTRUCTURE -- write tests/golden/geodesic.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): PlaceCells.get_state with wall_geometry "geodesic" (ratinabox/Neurons.py:936-981,
Environment.get_distances_between___accounting_for_environment, Environment.py:677-779).

    python oracle/gen_geodesic_golden.py

Records, for three one-wall layouts -- both ends inside the box (ep_valid 3), only end 0 inside (1, in an aspect-2 box)
and only end 1 inside (2) -- the wall, the box's aspect, the cell centres, the positions (random ones and rings within
3 widths of each end inside the box, in the wall's shadow, where detours with rates above 1e-3 lie) and get_state for
every description with min_fr > 0 and max_fr != 1.  For a wall with no end inside the box, the name of the exception
PlaceCells.get_state, PhasePrecessingPlaceCells.update and the RandomSpatialNeurons constructor raise.  Geometry jitter
is off (np.random.normal of scale 1e-9 / 1e-6 returns zeros), as in gen_pppc_golden.py.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from gen_pppc_golden import no_jitter  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
DESCS = ("gaussian", "gaussian_threshold", "diff_of_gaussians", "top_hat", "one_hot")
WIDTH, MIN_FR, MAX_FR = 0.12, 0.25, 2.5
# name: (wall, aspect, ep_valid)
CASES = {
    "free": ([[0.5, 0.2], [0.5, 0.8]], 1.0, 3),
    "end0_aspect2": ([[1.2, 0.35], [0.9, 1.0]], 2.0, 1),
    "end1": ([[0.4, 0.0], [0.6, 0.55]], 1.0, 2),
}
NO_END_INSIDE = [[0.5, 0.0], [0.5, 1.0]]


def _positions(rs, wall, aspect):
    lo, hi = np.array([0.0, 0.0]), np.array([aspect, 1.0])
    P = [lo + rs.uniform(size=(120, 2)) * (hi - lo)]
    for e in np.asarray(wall, dtype=float):
        if (e > lo).all() and (e < hi).all():
            r = rs.uniform(0.0, 3 * WIDTH, 180)[:, None]
            a = rs.uniform(0, 2 * np.pi, 180)[:, None]
            P.append(e + r * np.concatenate([np.cos(a), np.sin(a)], 1))
    P = np.concatenate(P)
    return P[((P > lo) & (P < hi)).all(axis=1)]


def _centres(rs, wall, aspect):
    lo, hi = np.array([0.0, 0.0]), np.array([aspect, 1.0])
    C = [lo + rs.uniform(size=(24, 2)) * (hi - lo)]
    for e in np.asarray(wall, dtype=float):
        if (e > lo).all() and (e < hi).all():
            r = rs.uniform(0.2, 2.0, 20)[:, None] * WIDTH
            a = rs.uniform(0, 2 * np.pi, 20)[:, None]
            C.append(e + r * np.concatenate([np.cos(a), np.sin(a)], 1))
    C = np.concatenate(C)
    return C[((C > lo) & (C < hi)).all(axis=1)]


def _raised(fn):
    try:
        fn()
    except Exception as e:                                   # the type is the record
        return type(e).__name__
    return "none"


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import PlaceCells, RandomSpatialNeurons
    from ratinabox.contribs.PhasePrecessingPlaceCells import PhasePrecessingPlaceCells
    out = {"cases": np.array(list(CASES)), "width": WIDTH, "min_fr": MIN_FR, "max_fr": MAX_FR}
    rs = np.random.RandomState(20)
    with no_jitter():
        for case, (wall, aspect, ep_valid) in CASES.items():
            np.random.seed(1)
            Env = Environment({"aspect": aspect})
            Env.add_wall(wall)
            Ag = Agent(Env)
            P, C = _positions(rs, wall, aspect), _centres(rs, wall, aspect)
            out[f"{case}_wall"], out[f"{case}_aspect"], out[f"{case}_ep_valid"] = np.array(wall), aspect, ep_valid
            out[f"{case}_pos"], out[f"{case}_centres"] = P, C
            for desc in DESCS:
                pc = PlaceCells(Ag, {"place_cell_centres": C, "widths": WIDTH, "description": desc,
                                     "wall_geometry": "geodesic", "min_fr": MIN_FR, "max_fr": MAX_FR})
                assert pc.wall_geometry == "geodesic"
                out[f"{case}_{desc}"] = pc.get_state(evaluate_at=None, pos=P)
        np.random.seed(2)
        Env = Environment()
        Env.add_wall(NO_END_INSIDE)
        Ag = Agent(Env)
        pc = PlaceCells(Ag, {"n": 10})
        out["no_end_wall"] = np.array(NO_END_INSIDE)
        out["no_end_place_get_state"] = np.array(_raised(lambda: pc.get_state(evaluate_at=None, pos=np.array([[0.2, 0.5]]))))
        Ag.update()
        pp = PhasePrecessingPlaceCells(Ag, {"n": 10})
        out["no_end_pppc_update"] = np.array(_raised(pp.update))
        out["no_end_rsn_init"] = np.array(_raised(lambda: RandomSpatialNeurons(Ag, {"n": 4, "lengthscale": 0.1})))
    path = os.path.join(GOLD, "geodesic.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

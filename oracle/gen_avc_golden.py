"""TEST INFRASTRUCTURE -- write tests/golden/avc.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): AgentVectorCells and FieldOfViewAVCs (ratinabox/Neurons.py:2151-2351).

    python oracle/gen_avc_golden.py

Records: both classes' default_params merged over their MRO (JSON); a native seeded run in ovc.npz's two-wall box with
two Agents, ``Ag1.update(); Ag2.update()`` then AgentVectorCells (allocentric), AgentVectorCells(walls_occlude=False)
and FieldOfViewAVCs both ways, 200 steps (global RNG, line-of-sight jitter on: the RNG state after construction is
recorded so the oracle can replay every draw); get_state at 384 positions (geometry jitter off) against partners placed
at random, at wall ends, on wall lines, behind a wall, beyond a wall end and at the position itself, allocentric and
egocentric with one head direction per position; ``tuning_type_agent = None``; a NaN partner (get_state and update); the
Agent as its own partner; FieldOfViewAVCs' n warning and the [1,0] warning; get_head_direction_averaged_state of a
FieldOfViewAVCs population.
"""
import contextlib
import io
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]        # ovc.npz's box
WALL_ENDS = np.array([[0.3, 0.5], [0.7, 0.5], [0.3, 0.0], [0.7, 1.0]])
POPS = {"allo": ("AgentVectorCells", {"n": 12}),
        "eucl": ("AgentVectorCells", {"n": 6, "walls_occlude": False, "min_fr": 0.2, "max_fr": 1.5}),
        "fov": ("FieldOfViewAVCs", {})}


@contextlib.contextmanager
def no_jitter():
    orig = np.random.normal

    def patched(loc=0.0, scale=1.0, size=None):
        if scale in (1e-9, 1e-6):
            return np.zeros(size)
        return orig(loc=loc, scale=scale, size=size)

    np.random.normal = patched
    try:
        yield
    finally:
        np.random.normal = orig


def recorded(fn):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf), warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        r = fn()
    return r, [str(x.message) for x in w]


def partners_for(pos, rs):
    """One partner per position, cycling through the geometric cases the line-of-sight test must get right."""
    out, kind = [], []
    for a, p in enumerate(pos):
        k = a % 6
        if k == 0:
            q = rs.uniform(0.02, 0.98, size=2)                                      # anywhere
        elif k == 1:
            q = WALL_ENDS[(a // 6) % 4].copy()                                       # a wall end
        elif k == 2:
            q = np.array([0.3, rs.uniform(0.0, 0.5)]) if (a // 6) % 2 else np.array([0.7, rs.uniform(0.5, 1.0)])   # on a wall
        elif k == 3:
            q = p.copy()                                                             # the position itself: distance 0
        elif k == 4:
            q = np.array([0.6 - p[0], p[1]])                                         # mirrored across x = 0.3
        else:
            e = WALL_ENDS[(a // 6) % 2]
            q = e + 0.5 * (e - p)                                                    # beyond a wall end, in line with it
        out.append(q)
        kind.append(k)
    return np.array(out), np.array(kind)


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import AgentVectorCells, FieldOfViewAVCs
    RN = type("RN", (), {"AgentVectorCells": AgentVectorCells, "FieldOfViewAVCs": FieldOfViewAVCs})
    out = {}
    d = {}
    for name in ("AgentVectorCells", "FieldOfViewAVCs"):
        merged = {}
        for c in reversed(getattr(RN, name).__mro__):
            merged.update(getattr(c, "default_params", {}))
        d[name] = merged
    out["default_params_json"] = np.array(json.dumps(d, sort_keys=True))

    # ---- native seeded run: two Agents, AVCs both ways
    np.random.seed(41)
    Env = Environment()
    for w in WALLS:
        Env.add_wall(w)
    Ag1 = Agent(Env, {"dt": 0.02})
    Ag2 = Agent(Env, {"dt": 0.02, "speed_mean": 0.15})
    pops = {}
    for tag, (me, other) in (("1", (Ag1, Ag2)), ("2", (Ag2, Ag1))):
        for k, (cls, prm) in POPS.items():
            pops[k + tag] = getattr(RN, cls)(me, other, dict(prm))
    for k, P in pops.items():
        out[f"{k}_tuning"] = np.stack((P.tuning_distances, P.tuning_angles, P.sigma_distances, P.sigma_angles))
        out[f"{k}_geom"] = np.array(P.wall_geometry)
        out[f"{k}_frame"] = np.array(P.reference_frame)
        out[f"{k}_fr_range"] = np.array([P.min_fr, P.max_fr], dtype=float)
    out["fov_default_n"] = np.array(pops["fov1"].n)
    for i, Ag in (("1", Ag1), ("2", Ag2)):
        out[f"pos0_{i}"], out[f"vel0_{i}"] = Ag.pos.copy(), Ag.velocity.copy()
    st = np.random.get_state()
    out["rng_keys"], out["rng_pos"], out["rng_has_gauss"], out["rng_cached"] = st[1], st[2], st[3], st[4]
    for _ in range(200):
        Ag1.update()
        Ag2.update()
        for P in pops.values():
            P.update()
    for i, Ag in (("1", Ag1), ("2", Ag2)):
        out[f"pos_{i}"], out[f"head_{i}"] = np.array(Ag.history["pos"]), np.array(Ag.history["head_direction"])
    for k, P in pops.items():
        out[f"{k}_fr"] = np.array(P.history["firingrate"])
        out[f"{k}_spikes"] = np.array(P.history["spikes"])

    # ---- mode A: get_state at given positions against placed partners (jitter off)
    rs = np.random.RandomState(43)
    A = 384
    pos = rs.uniform(0.02, 0.98, size=(A, 2))
    partner, kind = partners_for(pos, rs)
    ang = rs.uniform(0, 2 * np.pi, size=A)
    hd = np.stack((np.cos(ang), np.sin(ang)), axis=1)
    out["A_pos"], out["A_partner"], out["A_kind"], out["A_hd"] = pos, partner, kind, hd
    with no_jitter():
        for k in POPS:
            P = pops[k + "1"]
            cols = []
            for a in range(A):
                Ag2.pos = partner[a]
                if P.reference_frame == "egocentric":
                    cols.append(P.get_state(evaluate_at=None, pos=pos[a], head_direction=hd[a])[:, 0])
                else:
                    cols.append(P.get_state(evaluate_at=None, pos=pos[a])[:, 0])
            out[f"A_{k}"] = np.stack(cols, axis=1)
        # one partner for every position, allocentric, and the [1,0] default of the egocentric cells (with its warning)
        Ag2.pos = np.array([0.62, 0.41])
        out["B_partner"] = Ag2.pos.copy()
        out["B_allo"] = pops["allo1"].get_state(evaluate_at=None, pos=pos)
        r, w = recorded(lambda: pops["fov1"].get_state(evaluate_at=None, pos=pos[:16]))
        out["B_fov_default_hd"], out["B_fov_warnings"] = r, np.array(w)

        # ---- the Agent as its own partner, at the agent and through update()
        S = RN.AgentVectorCells(Ag1, Ag1, {"n": 9, "min_fr": 0.1})
        F = RN.FieldOfViewAVCs(Ag1, Ag1, {"spatial_resolution": 0.05})
        out["self_tuning"] = np.stack((S.tuning_distances, S.tuning_angles, S.sigma_distances, S.sigma_angles))
        out["self_fov_tuning"] = np.stack((F.tuning_distances, F.tuning_angles, F.sigma_distances, F.sigma_angles))
        out["self_pos"], out["self_hd"] = Ag1.pos.copy(), np.array(Ag1.head_direction, dtype=float)
        out["self_rates"] = S.get_state()
        out["self_fov_rates"] = F.get_state()

        # ---- NaN partner: NaN rates and, through update(), NaN firing rates and no spikes
        Ag2.pos = np.array([np.nan, np.nan])
        out["nan_rates"] = pops["allo1"].get_state()
        out["nan_fov_rates"] = pops["fov1"].get_state()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            pops["allo1"].update()
        out["nan_update_fr"] = pops["allo1"].firingrate.copy()
        out["nan_update_spikes"] = np.array(pops["allo1"].history["spikes"][-1])

        # ---- no partner: zeros, not min_fr
        E = pops["eucl1"]
        E.tuning_type_agent = None
        out["none_rates"] = E.get_state()
        out["none_rates_pos"] = E.get_state(evaluate_at=None, pos=pos[:5])

    # ---- construction: None partner, the FoV n warning
    try:
        RN.AgentVectorCells(Ag1, None)
        out["none_init_error"] = np.array("")
    except Exception as e:                                  # noqa: BLE001
        out["none_init_error"] = np.array(type(e).__name__)
    r, w = recorded(lambda: RN.FieldOfViewAVCs(Ag1, Ag2, {"n": 7}))
    out["fov_n7_n"], out["fov_n7_warnings"] = np.array(r.n), np.array(w)
    r, w = recorded(lambda: RN.AgentVectorCells(Ag1, Ag2, {"n": 7}))
    out["avc_n7_warnings"] = np.array(w, dtype=str).reshape(-1)

    # ---- get_head_direction_averaged_state of a FieldOfViewAVCs population
    Ag2.pos = np.array([0.45, 0.62])
    out["avg_partner"] = Ag2.pos.copy()
    Pf = np.random.RandomState(44).uniform(0.05, 0.95, size=(6, 2))
    out["avg_P"] = Pf
    with no_jitter():
        out["avg_fov"] = pops["fov1"].get_head_direction_averaged_state(evaluate_at=None, pos=Pf, angular_resolution_degrees=30)
    np.savez_compressed(os.path.join(GOLD, "avc.npz"), **out)
    print("avc.npz", os.path.getsize(os.path.join(GOLD, "avc.npz")) // 1024, "KiB;",
          "fov n =", int(out["fov_default_n"]), "; max rates", {k: float(out[f"A_{k}"].max()) for k in POPS})


if __name__ == "__main__":
    main()

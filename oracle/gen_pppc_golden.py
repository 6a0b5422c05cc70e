"""TEST INFRASTRUCTURE -- write tests/golden/pppc.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): ratinabox/contribs/PhasePrecessingPlaceCells.py.

    python oracle/gen_pppc_golden.py

Records: the class's default_params (JSON) and the params an instance ends up with; seeded native runs (Agent + cells,
dt = 0.05 s, so every other step crosses a 10 Hz theta cycle) for each of the four allowed descriptions in the open box,
for a two-wall box with line_of_sight and a one-wall box with geodesic, and for the reference's own example (kappa 2,
precess_fraction 1, theta_freq 5) with min_fr > 0; get_state at clocks on and next to theta-cycle boundaries; a zero
velocity; kappa edited versus sigma edited after construction; get_state(pos=P) / "all" with the printed text; the
one_hot AssertionError.  Each record keeps the inputs the oracle needs (positions, velocities, clocks, centres, widths).
Geometry jitter is off (np.random.normal of scale 1e-9 / 1e-6 returns zeros), as in gen_kin_golden.py.
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
WALL1 = [[[0.5, 0.2], [0.5, 0.8]]]


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


def printed(fn):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        r = fn()
    return r, buf.getvalue()


def cell_params(P):
    return {"description": P.description, "wall_geometry": P.wall_geometry, "min_fr": float(P.min_fr),
            "max_fr": float(P.max_fr), "theta_freq": float(P.theta_freq), "sigma": float(P.sigma),
            "precess_fraction": float(P.precess_fraction), "widths": float(P.widths)}


def native_run(out, key, walls, params, n_steps=24, seed=0):
    """Agent + cells: per step the agent's pos / velocity / t, get_state(), theta_modulation_factors() and firingrate."""
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.contribs.PhasePrecessingPlaceCells import PhasePrecessingPlaceCells
    np.random.seed(seed)
    Env = Environment()
    for w in walls:
        Env.add_wall(w)
    Ag = Agent(Env, {"dt": 0.05})
    P = PhasePrecessingPlaceCells(Ag, params)
    rec = {k: [] for k in ("pos", "vel", "t", "state", "factors", "firingrate")}
    for _ in range(n_steps):
        Ag.update()
        P.update()
        rec["pos"].append(np.array(Ag.pos, dtype=float))
        rec["vel"].append(np.array(Ag.velocity, dtype=float))
        rec["t"].append(float(Ag.t))
        rec["state"].append(P.get_state()[:, 0])
        rec["factors"].append(P.theta_modulation_factors()[:, 0])
        rec["firingrate"].append(np.array(P.firingrate, dtype=float))
    for k, v in rec.items():
        out[f"{key}_{k}"] = np.array(v)
    out[f"{key}_centres"] = np.array(P.place_cell_centres, dtype=float)
    out[f"{key}_widths"] = np.array(P.place_cell_widths, dtype=float)
    out[f"{key}_walls"] = np.array(Env.walls, dtype=float)
    out[f"{key}_params"] = np.array(json.dumps(cell_params(P)))
    return Ag, P


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.contribs.PhasePrecessingPlaceCells import PhasePrecessingPlaceCells
    out = {}
    out["default_params_json"] = np.array(json.dumps(PhasePrecessingPlaceCells.default_params, sort_keys=True))
    np.random.seed(1)
    P0 = PhasePrecessingPlaceCells(Agent(Environment()))
    inst = {k: (v if not isinstance(v, np.ndarray) else None) for k, v in P0.params.items()}
    inst["sigma"] = float(P0.sigma)
    out["instance_params_json"] = np.array(json.dumps(inst, sort_keys=True, default=float))

    with no_jitter():
        for i, desc in enumerate(("gaussian", "gaussian_threshold", "diff_of_gaussians", "top_hat")):
            # (top_hat with the integer default min_fr / max_fr makes an int64 rate array, which the in-place `*=` of
            # get_state cannot take: recorded below; the run uses max_fr = 1.0)
            prm = {"n": 37, "description": desc, "widths": 0.25, **({"max_fr": 1.0} if desc == "top_hat" else {})}
            native_run(out, f"desc_{desc}", [], prm, seed=10 + i)
        native_run(out, "los2", WALLS2, {"n": 50, "wall_geometry": "line_of_sight", "widths": 0.2}, seed=20)
        native_run(out, "geo1", WALL1, {"n": 50, "wall_geometry": "geodesic", "description": "gaussian"}, seed=21)
        Ag, P = native_run(out, "example", [], {"n": 40, "widths": 0.3, "theta_freq": 5, "precess_fraction": 1, "kappa": 2,
                                                "max_fr": 10.0, "min_fr": 0.5, "description": "gaussian"}, seed=22)

        # ---- clocks on and next to theta-cycle boundaries (theta_freq 5: period 0.2 s), the agent's state fixed
        ts = []
        for k in (0, 1, 3, 7, 50):
            for e in (-1e-9, 0.0, 1e-9, 0.05, 0.1):
                ts.append(k * 0.2 + e)
        ts += [0.6000000000000001, 0.30000000000000004, 12345.678]
        out["clock_t"] = np.array(ts)
        out["clock_pos"], out["clock_vel"] = np.array(Ag.pos, dtype=float), np.array(Ag.velocity, dtype=float)
        st = []
        for t in ts:
            Ag.t = t
            st.append(P.get_state()[:, 0])
        out["clock_state"] = np.array(st)

        # ---- zero velocity: d = 0, the factor depends on the phase only
        Ag.t = 0.37
        Ag.velocity = np.array([0.0, 0.0])
        out["zero_t"], out["zero_pos"] = np.array(Ag.t), np.array(Ag.pos, dtype=float)
        out["zero_state"] = P.get_state()[:, 0]

        # ---- kappa edited (ignored) versus sigma edited (used) after construction
        Ag.velocity = np.array([0.11, -0.07])
        out["edit_vel"] = np.array(Ag.velocity, dtype=float)
        out["edit_before"] = P.get_state()[:, 0]
        P.kappa = 7.0
        out["edit_kappa"] = P.get_state()[:, 0]
        P.sigma = np.sqrt(1 / 4.0)
        out["edit_sigma"] = P.get_state()[:, 0]
        out["edit_sigma_value"] = np.array(P.sigma)

        # ---- away from the agent: PlaceCells rates and the message
        Pp = np.random.RandomState(5).uniform(0.05, 0.95, size=(9, 2))
        out["away_P"] = Pp
        r, txt = printed(lambda: P.get_state(evaluate_at=None, pos=Pp))
        out["away_pos"], out["away_pos_printed"] = r, np.array(txt)
        r, txt = printed(lambda: P.get_state(evaluate_at="all"))
        out["away_all"], out["away_all_printed"] = r[:, ::97], np.array(txt)           # every 97th point (fixture size)
        out["away_all_coords"] = np.array(Ag.Environment.flattened_discrete_coords, dtype=float)[::97]

    # ---- one_hot is refused by a bare assert
    try:
        PhasePrecessingPlaceCells(Agent(Environment()), {"description": "one_hot"})
        out["one_hot_raises"] = np.array("")
    except AssertionError as e:
        out["one_hot_raises"] = np.array(f"AssertionError:{e}")
    try:
        np.random.seed(2)
        Ag = Agent(Environment())
        P = PhasePrecessingPlaceCells(Ag, {"description": "top_hat"})
        Ag.update()
        P.update()
        out["top_hat_int_raises"] = np.array("")
    except Exception as e:
        out["top_hat_int_raises"] = np.array(type(e).__name__)
    np.savez_compressed(os.path.join(GOLD, "pppc.npz"), **out)
    print("pppc.npz", os.path.getsize(os.path.join(GOLD, "pppc.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()

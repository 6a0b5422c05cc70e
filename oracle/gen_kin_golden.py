"""TEST INFRASTRUCTURE -- write tests/golden/kin.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): HeadDirectionCells, VelocityCells and SpeedCell (ratinabox/Neurons.py:2357-2651) and
Neurons.get_head_direction_averaged_state (:176-192).

    python oracle/gen_kin_golden.py

Records: each class's default_params (JSON), preferred_angles and angular_tunings; a seeded native run (Agent +
HeadDirectionCells, 40 steps) with the agent's head direction / velocity / measured velocity and get_state() /
get_state(use_velocity=True) at every step; get_state with a head_direction kwarg, with the deprecated vel kwarg (its
warning) and with none (the printed [1,0] default), also at "all" and at pos=P; VelocityCells and SpeedCell with
min_fr > 0 and with max_fr < min_fr; a spread near kappa = 700; a zero velocity (NaN); SpeedCell's default 10-wide
firingrate next to its n=1 run; get_head_direction_averaged_state for HeadDirectionCells at "all" and for a
FieldOfViewBVCs population at pos=P (geometry jitter off: np.random.normal of scale 1e-9 / 1e-6 returns zeros).
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
KAPPA700_DEG = float(np.degrees(1 / np.sqrt(700.0)))        # angular spread with kappa = 1/sigma^2 = 700


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
    with contextlib.redirect_stdout(buf), warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        r = fn()
    return r, buf.getvalue(), [str(x.message) for x in w]


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import HeadDirectionCells, VelocityCells, SpeedCell, FieldOfViewBVCs
    out = {}
    d = {}
    for cls in (HeadDirectionCells, VelocityCells, SpeedCell):
        d[cls.__name__] = dict(cls.default_params)
    out["default_params_json"] = np.array(json.dumps(d, sort_keys=True))

    # ---- defaults and a seeded native run
    np.random.seed(11)
    Env = Environment()
    Ag = Agent(Env, {"dt": 0.05})
    H = HeadDirectionCells(Ag)
    V = VelocityCells(Ag)
    out["hdc_preferred_angles"], out["hdc_angular_tunings"] = H.preferred_angles, H.angular_tunings
    out["vel_preferred_angles"], out["vel_angular_tunings"] = V.preferred_angles, V.angular_tunings
    out["vel_one_sigma_speed"] = np.array(V.one_sigma_speed)
    keys = ("hd", "vel", "mvel", "hdc", "hdc_usevel", "velc")
    run = {k: [] for k in keys}
    for _ in range(40):
        Ag.update()
        H.update()
        V.update()
        run["hd"].append(np.array(Ag.head_direction, dtype=float))
        run["vel"].append(np.array(Ag.velocity, dtype=float))
        run["mvel"].append(np.array(Ag.history["vel"][-1], dtype=float))
        run["hdc"].append(H.get_state())
        run["hdc_usevel"].append(H.get_state(use_velocity=True))
        run["velc"].append(V.get_state())
    for k in keys:
        out[f"run_{k}"] = np.array(run[k])
    out["run_hdc_firingrate"] = H.firingrate.copy()

    # ---- kwargs away from the agent (the agent's state is irrelevant there, but VelocityCells' speed factor)
    hd = np.array([-0.3, 0.8])
    P = np.random.RandomState(5).uniform(0.05, 0.95, size=(7, 2))
    out["kw_hd"], out["kw_P"] = hd, P
    out["kw_head_direction"] = H.get_state(evaluate_at=None, head_direction=hd)
    out["kw_head_direction_all"] = H.get_state(evaluate_at="all", head_direction=hd)
    out["kw_head_direction_pos"] = H.get_state(evaluate_at=None, pos=P, head_direction=hd)
    r, p, w = printed(lambda: H.get_state(evaluate_at=None, vel=hd))
    out["kw_vel"], out["kw_vel_warnings"] = r, np.array(w)
    r, p, w = printed(lambda: H.get_state(evaluate_at=None))
    out["kw_none"], out["kw_none_printed"] = r, np.array(p)
    r, p, w = printed(lambda: H.get_state(evaluate_at=None, use_velocity=True))
    out["kw_none_usevel"], out["kw_none_usevel_printed"] = r, np.array(p)
    out["kw_velocity_usevel"] = H.get_state(evaluate_at=None, use_velocity=True, velocity=hd)
    out["kw_agent_velocity"] = np.array(Ag.velocity, dtype=float)
    out["kw_velc_velocity"] = V.get_state(evaluate_at=None, velocity=hd)
    out["kw_velc_velocity_pos"] = V.get_state(evaluate_at=None, pos=P, velocity=hd)

    # ---- min_fr > 0, max_fr < min_fr; a narrow spread; SpeedCell
    cases = {"lo": {"min_fr": 0.3, "max_fr": 2.5}, "inv": {"min_fr": 1.5, "max_fr": 0.2}}
    vel = np.array([0.07, -0.12])
    out["fr_vel"] = vel
    for name, prm in cases.items():
        Vc = VelocityCells(Ag, dict(prm, n=13, angular_spread_degrees=30))
        Sc = SpeedCell(Ag, dict(prm))
        Hc = HeadDirectionCells(Ag, dict(prm, n=13, angular_spread_degrees=30))
        out[f"fr_{name}_params"] = np.array(json.dumps(prm))
        out[f"fr_{name}_velc"] = Vc.get_state()
        out[f"fr_{name}_velc_kw"] = Vc.get_state(evaluate_at=None, velocity=vel)
        out[f"fr_{name}_hdc"] = Hc.get_state()
        out[f"fr_{name}_speed_agent"] = Sc.get_state()
        out[f"fr_{name}_speed_kw"] = Sc.get_state(evaluate_at=None, vel=vel)
    out["fr_agent_hd"], out["fr_agent_vel"] = np.array(Ag.head_direction, dtype=float), np.array(Ag.velocity, dtype=float)
    out["fr_agent_mvel"] = np.array(Ag.history["vel"][-1], dtype=float)
    out["narrow_deg"] = np.array(KAPPA700_DEG)
    Hn = HeadDirectionCells(Ag, {"n": 36, "angular_spread_degrees": KAPPA700_DEG})
    th = np.linspace(0, 2 * np.pi, 200, endpoint=False) + 0.0123
    out["narrow_theta"] = th
    out["narrow"] = np.stack([Hn.get_state(evaluate_at=None, head_direction=[np.cos(t), np.sin(t)])[:, 0] for t in th], axis=1)

    # ---- zero velocity: 0/0
    Ag.velocity = np.array([0.0, 0.0])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out["zero_velc"] = V.get_state()
        out["zero_hdc_usevel"] = H.get_state(use_velocity=True)

    # ---- SpeedCell: default (10-wide noise) and n=1
    np.random.seed(12)
    Ag2 = Agent(Environment(), {"dt": 0.05})
    S10 = SpeedCell(Ag2)
    r, p, w = printed(lambda: SpeedCell(Ag2, {"n": 1}))
    S1 = r
    r, p, w = printed(lambda: SpeedCell(Ag2, {"n": 4}))
    out["speed_n4_warnings"] = np.array(w)
    sp = {"mvel": [], "s10": [], "s1": []}
    for _ in range(5):
        Ag2.update()
        S10.update()
        S1.update()
        sp["mvel"].append(np.array(Ag2.history["vel"][-1], dtype=float))
        sp["s10"].append(S10.firingrate.copy())
        sp["s1"].append(S1.firingrate.copy())
    for k, v in sp.items():
        out[f"speed_run_{k}"] = np.array(v)
    out["speed_one_sigma_speed"] = np.array(S10.one_sigma_speed)
    out["speed_default_n"] = np.array(S10.n)
    out["speed_default_history_width"] = np.array(np.array(S10.history["firingrate"]).shape[-1])

    # ---- get_head_direction_averaged_state
    np.random.seed(13)
    Ag3 = Agent(Environment(), {"dt": 0.05})
    H3 = HeadDirectionCells(Ag3, {"n": 8, "angular_spread_degrees": 30, "min_fr": 0.1, "max_fr": 1.7})
    out["avg_hdc_all"] = H3.get_head_direction_averaged_state(evaluate_at="all")
    out["avg_hdc_all_res30"] = H3.get_head_direction_averaged_state(evaluate_at="all", angular_resolution_degrees=30)
    out["avg_hdc_agent"] = H3.get_head_direction_averaged_state()
    out["avg_agent_hd"] = np.array(Ag3.head_direction, dtype=float)
    Env4 = Environment()
    Env4.add_wall([[0.3, 0.0], [0.3, 0.5]])
    F = FieldOfViewBVCs(Agent(Env4, {"dt": 0.05}), {"min_fr": 0.0, "max_fr": 2.0})
    Pf = np.random.RandomState(6).uniform(0.05, 0.95, size=(6, 2))
    out["avg_fov_P"] = Pf
    with no_jitter():
        out["avg_fov"] = F.get_head_direction_averaged_state(evaluate_at=None, pos=Pf, angular_resolution_degrees=30)
    np.savez_compressed(os.path.join(GOLD, "kin.npz"), **out)
    print("kin.npz", os.path.getsize(os.path.join(GOLD, "kin.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()

"""TEST INFRASTRUCTURE -- write tests/golden/subagents.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): ratinabox/contribs/SubAgent.py, DumbAgent (:118-179), ReplayAgent (:358-431), ShiftAgent (:466-478)
and UnrelatedAgent (:480-489).

    python oracle/gen_subagents_golden.py

Geometry jitter is off (np.random.normal with scale 1e-9 / 1e-6 returns zeros), as in gen_tsa_golden.py.  One lead Agent
drives every SubAgent of a case; per step the fixture holds the lead's state after its update (pos, velocity, head
direction, t) and, per SubAgent, its pos, measured velocity, measured rotational velocity, head direction, distance
travelled and t, plus the draws it took from np.random:
  * DumbAgent: the two standard normals of its OU step (:154-159), the re-drawn position of a polygon / hole (NaN
    when none), and its displacement after the step;
  * ReplayAgent: (u, replay_speed, the Rayleigh duration before its clamp, x0, y0, direction) of the steps that draw
    them (NaN otherwise: no draw while replaying, :391), the flag and the replay's speed / duration / start / end after
    the step, and per replay the standard normals of the sham agent's rollout (:408-410) and its length;
  * UnrelatedAgent: the two standard normals of its Agent.update.
Cases: an open box (600 steps, dt = 0.01) with DumbAgent defaults, ShiftAgent at +-shift_m, UnrelatedAgent and a
ReplayAgent at replay_freq = 5; the two-inner-wall box of gen_tsa_golden.py with a fast lead and drift_distance = 0.2
(wall cuts); a periodic box; the holed polygon of tests/test_gpu_theta_sequence.py (wall cuts on the hole's edges, replay
starts inside the polygon; the cut keeps the DumbAgent inside, so its re-draw branch is not reached); a ReplayAgent
with replay_speed = 3 (long rollouts).  Also the default params, the derived attributes and the dt warning.
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
WALLS2 = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
HOLED = {"boundary": [[0, 0], [1.2, 0], [1.2, 0.4], [0.8, 1.0], [0, 1.0]],
         "holes": [[[0.4, 0.4], [0.6, 0.4], [0.6, 0.6], [0.4, 0.6]]]}


class Recorder:
    """np.random.normal / uniform / rayleigh and Environment.sample_positions, recorded per context (the object whose
    update is running); geometry jitter returns zeros."""

    def __init__(self):
        self.normal0, self.uniform0, self.rayleigh0 = np.random.normal, np.random.uniform, np.random.rayleigh
        self.ctx = None
        self.log = []

    def normal(self, loc=0.0, scale=1.0, size=None):
        if scale in (1e-9, 1e-6):
            return np.zeros(size)
        g = self.normal0(loc=0.0, scale=1.0, size=size)
        self.log.append((self.ctx, "normal", np.asarray(g, dtype=float).reshape(-1).tolist()))
        return loc + scale * g

    def uniform(self, low=0.0, high=1.0, size=None):
        u = self.uniform0(low, high, size)
        self.log.append((self.ctx, "uniform", np.asarray(u, dtype=float).reshape(-1).tolist()))
        return u

    def rayleigh(self, scale=1.0, size=None):
        r = self.rayleigh0(scale=scale, size=size)
        self.log.append((self.ctx, "rayleigh", np.asarray(r, dtype=float).reshape(-1).tolist()))
        return r

    def install(self):
        np.random.normal, np.random.uniform, np.random.rayleigh = self.normal, self.uniform, self.rayleigh

    def remove(self):
        np.random.normal, np.random.uniform, np.random.rayleigh = self.normal0, self.uniform0, self.rayleigh0

    def take(self, ctx, kind):
        out = [v for c, k, v in self.log if c == ctx and k == kind]
        return out


def in_context(rec, obj, meth, ctx):
    orig = getattr(obj, meth)

    def wrapped(*a, **k):
        prev, rec.ctx = rec.ctx, ctx
        try:
            return orig(*a, **k)
        finally:
            rec.ctx = prev
    setattr(obj, meth, wrapped)


def env_of(kind):
    from ratinabox.Environment import Environment
    if kind == "periodic":
        return Environment({"boundary_conditions": "periodic"})
    if kind == "holed":
        return Environment(HOLED)
    Env = Environment()
    if kind == "walls":
        for w in WALLS2:
            Env.add_wall(w)
    return Env


def state(A):
    return [np.array(A.pos, dtype=float), np.array(A.measured_velocity, dtype=float), float(A.measured_rotational_velocity),
            np.array(A.head_direction, dtype=float), float(A.distance_travelled), float(A.t)]


def run_case(out, key, env_kind, lead_params, subs, n_steps, seed):
    """subs: name -> (class name, params).  Records the lead and every SubAgent for n_steps steps."""
    from ratinabox.Agent import Agent
    import ratinabox.contribs.SubAgent as S
    np.random.seed(seed)
    rec = Recorder()
    rec.install()
    try:
        Env = env_of(env_kind)
        Lead = Agent(Env, lead_params)
        objs = {name: getattr(S, cls)(Lead, p) for name, (cls, p) in subs.items()}
        meta = {"env": env_kind, "lead_params": lead_params, "subs": subs,
                "lead_pos0": list(map(float, Lead.pos)), "lead_vel0": list(map(float, Lead.velocity)),
                "lead_hd0": list(map(float, Lead.head_direction)), "init": {}}
        for name, o in objs.items():
            meta["init"][name] = {"mv": list(map(float, o.measured_velocity)), "hd": list(map(float, o.head_direction))}
            if isinstance(o, S.ReplayAgent):
                sh = o.ReplayAgent
                meta["init"][name]["sham_mv"] = list(map(float, sh.measured_velocity))
                meta["init"][name]["sham_hd"] = list(map(float, sh.head_direction))
                meta["init"][name]["sham_dist"] = float(sh.distance_travelled)
                in_context(rec, sh, "update", name + ".sham")
                in_context(rec, sh, "initialise_position_and_velocity", name + ".init")
            in_context(rec, o, "update", name)
        samp = Env.sample_positions

        def sample_positions(*a, **k):
            p = samp(*a, **k)
            rec.log.append((rec.ctx, "sample", np.asarray(p, dtype=float).reshape(-1).tolist()))
            return p
        Env.sample_positions = sample_positions
        lead_rows, rows = [], {name: [] for name in objs}
        extra = {name: [] for name in objs}
        replays = {name: [] for name in objs}
        for s in range(n_steps):
            Lead.update()
            lead_rows.append([np.array(Lead.pos, dtype=float), np.array(Lead.velocity, dtype=float),
                              np.array(Lead.head_direction, dtype=float), float(Lead.t)])
            for name, o in objs.items():
                rec.log = []
                o.update()
                rows[name].append(state(o))
                if isinstance(o, S.DumbAgent):
                    xi = rec.take(name, "normal")
                    smp = rec.take(name, "sample")
                    extra[name].append((np.array(xi[0]), np.array(smp[-1]) if smp else np.full(2, np.nan),
                                        np.array(o.displacement, dtype=float)))
                elif isinstance(o, S.ReplayAgent):
                    u = rec.take(name, "uniform")
                    ray = rec.take(name, "rayleigh")
                    draws = np.full(6, np.nan)
                    if u:
                        draws[0] = u[0][0]
                    if ray:
                        draws[1], draws[2] = ray[0][0], ray[1][0]
                        smp = rec.take(name + ".init", "sample")
                        draws[3:5] = smp[-1]
                        draws[5] = rec.take(name + ".init", "uniform")[-1][0]
                        replays[name].append({"step": s, "normals": []})
                    sham_n = rec.take(name + ".sham", "normal")
                    if sham_n:
                        replays[name][-1]["normals"].extend(sum(sham_n, []))
                    extra[name].append((draws, bool(o.is_undergoing_replay), float(o.replay_speed),
                                        float(o.replay_duration), float(getattr(o, "replay_start_time", np.nan)),
                                        float(getattr(o, "replay_end_time", np.nan))))
                elif isinstance(o, S.UnrelatedAgent):
                    extra[name].append(np.array(sum(rec.take(name, "normal"), [])))
    finally:
        rec.remove()
    lp, lv, lhd, lt = (np.array(x) for x in zip(*lead_rows))
    out.update({f"{key}_lead_pos": lp, f"{key}_lead_vel": lv, f"{key}_lead_hd": lhd, f"{key}_lead_t": lt})
    for name, o in objs.items():
        p, mv, mr, hd, d, t = (np.array(x) for x in zip(*rows[name]))
        k = f"{key}_{name}"
        out.update({f"{k}_pos": p, f"{k}_mv": mv, f"{k}_mrot": mr, f"{k}_hd": hd, f"{k}_dist": d, f"{k}_t": t})
        if isinstance(o, S.DumbAgent):
            xi, rs, disp = (np.array(x) for x in zip(*extra[name]))
            out.update({f"{k}_xi": xi, f"{k}_resample": rs, f"{k}_disp": disp})
            meta["init"][name].update({"tau_v": o.tau_v, "sigma": o.sigma, "acceleration_scale": o.acceleration_scale})
        elif isinstance(o, S.ReplayAgent):
            draws, flag, sp, du, st, en = (np.array(x) for x in zip(*extra[name]))
            out.update({f"{k}_draws": draws, f"{k}_flag": flag, f"{k}_speed": sp, f"{k}_duration": du,
                        f"{k}_start": st, f"{k}_end": en})
            R = replays[name]
            K = max([len(r["normals"]) // 2 for r in R] + [1])
            xi = np.full((max(len(R), 1), K, 2), np.nan)
            for i, r in enumerate(R):
                xi[i, : len(r["normals"]) // 2] = np.array(r["normals"]).reshape(-1, 2)
            out.update({f"{k}_replay_start": np.array([r["step"] for r in R], dtype=np.int64), f"{k}_replay_xi": xi,
                        f"{k}_replay_len": np.array([len(r["normals"]) // 2 for r in R], dtype=np.int64)})
            meta["init"][name]["mean_replay_speed"] = o.mean_replay_speed
        elif isinstance(o, S.UnrelatedAgent):
            out[f"{k}_xi"] = np.array(extra[name])
    out[f"{key}_meta"] = np.array(json.dumps(meta))


CASES = {
    "open": ("open", {"dt": 0.01}, {"dumb": ("DumbAgent", {}), "shift": ("ShiftAgent", {"shift_m": 0.05}),
                                    "back": ("ShiftAgent", {"shift_m": -0.05}), "unrel": ("UnrelatedAgent", {}),
                                    "replay": ("ReplayAgent", {"replay_freq": 5.0})}, 600, 11),
    "walls": ("walls", {"dt": 0.01, "speed_mean": 0.5, "speed_std": 0.5},
              {"dumb": ("DumbAgent", {"drift_distance": 0.2}), "shift": ("ShiftAgent", {}),
               "replay": ("ReplayAgent", {"replay_freq": 5.0})}, 500, 12),
    "periodic": ("periodic", {"dt": 0.01, "speed_mean": 0.3, "speed_std": 0.3},
                 {"dumb": ("DumbAgent", {"drift_distance": 0.2}), "shift": ("ShiftAgent", {"shift_m": 0.1}),
                  "replay": ("ReplayAgent", {"replay_freq": 5.0})}, 400, 13),
    "holed": ("holed", {"dt": 0.01, "speed_mean": 0.2, "speed_std": 0.2},
              {"dumb": ("DumbAgent", {"drift_distance": 0.3, "drift_timescale": 1.0}),
               "replay": ("ReplayAgent", {"replay_freq": 5.0})}, 400, 14),
    "fast": ("open", {"dt": 0.01}, {"replay": ("ReplayAgent", {"replay_freq": 5.0, "replay_speed": 3.0})}, 400, 15),
}


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    import ratinabox.contribs.SubAgent as S
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    out = {}
    out["default_params_json"] = np.array(json.dumps({c: getattr(S, c).default_params for c in
                                                      ("DumbAgent", "ReplayAgent", "ShiftAgent", "UnrelatedAgent")},
                                                     sort_keys=True))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for key, (env_kind, lead_params, subs, n, seed) in CASES.items():
            run_case(out, key, env_kind, lead_params, subs, n, seed)
        out["cases_json"] = np.array(json.dumps(list(CASES)))
        D = S.DumbAgent(Agent(Environment(), {"dt": 0.01}), {"drift_distance": 0.1, "drift_timescale": 2.0})
        out["derived_json"] = np.array(json.dumps({"tau_v": D.tau_v, "sigma": D.sigma,
                                                   "acceleration_scale": D.acceleration_scale}))
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        S.DumbAgent(Agent(Environment(), {"dt": 0.01}), {"dt": 0.005})
    out["dt_warning"] = np.array([str(x.message) for x in w if "dt" in str(x.message)][0])
    np.savez_compressed(os.path.join(GOLD, "subagents.npz"), **out)
    print("subagents.npz", os.path.getsize(os.path.join(GOLD, "subagents.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()

"""TEST INFRASTRUCTURE -- write tests/golden/tsa.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): ratinabox/contribs/SubAgent.py, ThetaSequenceAgent.

    python oracle/gen_tsa_golden.py

Cases (geometry jitter off, as in gen_pppc_golden.py):
  * native runs, dt = 0.01 s: an open box (900 steps, past the 781-row look-behind window), a box with two inner walls
    with a fast lead (long eager rollouts), the ThetaSequenceAgent's own speed_mean and a forward_agent_update_kwargs (1100 steps: the stash's
    counter wraps at keep_count = 1000), and a periodic box (500 steps).  Per step: the lead's state after its update
    (pos, velocity, rotational velocity, distance travelled, t), theta_phase, and the ThetaSequenceAgent's pos, measured
    velocity / rotational velocity, head direction, distance travelled and t.  Per forward rollout: the step index it
    started at, the standard normals of its OU draws, and its first FWD_KEEP positions and distances.
  * replays of a hand-made lead (its state assigned before each ThetaSequenceAgent.update) whose LAST step makes the
    reference raise: a slow lead (look-behind target before the window), a gap in the lead's distances (idx < 3), and a
    lead distance edited up / down during a look-ahead.  The exception's type and text are recorded.
  * the two constructor asserts and the dt warning, as text.
"""
import contextlib
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
FWD_KEEP = 16          # rollout samples kept per rollout (a sweep's look-ahead reaches a few of them)
WALLS2 = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]


class Recorder:
    """np.random.normal with geometry jitter off; the forward agent's standard normals recorded per rollout."""

    def __init__(self):
        self.orig = np.random.normal
        self.active = False
        self.rollouts = []

    def normal(self, loc=0.0, scale=1.0, size=None):
        if scale in (1e-9, 1e-6):
            return np.zeros(size)
        g = self.orig(loc=0.0, scale=1.0, size=size)
        if self.active:
            self.rollouts[-1].extend(np.asarray(g, dtype=float).reshape(-1).tolist())
        return loc + scale * g


@contextlib.contextmanager
def recording(TSA, rec):
    """Patch np.random.normal, and mark the forward agent's updates (one rollout per first look-ahead step)."""
    fwd = TSA.ForwardSequenceAgent
    orig_update = fwd.update
    state = {"last": 0}

    def update(*a, **k):
        rec.active = True
        try:
            return orig_update(*a, **k)
        finally:
            rec.active = False

    fwd.update = update
    np.random.normal = rec.normal
    try:
        yield state
    finally:
        np.random.normal = rec.orig
        fwd.update = orig_update


def env_of(kind):
    from ratinabox.Environment import Environment
    if kind == "periodic":
        return Environment({"boundary_conditions": "periodic"})
    Env = Environment()
    if kind == "walls":
        for w in WALLS2:
            Env.add_wall(w)
    return Env


def lead_state(Ag):
    return (np.array(Ag.pos, dtype=float), np.array(Ag.velocity, dtype=float), float(Ag.rotational_velocity),
            float(Ag.distance_travelled), float(Ag.t))


def tsa_state(T):
    return (np.array(T.pos, dtype=float), np.array(T.measured_velocity, dtype=float), float(T.measured_rotational_velocity),
            np.array(T.head_direction, dtype=float), float(T.distance_travelled), float(T.t))


def save_run(out, key, rows, trows, phases, raised, rec, roll_start, roll_paths, meta):
    lp, lv, lr, ld, lt = (np.array(x) for x in zip(*rows))
    out.update({f"{key}_lead_pos": lp, f"{key}_lead_vel": lv, f"{key}_lead_rot": lr, f"{key}_lead_dist": ld,
                f"{key}_lead_t": lt, f"{key}_phase": np.array(phases), f"{key}_raised": np.array(raised)})
    tp, tmv, tmr, thd, tdist, tt = (np.array(x) for x in zip(*trows))
    out.update({f"{key}_tsa_pos": tp, f"{key}_tsa_mv": tmv, f"{key}_tsa_mrot": tmr, f"{key}_tsa_hd": thd,
                f"{key}_tsa_dist": tdist, f"{key}_tsa_t": tt})
    K = max([len(r) // 2 for r in rec.rollouts] + [1])
    xi = np.full((len(rec.rollouts), K, 2), np.nan)
    for i, r in enumerate(rec.rollouts):
        xi[i, : len(r) // 2] = np.array(r).reshape(-1, 2)
    P = FWD_KEEP
    fd = np.full((len(roll_paths), P), np.nan)
    fp = np.full((len(roll_paths), P, 2), np.nan)
    for i, (d, p) in enumerate(roll_paths):
        fd[i, : min(len(d), P)], fp[i, : min(len(d), P)] = d[:P], p[:P]
    out.update({f"{key}_fwd_xi": xi, f"{key}_fwd_start": np.array(roll_start, dtype=np.int64), f"{key}_fwd_dist": fd,
                f"{key}_fwd_pos": fp, f"{key}_meta": np.array(json.dumps(meta))})


def run_case(out, key, env_kind, lead_params, tsa_params, n_steps, seed, fwd_kwargs=None, script=None):
    """Native run (script None) or a replay of `script` rows (pos, dist, t) assigned to the lead before each update."""
    from ratinabox.Agent import Agent
    from ratinabox.contribs.SubAgent import ThetaSequenceAgent
    np.random.seed(seed)
    rec = Recorder()
    np.random.normal = rec.normal
    try:
        Env = env_of(env_kind)
        Ag = Agent(Env, lead_params)
        TSA = ThetaSequenceAgent(Ag, tsa_params)
    finally:
        np.random.normal = rec.orig
    meta = {"env": env_kind, "lead_params": lead_params, "tsa_params": tsa_params, "fwd_kwargs": fwd_kwargs or {},
            "avg_speed": float(Ag.average_measured_speed), "lead_pos0": list(map(float, Ag.pos)),
            "fwd_mv0": list(map(float, TSA.ForwardSequenceAgent.measured_velocity)),
            "fwd_hd0": list(map(float, TSA.ForwardSequenceAgent.head_direction)), "error": ""}
    rows, trows, phases, raised, roll_start, roll_paths = [], [], [], [], [], []
    with recording(TSA, rec):
        for s in range(n_steps):
            if script is None:
                Ag.update()
            else:
                p, d, t = script[s]
                Ag.pos, Ag.distance_travelled, Ag.t = np.array(p, dtype=float), float(d), float(t)
                Ag.history["distance_travelled"].append(float(d))
            rows.append(lead_state(Ag))
            phase = (Ag.t % (1 / TSA.theta_freq)) / ((1 / TSA.theta_freq))
            phases.append(phase)
            first = phase >= 0.5 and TSA.last_theta_phase < 0.5 and phase < 0.5 + TSA.theta_frac / 2
            if first:
                rec.rollouts.append([])
                roll_start.append(s)
            try:
                TSA.update(forward_agent_update_kwargs=fwd_kwargs or {})
            except Exception as e:          # the reference raises: the last step of a replay
                assert script is not None and s == n_steps - 1, f"{key}: step {s} raised {e!r}"
                meta["error"] = f"{type(e).__name__}:{e}"
                raised.append(True)
                trows.append((np.full(2, np.nan), np.full(2, np.nan), np.nan, np.full(2, np.nan), np.nan, np.nan))
                break
            raised.append(False)
            if first:                       # the eager rollout's samples, as interp1d holds them
                roll_paths.append((np.array(TSA.pos_interp.x), np.array(TSA.pos_interp.y)))
            trows.append(tsa_state(TSA))
    save_run(out, key, rows, trows, phases, raised, rec, roll_start, roll_paths, meta)
    return Ag, TSA


def line_script(dists, ts, y=0.5):
    return [((0.1 + 0.5 * d, y), d, t) for d, t in zip(dists, ts)]


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    out = {}
    from ratinabox.contribs.SubAgent import ThetaSequenceAgent
    out["default_params_json"] = np.array(json.dumps(ThetaSequenceAgent.default_params, sort_keys=True))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        run_case(out, "open", "open", {"dt": 0.01}, {}, 900, seed=3)
        run_case(out, "walls", "walls", {"dt": 0.01, "speed_mean": 0.5, "speed_std": 0.5}, {"speed_mean": 0.4}, 1100, seed=4,
                 fwd_kwargs={"thigmotaxis": 0.2})
        run_case(out, "periodic", "periodic", {"dt": 0.01, "speed_mean": 0.3, "speed_std": 0.3}, {"speed_mean": 0.3}, 500,
                 seed=5)

        # ---- replays whose last step raises.  Lead t: 0.1 k + 0.01 (phase 0.1, before the sweep) until the last step.
        n = 12
        pre = [0.1 * k + 0.01 for k in range(1, n)]
        # slow lead: the look-behind target (phase 0.3: 0.1 m back) precedes every recorded distance
        d = [0.2 + 1e-4 * k for k in range(n)]
        run_case(out, "slow", "open", {"dt": 0.01}, {}, n, seed=6, script=line_script(d, pre + [0.1 * n + 0.03]))
        # a gap in the distances: the target falls between rows 1 and 2 of the window (idx < 3, empty slice)
        d = [0.20, 0.21] + [0.40 + 1e-3 * k for k in range(n - 2)]
        run_case(out, "gap", "open", {"dt": 0.01}, {}, n, seed=7, script=line_script(d, pre + [0.1 * n + 0.03]))
        # look ahead: the lead's distance edited up (query past the rollout's end) / down (before its start)
        for key, jump in (("ahead_up", 1.0), ("ahead_down", -0.5)):
            ts = pre[:-1] + [0.1 * (n - 1) + 0.05, 0.1 * (n - 1) + 0.06]
            d = [0.2 + 0.004 * k for k in range(n)]
            d[-1] += jump
            run_case(out, key, "open", {"dt": 0.01}, {}, n, seed=8, script=line_script(d, ts))

    # ---- asserts and the dt warning
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    for key, lead_p, p in (("assert_dt", {"dt": 0.02}, {}), ("assert_v", {"dt": 0.01}, {"v_sequence": 0.1})):
        try:
            ThetaSequenceAgent(Agent(Environment(), lead_p), p)
            out[key] = np.array("")
        except AssertionError as e:
            out[key] = np.array(str(e))
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        ThetaSequenceAgent(Agent(Environment(), {"dt": 0.01}), {"dt": 0.005})
    out["dt_warning"] = np.array([str(x.message) for x in w if "dt" in str(x.message)][0])
    np.savez_compressed(os.path.join(GOLD, "tsa.npz"), **out)
    print("tsa.npz", os.path.getsize(os.path.join(GOLD, "tsa.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()

"""DumbAgent, ShiftAgent, ReplayAgent and UnrelatedAgent on the device (ratinabox_b200.contribs) against the live
reference's fixture (tests/golden/subagents.npz, teacher-forced), the NumPy restatement (oracle/riab_oracle_subagents.py)
on the device's Philox draws, statistics of the replay draws, the DumbAgent's wall invariant, sharding, populations and
history rings.  GPU only."""
import numpy as np
import pytest

from riab_oracle_subagents import OracleDumb, OracleReplay
import philox_np
from test_gpu_theta_sequence import HOLED, TOL, _close, _env
from test_oracle_subagents import CASES, G, meta, oracle_env

pytestmark = pytest.mark.gpu

CLASSES = ("DumbAgent", "ShiftAgent", "ReplayAgent", "UnrelatedAgent")


def _classes():
    from ratinabox_b200 import contribs
    return {c: getattr(contribs, c) for c in CLASSES}


@pytest.mark.parametrize("case", CASES)
def test_teacher_forced_against_the_reference(case):
    """The lead's recorded state is assigned before every update and the reference's draws are injected: DumbAgent and
    ShiftAgent positions bit for bit, ReplayAgent positions within 1e-12 m with identical flags and replay times, the
    UnrelatedAgent's within 1e-12 m, and every SubAgent's own state within the forced-step tolerances."""
    import ratinabox_b200 as rb
    cls = _classes()
    m = meta(case)
    Lead = rb.Agent(_env(rb, m["env"]), m["lead_params"])
    Lead.pos, Lead.velocity = np.array(m["lead_pos0"]), np.array(m["lead_vel0"])
    subs = {}
    for name, (c, p) in m["subs"].items():
        o = cls[c](Lead, p)
        o.measured_velocity, o.head_direction = np.array(m["init"][name]["mv"]), np.array(m["init"][name]["hd"])
        if c == "ReplayAgent":
            o._sham["measured_velocity"].copy_(o._sham["measured_velocity"].new_tensor(m["init"][name]["sham_mv"])[None])
            o._sham["head_direction"].copy_(o._sham["head_direction"].new_tensor(m["init"][name]["sham_hd"])[None])
        subs[name] = o
    r = {name: -1 for name in subs}
    for s in range(len(G[f"{case}_lead_t"])):
        Lead.pos, Lead.velocity = G[f"{case}_lead_pos"][s], G[f"{case}_lead_vel"][s]
        Lead.head_direction, Lead.t = G[f"{case}_lead_hd"][s], float(G[f"{case}_lead_t"][s])
        for name, o in subs.items():
            k, c = f"{case}_{name}", m["subs"][name][0]
            if c == "DumbAgent":
                o.update(_xi_displacement=G[f"{k}_xi"][s][None], _resample_pos=G[f"{k}_resample"][s][None])
                assert np.array_equal(o.pos, G[f"{k}_pos"][s]), (k, s)
                assert np.array_equal(o.displacement, G[f"{k}_disp"][s]), (k, s)
            elif c == "ShiftAgent":
                o.update()
                assert np.array_equal(o.pos, G[f"{k}_pos"][s]), (k, s)
            elif c == "ReplayAgent":
                starts = list(G[f"{k}_replay_start"])
                if s in starts:
                    r[name] = starts.index(s)
                kw = {"_xi_replay": np.nan_to_num(G[f"{k}_replay_xi"][r[name]])[None]} if r[name] >= 0 else {}
                o.update(_replay_draws=G[f"{k}_draws"][s][None], **kw)
                _close(o.pos, G[f"{k}_pos"][s], 1e-12, f"{k} step {s}: pos")
                assert o.is_undergoing_replay == G[f"{k}_flag"][s], (k, s)
                got = [o.replay_speed, o.replay_duration, o.replay_start_time, o.replay_end_time]
                want = [G[f"{k}_{f}"][s] for f in ("speed", "duration", "start", "end")]
                assert np.array_equal(got, want, equal_nan=True), (k, s, got, want)
            else:
                o.update(_xi=G[f"{k}_xi"][s][None])
                _close(o.pos, G[f"{k}_pos"][s], 1e-12, f"{k} step {s}: pos")
            if s > 0:
                _close(o.measured_velocity, G[f"{k}_mv"][s], TOL["measured_velocity"], f"{k} step {s}: mv")
                _close(o.measured_rotational_velocity, G[f"{k}_mrot"][s], TOL["measured_rotational_velocity"],
                       f"{k} step {s}: mrot")
                _close(o.head_direction, G[f"{k}_hd"][s], TOL["head_direction"], f"{k} step {s}: hd")
            _close(o.distance_travelled, G[f"{k}_dist"][s], 1e-9, f"{k} step {s}: distance")
            assert o.t == G[f"{k}_t"][s]
    for name, (c, _) in m["subs"].items():
        if c == "ReplayAgent":
            assert np.array_equal(subs[name].history["replay"], G[f"{case}_{name}_flag"])


def _uniforms(seed, agents, sub, step, stream):
    r = philox_np.philox4x32(philox_np.counter(agents, sub, step, stream), (seed & 0xFFFFFFFF, seed >> 32))
    return philox_np.u01_53(r[..., 0], r[..., 1]), philox_np.u01_53(r[..., 2], r[..., 3])


def _normals(seed, agents, sub, step, stream):
    """philox_normals of riab_common.cuh for counter (agent, sub, step, stream), as philox_np.agent_normals."""
    r = philox_np.philox4x32(philox_np.counter(agents, sub, step, stream), (seed & 0xFFFFFFFF, seed >> 32))
    f32 = np.float32
    u1 = (r[..., 0].astype(f32).astype(np.float64) * 2.0 ** -32 + 2.0 ** -33).astype(f32)
    u2 = (r[..., 2].astype(f32) * f32(2.0 ** -32)).astype(f32)
    rad = np.sqrt(f32(-2.0) * np.log(u1)).astype(f32)
    ang = (f32(2.0) * u2).astype(np.float64) * np.pi
    return np.stack(((rad * np.cos(ang).astype(f32)).astype(np.float64),
                     (rad * np.sin(ang).astype(f32)).astype(np.float64)), axis=-1)


def _replay_draws(seed, agent, step, mean_speed, mean_duration, ext):
    """The ReplayAgent's Philox draws of one (agent, update) in the tap's layout (rectangular environment)."""
    a = np.array([agent], dtype=np.uint64)
    u, us = _uniforms(seed, a, 0, step, 7)
    ud, udir = _uniforms(seed, a, 1, step, 7)
    ux, uy = _uniforms(seed, a, 2, step, 7)
    return np.array([u[0], mean_speed * np.sqrt(-2.0 * np.log(1.0 - us[0])),
                     mean_duration * np.sqrt(-2.0 * np.log(1.0 - ud[0])), ext[0] + (ext[1] - ext[0]) * ux[0],
                     ext[2] + (ext[3] - ext[2]) * uy[0], 2 * np.pi * udir[0]])


def test_philox_draws_against_the_oracle():
    """1 024 agents on the device's Philox draws; the oracle, fed the NumPy mirror of the same streams, for a sample of
    agents: replay decisions and flags identical, DumbAgent and ReplayAgent positions within 1e-5 m (the float32
    Box-Muller normals agree to a few ulps)."""
    import ratinabox_b200 as rb
    from ratinabox_b200.contribs import DumbAgent, ReplayAgent
    A, T, sample = 1024, 300, np.array([0, 3, 100, 513, 1023])
    np.random.seed(5)
    Lead = rb.Agent(_env(rb, "walls"), {"dt": 0.01, "n_agents": A, "seed": 2, "speed_mean": 0.3, "speed_std": 0.3})
    D = DumbAgent(Lead, {"seed": 21, "drift_distance": 0.2})
    R = ReplayAgent(Lead, {"seed": 22, "replay_freq": 5.0})
    env = oracle_env("walls")
    sham = R._sham
    od = [OracleDumb(env, {"drift_distance": 0.2}) for _ in sample]
    orr = [OracleReplay(env, {"replay_freq": 5.0}, 0.01, (sham["measured_velocity"][a].cpu().numpy(),
                                                         sham["head_direction"][a].cpu().numpy(), 0.0)) for a in sample]
    idx = np.zeros(len(sample), dtype=int)
    worst_d = worst_r = 0.0
    n_rep = 0
    for s in range(T):
        Lead.update()
        lp, lt = Lead.pos[sample], Lead.t
        D.update(); R.update()
        dp, rp, flags = D.pos[sample], R.pos[sample], R.is_undergoing_replay[sample]
        for j, a in enumerate(sample):
            ag = np.array([a], dtype=np.uint64)
            want = od[j].step(lp[j], 0.01, _normals(21, ag, 0, s, 6)[0])
            worst_d = max(worst_d, float(np.abs(want - dp[j]).max()))
            was = orr[j].is_undergoing_replay
            draws = _replay_draws(22, a, s, 1.0, 0.1, env.extent)
            xi = _normals(22, np.full(4096, a, dtype=np.uint64), idx[j], np.arange(4096), 8) if not was else None
            want = orr[j].step(lp[j], lt, draws, xi)
            if not was and orr[j].is_undergoing_replay:
                idx[j] += 1
                n_rep += 1
            assert orr[j].is_undergoing_replay == flags[j], (s, a)
            if np.isfinite(want).all():
                worst_r = max(worst_r, float(np.abs(want - rp[j]).max()))
    assert n_rep > 5
    assert worst_d <= 1e-5 and worst_r <= 1e-5, (worst_d, worst_r)


def test_replay_statistics():
    """65 536 agents with production draws: the start rate per tracking step is replay_freq dt, the mean replay_speed is
    mean sqrt(pi / 2), the share of durations clamped to mean / 2 is 1 - exp(-1/8); each within 5 sigma.  In the holed
    polygon every replay starts inside the environment."""
    import ratinabox_b200 as rb
    from ratinabox_b200.contribs import ReplayAgent
    A = 65536
    Lead = rb.Agent(rb.Environment(HOLED), {"dt": 0.01, "n_agents": A, "save_history": False})
    R = ReplayAgent(Lead, {"replay_freq": 5.0, "save_history": False, "seed": 3})
    E = rb.Environment(HOLED)
    tracking = starts = 0
    speeds, durs = [], []
    for _ in range(40):
        Lead.update()
        was = R.is_undergoing_replay
        R.update()
        now = R.is_undergoing_replay
        new = ~was & now
        tracking += int((~was).sum())
        starts += int(new.sum())
        speeds.append(R.replay_speed[new]); durs.append(R.replay_duration[new])
        p = R.pos[new]
        assert all(E.check_if_position_is_in_environment(q) for q in p[:2000])
    p = 5.0 * 0.01
    assert abs(starts - p * tracking) <= 5 * np.sqrt(tracking * p * (1 - p))
    sp, du = np.concatenate(speeds), np.concatenate(durs)
    assert abs(sp.mean() - np.sqrt(np.pi / 2)) <= 5 * np.sqrt((4 - np.pi) / 2 / len(sp))
    q = 1 - np.exp(-1 / 8)
    frac = np.mean(du == 0.05)
    assert abs(frac - q) <= 5 * np.sqrt(q * (1 - q) / len(du))


def test_dumb_agent_never_crosses_a_wall():
    """The two-wall box, 500 steps, 4 096 agents with drift_distance 0.2: no segment from the lead's position to the
    DumbAgent's strictly crosses any wall."""
    import ratinabox_b200 as rb
    from ratinabox_b200.contribs import DumbAgent
    A = 4096
    Lead = rb.Agent(_env(rb, "walls"), {"dt": 0.01, "n_agents": A, "speed_mean": 0.5, "speed_std": 0.5,
                                        "save_history": False})
    D = DumbAgent(Lead, {"drift_distance": 0.2, "save_history": False})
    walls = oracle_env("walls").walls
    a0, sa = walls[:, 0][None], (walls[:, 1] - walls[:, 0])[None]
    for _ in range(500):
        Lead.update(); D.update()
        lp, dp = Lead.pos, D.pos
        d0 = (lp[:, None] - a0)
        sb = (dp - lp)[:, None]
        den_a = sa[..., 0] * -sb[..., 1] + sa[..., 1] * sb[..., 0]
        la = (d0[..., 0] * -sb[..., 1] + d0[..., 1] * sb[..., 0]) / np.where(den_a == 0, np.inf, den_a)
        den_b = sb[..., 0] * -sa[..., 1] + sb[..., 1] * sa[..., 0]
        lb = (-d0[..., 0] * -sa[..., 1] + -d0[..., 1] * sa[..., 0]) / np.where(den_b == 0, np.inf, den_b)
        assert not ((la > 0) & (la < 1) & (lb > 0) & (lb < 1)).any()


@pytest.mark.parametrize("kind", CLASSES)
def test_sharding_independence(kind):
    """Rows 4..7 of n_agents = 8 equal a shard of n_agents = 4 with id_offset = 4, bit for bit."""
    import ratinabox_b200 as rb
    cls = _classes()[kind]
    E = _env(rb, "walls")
    L8 = rb.Agent(E, {"dt": 0.01, "n_agents": 8, "seed": 3})
    L4 = rb.Agent(E, {"dt": 0.01, "n_agents": 4, "seed": 3, "id_offset": 4})
    for k in ("pos", "velocity", "rotational_velocity", "measured_velocity", "head_direction"):
        setattr(L4, k, getattr(L8, k)[4:])
    p = {"seed": 5, "replay_freq": 5.0} if kind == "ReplayAgent" else {"seed": 5}
    S8, S4 = cls(L8, p), cls(L4, p)
    for k in ("measured_velocity", "head_direction"):
        setattr(S4, k, getattr(S8, k)[4:])
    if kind == "ReplayAgent":
        for k in S8._sham:
            S4._sham[k].copy_(S8._sham[k][4:])
    for _ in range(200):
        L8.update(); L4.update()
        S8.update(); S4.update()
        assert np.array_equal(S8.pos[4:], S4.pos, equal_nan=True)
    if kind == "ReplayAgent":
        assert S8.history["replay"][:, 4:].any()


def test_populations_shapes_rings_and_run():
    """PlaceCells(SubAgent) agree with get_state(pos=...); n_agents = 1 has the reference's shapes; replay flags stay
    aligned with the position rows across a ring that doubles and a ring that wraps; run() raises."""
    import ratinabox_b200 as rb
    cls = _classes()
    Lead = rb.Agent(rb.Environment(), {"dt": 0.01, "n_agents": 64})
    subs = [cls["DumbAgent"](Lead), cls["ShiftAgent"](Lead), cls["ReplayAgent"](Lead, {"replay_freq": 5.0}),
            cls["UnrelatedAgent"](Lead)]
    pcs = [rb.PlaceCells(s, {"n": 40, "min_fr": 0.0, "max_fr": 1.0}) for s in subs]
    for _ in range(30):
        Lead.update()
        for s, pc in zip(subs, pcs):
            s.update(); pc.update()
            P = s.pos
            ok = np.isfinite(P[:, 0])
            assert np.abs(pc.firingrate[ok] - pc.get_state(evaluate_at=None, pos=P[ok]).T).max() <= 1e-6
    assert not np.array_equal(subs[3].pos, Lead.pos)
    for s in subs:
        with pytest.raises(NotImplementedError):
            s.run(3)
    Lead1 = rb.Agent(rb.Environment(), {"dt": 0.01})
    D1, R1 = cls["DumbAgent"](Lead1), cls["ReplayAgent"](Lead1, {"replay_freq": 5.0})
    for _ in range(20):
        Lead1.update(); D1.update(); R1.update()
    assert D1.pos.shape == (2,) and D1.displacement.shape == (2,) and D1.displacement_velocity.shape == (2,)
    assert R1.history["replay"].shape == (20,) and R1.history["replay"].dtype == bool
    assert isinstance(R1.is_undergoing_replay, bool) and isinstance(R1.replay_speed, float)
    with pytest.raises(AttributeError):
        R1.replay_speed = 2.0
    d = D1.displacement
    D1.displacement = d * 0.5                                  # assignment is uploaded before the next update
    assert np.array_equal(D1.displacement, d * 0.5)
    # rings: 1 024 rows double to 2 048; a 300-row byte limit wraps.  The flag row of step s must be the flag read
    # right after step s, and the position row the position read then.
    for limit, n in ((2 << 30, 1500), (300 * 8 * 4 * 3, 700)):
        L = rb.Agent(rb.Environment(), {"dt": 0.01, "n_agents": 3})
        R = cls["ReplayAgent"](L, {"replay_freq": 5.0, "history_bytes_limit": limit})
        flags, pos = [], []
        for _ in range(n):
            L.update(); R.update()
            flags.append(R.is_undergoing_replay.copy()); pos.append(R.pos.astype(np.float32))
        h = R.get_history_arrays()
        T = h["replay"].shape[0]
        assert T == min(n, R._hist_cap) and (limit != 2 << 30 or T == n)
        assert np.array_equal(h["replay"], np.array(flags[n - T:]))
        assert np.array_equal(h["pos"].astype(np.float32), np.array(pos[n - T:]))

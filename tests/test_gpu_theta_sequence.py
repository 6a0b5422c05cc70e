"""ThetaSequenceAgent on the device (ratinabox_b200.contribs.ThetaSequenceAgent) against the live reference's fixture
(tests/golden/tsa.npz, teacher-forced), the NumPy restatement (oracle/riab_oracle_tsa.py) on Philox normals, itself under
sharding, and through PlaceCells.  GPU only."""
import json
import os

import numpy as np
import pytest

import riab_oracle as O
from riab_oracle_tsa import OracleTSA
import philox_np
from test_oracle_tsa import G, REPLAYS, RUNS, WALLS2, replay

pytestmark = pytest.mark.gpu

# per step, as in test_gpu_trajectory.py: positions 1e-12 m; velocities are displacements / dt
TOL = {"pos": 1e-12, "measured_velocity": 1e-10, "measured_rotational_velocity": 1e-8, "head_direction": 1e-10,
       "distance_travelled": 1e-10}
HOLED = {"boundary": [[0, 0], [1.2, 0], [1.2, 0.4], [0.8, 1.0], [0, 1.0]],
         "holes": [[[0.4, 0.4], [0.6, 0.4], [0.6, 0.6], [0.4, 0.6]]]}


def _close(got, want, tol, what):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), what
    ok = ~np.isnan(want)
    if ok.any():
        err = np.abs(got[ok] - want[ok]).max()
        assert err <= tol, f"{what}: {err:.3e} > {tol:.1e}"


def _env(rb, kind):
    if kind == "periodic":
        return rb.Environment({"boundary_conditions": "periodic"})
    if kind == "holed":
        return rb.Environment(HOLED)
    E = rb.Environment()
    for w in (WALLS2 if kind == "walls" else ()):
        E.add_wall(w)
    return E


@pytest.mark.parametrize("key", RUNS + REPLAYS)
def test_teacher_forced_against_the_reference(key):
    """The lead's recorded state is assigned before every update and the forward rollouts take the recorded normals:
    positions within 1e-12 m with the reference's NaN mask where it returns, the oracle's defined position where it
    raises, and the ThetaSequenceAgent's own state within the forced-step tolerances."""
    import ratinabox_b200 as rb
    from ratinabox_b200.contribs import ThetaSequenceAgent
    m = json.loads(str(G[f"{key}_meta"]))
    Lead = rb.Agent(_env(rb, m["env"]), m["lead_params"])
    Lead.pos = np.array(m["lead_pos0"])
    TSA = ThetaSequenceAgent(Lead, m["tsa_params"])
    defined, _, _ = replay(key, "lazy")
    starts, xi = list(G[f"{key}_fwd_start"]), G[f"{key}_fwd_xi"]
    raised = G[f"{key}_raised"]
    r = -1
    for s in range(len(G[f"{key}_lead_t"])):
        Lead.pos, Lead.velocity = G[f"{key}_lead_pos"][s], G[f"{key}_lead_vel"][s]
        Lead.rotational_velocity, Lead.distance_travelled = G[f"{key}_lead_rot"][s], G[f"{key}_lead_dist"][s]
        Lead.t = float(G[f"{key}_lead_t"][s])
        if s in starts:
            r = starts.index(s)
        kw = {"_xi_forward": np.nan_to_num(xi[r])[None]} if r >= 0 else {}
        TSA.update(forward_agent_update_kwargs=m["fwd_kwargs"], **kw)
        if raised[s]:
            _close(TSA.pos, defined[s], 1e-12, f"{key} step {s}: defined position")
            continue
        _close(TSA.pos, G[f"{key}_tsa_pos"][s], TOL["pos"], f"{key} step {s}: pos")
        if s > 0:
            _close(TSA.measured_velocity, G[f"{key}_tsa_mv"][s], TOL["measured_velocity"], f"{key} step {s}: mv")
            _close(TSA.measured_rotational_velocity, G[f"{key}_tsa_mrot"][s], TOL["measured_rotational_velocity"],
                   f"{key} step {s}: mrot")
            _close(TSA.head_direction, G[f"{key}_tsa_hd"][s], TOL["head_direction"], f"{key} step {s}: hd")
        _close(TSA.distance_travelled, G[f"{key}_tsa_dist"][s], TOL["distance_travelled"], f"{key} step {s}: distance")
        assert TSA.t == G[f"{key}_tsa_t"][s]


def theta_fwd_normals(seed, rollout, k, agents):
    """riab_theta.cuh: theta_fwd_normals (Philox stream 5, sub-index = rollout, step = rollout step), Box-Muller as
    philox_np.agent_normals."""
    r = philox_np.philox4x32(philox_np.counter(agents, rollout, k, 5), (seed & 0xFFFFFFFF, seed >> 32))
    f32 = np.float32
    u1 = (r[..., 0].astype(f32).astype(np.float64) * 2.0 ** -32 + 2.0 ** -33).astype(f32)
    u2 = (r[..., 2].astype(f32) * f32(2.0 ** -32)).astype(f32)
    rad = np.sqrt(f32(-2.0) * np.log(u1)).astype(f32)
    ang = (f32(2.0) * u2).astype(np.float64) * np.pi
    return np.stack(((rad * np.cos(ang).astype(f32)).astype(np.float64),
                     (rad * np.sin(ang).astype(f32)).astype(np.float64)), axis=-1)


def _philox_run(kind, A, n_steps, sample, oenv, lead_params=None, seed=0):
    import ratinabox_b200 as rb
    from ratinabox_b200.contribs import ThetaSequenceAgent
    np.random.seed(seed)
    lp = {"dt": 0.01, "n_agents": A, "seed": 7, **(lead_params or {})}
    Lead = rb.Agent(_env(rb, kind), lp)
    TSA = ThetaSequenceAgent(Lead, {"seed": 9})
    oras = [OracleTSA(oenv, {}, 0.01, Lead.speed_mean, Lead.average_measured_speed, None) for _ in sample]
    rollout, worst, nan_diff, finite = -1, 0.0, 0, 0
    for s in range(n_steps):
        Lead.update()
        pos, vel, rot = Lead.pos[sample], Lead.velocity[sample], Lead.rotational_velocity[sample]
        dist, t = Lead.distance_travelled[sample], Lead.t
        phase = (t % 0.1) / 0.1
        if phase >= 0.5 and TSA.last_theta_phase < 0.5 and phase < 0.75:
            rollout += 1
        TSA.update()
        got = TSA.pos[sample]
        for j, a in enumerate(sample):
            xi = theta_fwd_normals(9, max(rollout, 0), np.arange(64), np.full(64, a, dtype=np.uint64))
            want, _ = oras[j].step(pos[j], vel[j], rot[j], dist[j], t, xi)
            ok = ~np.isnan(want) & ~np.isnan(got[j])
            nan_diff += int(np.isnan(want[0]) != np.isnan(got[j][0]))
            finite += int(ok.all())
            if ok.any():
                worst = max(worst, float(np.abs(got[j][ok] - want[ok]).max()))
    return worst, nan_diff, finite, TSA


def test_philox_batch_against_the_oracle():
    """4 096 agents on the device's Philox forward normals against the oracle fed the NumPy mirror of the same draws for a
    sample of agents, over 30 theta cycles.  The draws agree up to the last float32 ulps of the Box-Muller transform; a
    rollout step lasts dt' = 0.625 s, where the rotational noise is about 8 rad per unit normal, so those ulps reach the
    positions as a few 1e-6 m."""
    sample = np.array([0, 1, 2, 17, 1000, 2049, 4095])
    worst, nan_diff, finite, _ = _philox_run("open", 4096, 300, sample, O.OracleEnvironment())
    assert finite > 0.3 * 300 * len(sample)
    assert nan_diff <= 2 and worst <= 1e-5, (nan_diff, worst)


def test_polygon_with_a_hole():
    """A polygon boundary with a hole: forward rollouts bounce off its walls like the oracle's."""
    sample = np.array([0, 5, 77, 200, 255])
    oenv = O.OracleEnvironment(boundary=HOLED["boundary"], holes=HOLED["holes"])
    worst, nan_diff, finite, TSA = _philox_run("holed", 256, 300, sample, oenv, {"speed_mean": 0.2, "speed_std": 0.2})
    assert finite > 0.3 * 300 * len(sample)
    assert nan_diff <= 2 and worst <= 1e-5, (nan_diff, worst)


def test_sharding_independence():
    """Rows 4..7 of n_agents = 8 equal a shard of n_agents = 4 with id_offset = 4, bit for bit."""
    import ratinabox_b200 as rb
    from ratinabox_b200.contribs import ThetaSequenceAgent
    E = _env(rb, "walls")
    L8 = rb.Agent(E, {"dt": 0.01, "n_agents": 8, "seed": 3})
    L4 = rb.Agent(E, {"dt": 0.01, "n_agents": 4, "seed": 3, "id_offset": 4})
    for k in ("pos", "velocity", "rotational_velocity", "measured_velocity", "head_direction"):
        setattr(L4, k, getattr(L8, k)[4:])
    T8, T4 = ThetaSequenceAgent(L8, {"seed": 5}), ThetaSequenceAgent(L4, {"seed": 5})
    seen = 0
    for _ in range(250):
        L8.update(); L4.update()
        T8.update(); T4.update()
        a, b = T8.pos[4:], T4.pos
        assert np.array_equal(a, b, equal_nan=True)
        seen += int(np.isfinite(b).all())
    assert seen > 50


def test_place_cells_on_the_sweep_and_one_agent_shapes():
    """PlaceCells(TSA): zero rates on NaN steps, get_state(pos=...) elsewhere; n_agents = 1 has the reference's shapes."""
    import ratinabox_b200 as rb
    from ratinabox_b200.contribs import ThetaSequenceAgent
    Lead = rb.Agent(rb.Environment(), {"dt": 0.01, "n_agents": 64})
    TSA = ThetaSequenceAgent(Lead)
    PCs = rb.PlaceCells(TSA, {"n": 50, "min_fr": 0.0, "max_fr": 1.0})
    n_nan = n_fin = 0
    for _ in range(60):
        Lead.update(); TSA.update(); PCs.update()
        P, fr = TSA.pos, PCs.firingrate
        bad = np.isnan(P[:, 0])
        assert np.all(fr[bad] == 0)
        if (~bad).any():
            want = PCs.get_state(evaluate_at=None, pos=P[~bad]).T
            assert np.abs(fr[~bad] - want).max() <= 1e-6
        n_nan += int(bad.sum()); n_fin += int((~bad).sum())
    assert n_nan > 0 and n_fin > 0
    Lead1 = rb.Agent(rb.Environment(), {"dt": 0.01})
    T1 = ThetaSequenceAgent(Lead1)
    P1 = rb.PlaceCells(T1, {"n": 7})
    for _ in range(30):
        Lead1.update(); T1.update(); P1.update()
    assert T1.pos.shape == (2,) and P1.firingrate.shape == (7,)
    assert T1.history["pos"].shape == (30, 2)
    assert abs(T1.t - (Lead1.t + 0.01)) < 1e-12            # one dt ahead of the lead, as in the reference


def test_errors():
    import ratinabox_b200 as rb
    from ratinabox_b200.contribs import ThetaSequenceAgent
    with pytest.raises(AssertionError, match=r"params\['dt'\] for the LeadAgent is too large"):
        ThetaSequenceAgent(rb.Agent(rb.Environment(), {"dt": 0.02}))
    with pytest.raises(AssertionError, match=r"params\['v_sequence'\] is too small"):
        ThetaSequenceAgent(rb.Agent(rb.Environment(), {"dt": 0.01}), {"v_sequence": 0.1})
    with pytest.warns(UserWarning, match="overwritten to match dt of the LeadAgent"):
        ThetaSequenceAgent(rb.Agent(rb.Environment(), {"dt": 0.01}), {"dt": 0.005})
    Lead = rb.Agent(rb.Environment(), {"dt": 0.01, "n_agents": 16})
    TSA = ThetaSequenceAgent(Lead)
    with pytest.raises(NotImplementedError):
        TSA.run(3)
    with pytest.raises(NotImplementedError):
        TSA.update(forward_agent_update_kwargs={"drift_velocity": np.zeros(2)})
    with pytest.raises(MemoryError):           # a look-behind ring of 6e10 lead steps
        ThetaSequenceAgent(rb.Agent(rb.Environment(), {"dt": 0.01, "speed_mean": 1e-9, "speed_std": 1e-9}))
    assert Lead.distance_travelled.shape == (16,) and np.all(Lead.distance_travelled == 0)

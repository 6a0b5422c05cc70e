"""Imported and forced trajectories on the device (Agent.import_trajectory, Agent.update(forced_next_position=...),
Agent.run following a trajectory) against the NumPy mirror of the spline (tests/spline_np.py), the live reference's
fixture (tests/golden/traj.npz), the float64 oracle (oracle/riab_oracle_traj.py) and each other's launch paths.  GPU only.
"""
import numpy as np
import pytest

import riab_oracle as O
import riab_oracle_traj as OT
import spline_np
from test_gpu_launch_paths import assert_same, check_spikes

pytestmark = pytest.mark.gpu

STATE = ("pos", "velocity", "rotational_velocity", "measured_velocity", "measured_rotational_velocity",
         "head_direction", "distance_travelled")
# per step, against the reference / oracle: positions 1e-12 m; velocities are displacements / dt, the rotational velocity
# an angle / dt (the device takes atan2 of the cross and dot products instead of two get_angle calls)
TOL = {"pos": 1e-12, "velocity": 1e-10, "measured_velocity": 1e-10, "rotational_velocity": 1e-8,
       "measured_rotational_velocity": 1e-8, "head_direction": 1e-10, "distance_travelled": 1e-10, "t": 0.0}
RATE_TOL = 1e-5


def _close(got, want, tol, what):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), what
    ok = ~np.isnan(want)
    if ok.any():
        err = np.abs(got[ok] - want[ok]).max()
        assert err <= tol, f"{what}: {err:.3e} > {tol:.1e}"


def _agent(rb, g, case, env, dt, n_agents=1):
    Ag = rb.Agent(env, {"dt": dt, "n_agents": n_agents})
    for k in STATE:
        setattr(Ag, k, g[f"{case}_s0_{k}"])
    Ag.t = float(g[f"{case}_s0_t"])
    return Ag


def _pops(rb, g, case, Ag):
    pc = rb.PlaceCells(Ag, {"place_cell_centres": g[f"{case}_pc_centres"], "widths": 0.2, "wall_geometry": "line_of_sight",
                            "min_fr": 0.0, "max_fr": 1.0})
    gc = rb.GridCells(Ag, {"gridscale": g[f"{case}_gc_gridscales"], "orientation": g[f"{case}_gc_orientations"],
                           "phase_offset": g[f"{case}_gc_phase_offsets"], "min_fr": 0.0, "max_fr": 1.0})
    fov = rb.FieldOfViewBVCs(Ag, {"min_fr": 0.0, "max_fr": 2.0})
    return {"pc": (pc, 1.0), "gc": (gc, 1.0), "fov": (fov, 2.0)}


def _box(rb, g):
    E = rb.Environment()
    for w in g["box_walls"]:
        E.add_wall(w)
    return E


@pytest.mark.parametrize("per_agent", [False, True])
def test_device_spline_equals_the_mirror_bit_for_bit(per_agent):
    import ratinabox_b200 as rb
    rng = np.random.default_rng(3)
    A, T = 5, 700
    times = np.concatenate([[0.0], np.cumsum(rng.uniform(0.001, 0.5, T - 1))]) + 2.0
    pos = rng.uniform(-3, 3, (A, T, 2) if per_agent else (T, 2))
    Ag = rb.Agent(rb.Environment({"scale": 8.0}), {"n_agents": A})
    Ag.import_trajectory(times=times, positions=pos)
    x = times - times.min()
    y = pos.transpose(1, 0, 2) if per_agent else pos[:, None, :]
    M = Ag._traj["M"].cpu().numpy()
    assert np.array_equal(Ag._traj["times"].cpu().numpy(), x)
    assert np.array_equal(M, spline_np.build(x, y))
    assert np.array_equal(Ag.pos, np.broadcast_to(y[0], (A, 2)))


@pytest.mark.parametrize("case,dt", [("syn", 0.05), ("sar", 0.1)])
def test_imported_against_the_reference(golden, case, dt):
    """Stepped update() + Neurons.update() along an imported trajectory (syn: 40 irregular samples run past t_max, in a
    box with two walls, with line-of-sight PlaceCells, GridCells and egocentric FieldOfViewBVCs; sar: a sargolini slice
    imported at t != 0), then the same from the same state with Ag.run()."""
    import ratinabox_b200 as rb
    g = golden("traj.npz")
    env = _box(rb, g) if case == "syn" else rb.Environment()
    Ag = _agent(rb, g, case, env, dt)
    pops = _pops(rb, g, case, Ag) if case == "syn" else {}
    Ag.import_trajectory(times=g[f"{case}_times"], positions=g[f"{case}_positions"])
    _close(Ag.pos, g[f"{case}_s0_pos"], 1e-15, "pos at import")
    n = g[f"{case}_t"].shape[0]
    for i in range(n):
        Ag.update()
        for N, _ in pops.values():
            N.update()
        for k in STATE:
            _close(getattr(Ag, k), g[f"{case}_{k}"][i], TOL[k], f"{case} step {i} {k}")
        assert Ag.t == g[f"{case}_t"][i]
        for name, (N, scale) in pops.items():
            _close(N.firingrate, g[f"{case}_rates_{name}"][i], RATE_TOL * scale, f"{case} step {i} {name}")
    h = Ag.get_history_arrays()
    _close(h["pos"][-n:], g[f"{case}_hist_pos"], 1e-6, "history pos")
    _close(Ag.pos, g[f"{case}_pos"][-1], 1e-9, "final pos")
    # Ag.run from the same state: the clock and the trajectory are followed on the device
    Ag2 = _agent(rb, g, case, env, dt)
    Ag2.import_trajectory(times=g[f"{case}_times"], positions=g[f"{case}_positions"])
    Ag2.run(n)
    for k in STATE:
        _close(getattr(Ag2, k), g[f"{case}_{k}"][-1], 1e-9, f"{case} run {k}")
    assert Ag2.t == Ag.t


def test_forced_against_the_reference_and_the_oracle(golden):
    """Forced positions with a NaN sample (zero rates, distance unchanged, velocities NaN) and a zero displacement (a
    nonzero draw of norm <= 1.5e-8 that becomes the velocity; the oracle fed the device's draw agrees afterwards)."""
    import ratinabox_b200 as rb
    g = golden("traj.npz")
    Ag = _agent(rb, g, "frc", _box(rb, g), 0.05)
    pops = _pops(rb, g, "frc", Ag)
    ora = OT.OracleTrajAgent(O.OracleEnvironment(walls=g["box_walls"]), g["frc_s0_pos"], g["frc_s0_velocity"], {"dt": 0.05})
    for k in STATE:
        setattr(ora, k, np.array(g[f"frc_s0_{k}"]) if g[f"frc_s0_{k}"].ndim else float(g[f"frc_s0_{k}"]))
    F = g["frc_forced"]
    for i in range(len(F)):
        Ag.update(forced_next_position=F[i].copy())
        for N, _ in pops.values():
            N.update()
        fb = np.zeros(2)
        if i == 9:
            mv = np.asarray(Ag.measured_velocity)
            assert 0 < np.linalg.norm(mv) <= 1.5e-8 and np.array_equal(np.asarray(Ag.velocity), mv)
            fb = mv
        ora.update(forced_next_position=F[i].copy(), fallback=fb)
        for k in STATE:
            _close(getattr(Ag, k), getattr(ora, k), TOL[k], f"frc step {i} {k}")
            if i < 9:
                _close(getattr(Ag, k), g[f"frc_{k}"][i], TOL[k], f"frc step {i} {k} (reference)")
        for name, (N, scale) in pops.items():
            # from step 9 on the head direction follows the device's zero-displacement draw, not the reference's: the
            # egocentric cells are compared up to there, the place and grid cells (positions only) throughout
            if i < 9 or name != "fov":
                _close(N.firingrate, g[f"frc_rates_{name}"][i], RATE_TOL * scale, f"frc step {i} {name}")
        if i == 15:
            assert all(np.all(N.firingrate == 0) for N, _ in pops.values())
            assert Ag.distance_travelled == g["frc_distance_travelled"][14]


def test_forced_across_a_periodic_boundary(golden):
    import ratinabox_b200 as rb
    g = golden("traj.npz")
    Ag = _agent(rb, g, "per", rb.Environment({"boundary_conditions": "periodic"}), 0.05)
    for i, p in enumerate(g["per_forced"]):
        Ag.update(forced_next_position=p.copy())
        for k in STATE:
            _close(getattr(Ag, k), g[f"per_{k}"][i], TOL[k], f"per step {i} {k}")


def test_forced_positions_batched_and_from_torch():
    """(2,) broadcast, (A, 2) per agent, device and page-locked torch tensors; run() refuses forced positions."""
    import torch
    import ratinabox_b200 as rb
    A = 6
    Ag = rb.Agent(rb.Environment(), {"n_agents": A, "dt": 0.05})
    P = np.random.default_rng(0).uniform(0.1, 0.9, (A, 2))
    Ag.update(forced_next_position=np.array([0.4, 0.6]))
    assert np.array_equal(Ag.pos, np.tile([0.4, 0.6], (A, 1)))
    Ag.update(forced_next_position=P)
    assert np.array_equal(Ag.pos, P)
    _close(Ag.measured_velocity, (P - [0.4, 0.6]) / 0.05, 1e-13, "measured velocity")
    assert np.array_equal(Ag.velocity, Ag.measured_velocity)
    Ag.update(forced_next_position=torch.as_tensor(P[::-1].copy(), device="cuda"))
    assert np.array_equal(Ag.pos, P[::-1])
    pinned = torch.as_tensor(P).pin_memory()
    Ag.update(forced_next_position=pinned)
    assert np.array_equal(Ag.pos, P)
    with pytest.raises(NotImplementedError):
        Ag.run(3, forced_next_position=P)
    with pytest.raises(AssertionError):
        Ag.update(forced_next_position=np.zeros((A + 1, 2)))


def _build(rb, kind, A, traj, per_agent, rows, fused=False):
    np.random.seed(7)
    E = rb.Environment()
    E.add_wall([[0.3, 0.0], [0.3, 0.5]])
    Ag = rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": 11, "fused_step": fused, "history_bytes_limit": 5 * A * 32})
    rs = np.random.RandomState(4)
    if kind == "place":
        Ns = rb.PlaceCells(Ag, {"n": 512, "place_cell_centres": rs.uniform(0, 1, (512, 2)), "widths": 0.15,
                                "wall_geometry": "line_of_sight", "save_spikes": True,
                                "history_bytes_limit": rows * A * 512 * 4})
    else:
        Ns = rb.GridCells(Ag, {"n": 512, "gridscale": rs.uniform(0.2, 1.0, 512), "orientation": rs.uniform(0, 1, 512),
                               "phase_offset": rs.uniform(0, 6, (512, 2)), "save_spikes": True,
                               "history_bytes_limit": rows * A * 512 * 4})
    times, pos = traj
    Ag.import_trajectory(times=times, positions=pos if not per_agent else pos[:A])
    return Ag, Ns


@pytest.mark.parametrize("kind,per_agent,rows", [("place", False, 3), ("grid", True, 2), ("place", True, 40)])
def test_launch_paths_agree_bit_for_bit(monkeypatch, kind, per_agent, rows):
    """The whole run (ONE launch), the per-step loop (RIAB_NO_WHOLE_RUN=1) and the stepped update() + Neurons.update()
    loop (plain and fused_step) give identical agent state, rates, history rings and spike rows, also when the rings
    wrap; every retained spike row equals the NumPy mirror of its stream."""
    import ratinabox_b200 as rb
    from ratinabox_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(8)
    T = 30
    times = np.cumsum(rng.uniform(0.05, 0.2, T))
    A = 300
    pos = rng.uniform(0.05, 0.95, (A, T, 2) if per_agent else (T, 2))
    steps = int(times[-1] / 0.02) + 15                  # past t_max
    res = {}
    for way in ("W", "R", "S", "F"):
        Ag, Ns = _build(rb, kind, A, (times, pos), per_agent, rows, fused=(way == "F"))
        Ag.update(); Ns.update()                        # one stepped step first: t != dt at the run
        c0 = lib.riab_launch_count()
        if way in ("W", "R"):
            with monkeypatch.context() as m:
                if way == "R":
                    m.setenv("RIAB_NO_WHOLE_RUN", "1")
                else:
                    m.delenv("RIAB_NO_WHOLE_RUN", raising=False)
                Ag.run(steps)
        else:
            for _ in range(steps):
                Ag.update(); Ns.update()
        launches = lib.riab_launch_count() - c0
        if way == "W":
            assert launches == 1, launches
        out = {k: np.asarray(getattr(Ag, k)).copy() for k in STATE}
        out["firingrate"], out["t"] = Ns.firingrate, Ag.t
        for k, v in Ag.get_history_arrays().items():
            out["agent." + k] = v
        for k, v in Ns.get_history_arrays().items():
            out["pop." + k] = v
        out["pop.dropped"] = Ns.history_dropped
        res[way] = out
        if way == "W":
            assert Ns.history_dropped > 0 or rows >= steps
            check_spikes(out, Ns, {"dt": 0.02}, A, steps + 1, f"{kind} spikes")
            # positions follow the spline at the accumulated clock
            x = times - times.min()
            y = pos.transpose(1, 0, 2) if per_agent else pos[:, None, :]
            M = spline_np.build(x, y)
            want = spline_np.evaluate(x, y, M, np.array(Ag.t % x[-1]))
            _close(Ag.pos, np.broadcast_to(want, (A, 2)), 1e-12, "final pos vs mirror")
    for way in ("R", "S", "F"):
        assert_same(res["W"], res[way], f"W vs {way}")


def test_live_reference_import_agrees():
    """With the reference staged (oracle/_ref), its import_trajectory + update() against the device."""
    import ref_shim
    rat = ref_shim.import_reference()
    if rat is None:
        pytest.skip("reference not staged")
    import ratinabox_b200 as rb
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    rng = np.random.default_rng(21)
    times = np.cumsum(rng.uniform(0.02, 0.3, 60))
    pos = 0.5 + 0.3 * np.stack([np.cos(times), np.sin(1.7 * times)], axis=1)
    R = Agent(Environment(), {"dt": 0.03})
    D = rb.Agent(rb.Environment(), {"dt": 0.03})
    for k in STATE:
        setattr(D, k, getattr(R, k))
    R.import_trajectory(times=times, positions=pos)
    D.import_trajectory(times=times, positions=pos)
    for i in range(int(times[-1] / 0.03) + 20):
        R.update()
        D.update()
        for k in STATE:
            _close(getattr(D, k), getattr(R, k), TOL[k], f"live step {i} {k}")

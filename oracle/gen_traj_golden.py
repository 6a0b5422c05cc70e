"""TEST INFRASTRUCTURE -- write tests/golden/traj.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): the imported / forced branches of Agent.update (ratinabox/Agent.py:202-259, :444-507) and
Agent.import_trajectory (:543-659).

    python oracle/gen_traj_golden.py

Every case stores the Agent's state before its first imported / forced step (``<case>_s0_<attr>``) and after every step
(``<case>_<attr>``, leading step axis), so a device Agent can be put into the same state and stepped alongside.
  * ``syn``: an irregularly sampled synthetic trajectory (40 samples) in a box with two inner walls, run past t_max
    (the wrap), with line-of-sight PlaceCells, GridCells and egocentric FieldOfViewBVCs (rates, noise_std = 0);
  * ``sar``: the first 3 000 samples of sargolini.npz, imported after 5 random steps (t != 0 at import);
  * ``frc``: forced positions in the walled box, with a NaN sample, a repeated position (zero displacement: the
    reference's 1e-8 randn fall-back is stored as ``frc_fallback``) and the same three populations;
  * ``per``: forced positions crossing the boundary of a periodic box;
  * ``prec``: forced_next_position passed to an Agent that imported a trajectory (the reference raises TypeError:
    ``err_precedence``) and that Agent's steps without it;
  * ``err_<case>``: the exception type names of import_trajectory for interpolate=False, T < 4, duplicate times and a
    periodic box.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
BOX_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
STATE = ("pos", "velocity", "rotational_velocity", "measured_velocity", "measured_rotational_velocity",
         "head_direction", "distance_travelled")


def _state(Ag):
    return {k: np.array(getattr(Ag, k), dtype=np.float64) for k in STATE} | {"t": np.array(Ag.t, dtype=np.float64)}


def _record(out, case, Ag, pops, steps, kw_of_step=lambda i: {}):
    for k, v in _state(Ag).items():
        out[f"{case}_s0_{k}"] = v
    rec = {k: [] for k in list(STATE) + ["t"] + [f"rates_{n}" for n in pops]}
    for i in range(steps):
        Ag.update(**kw_of_step(i))
        for N in pops.values():
            N.update()
        for k, v in _state(Ag).items():
            rec[k].append(v)
        for n, N in pops.items():
            rec[f"rates_{n}"].append(np.array(N.firingrate, dtype=np.float64).copy())
    for k, v in rec.items():
        out[f"{case}_{k}"] = np.array(v)
    h = Ag.history
    out[f"{case}_hist_pos"] = np.array(h["pos"][-steps:])
    out[f"{case}_hist_vel"] = np.array(h["vel"][-steps:])


def _pops(out, case, Ag, rng):
    from ratinabox.Neurons import PlaceCells, GridCells, FieldOfViewBVCs
    centres = rng.uniform(0.02, 0.98, (24, 2))
    gs, orient, phase = rng.uniform(0.2, 0.6, 12), rng.uniform(0, 2 * np.pi / 3, 12), rng.uniform(0, 1, (12, 2))
    out[f"{case}_pc_centres"], out[f"{case}_gc_gridscales"] = centres, gs
    out[f"{case}_gc_orientations"], out[f"{case}_gc_phase_offsets"] = orient, phase
    pc = PlaceCells(Ag, {"place_cell_centres": centres, "widths": 0.2, "wall_geometry": "line_of_sight",
                         "min_fr": 0.0, "max_fr": 1.0, "noise_std": 0.0})
    gc = GridCells(Ag, {"gridscale": gs, "orientation": orient, "phase_offset": phase, "min_fr": 0.0, "max_fr": 1.0,
                        "noise_std": 0.0})
    fov = FieldOfViewBVCs(Ag, {"min_fr": 0.0, "max_fr": 2.0, "noise_std": 0.0})
    return {"pc": pc, "gc": gc, "fov": fov}


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    import ratinabox
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    out = {"box_walls": np.array(BOX_WALLS, dtype=np.float64)}
    rng = np.random.default_rng(5)
    np.random.seed(0)

    # ---- syn: irregular samples, wrap past t_max, three populations
    Env = Environment()
    for w in BOX_WALLS:
        Env.add_wall(w)
    T = 40
    times = np.cumsum(rng.uniform(0.03, 0.45, T)) + 3.0            # shifted to 0 by import_trajectory
    ang = np.linspace(0, 3 * np.pi, T)
    positions = np.stack([0.5 + 0.35 * np.cos(ang) + rng.normal(0, 0.02, T),
                          0.5 + 0.3 * np.sin(1.3 * ang) + rng.normal(0, 0.02, T)], axis=1)
    out["syn_times"], out["syn_positions"] = times, positions
    Ag = Agent(Env, {"dt": 0.05})
    pops = _pops(out, "syn", Ag, rng)
    Ag.import_trajectory(times=times, positions=positions)
    steps = int(np.ceil((times[-1] - times[0]) / 0.05)) + 40          # past t_max: the wrap
    _record(out, "syn", Ag, pops, steps)

    # ---- sar: sargolini slice imported after a few random steps
    d = np.load(os.path.join(os.path.dirname(ratinabox.__file__), "data", "sargolini.npz"))
    out["sar_times"], out["sar_positions"] = d["t"][:3000], d["pos"][:3000]
    Env2 = Environment()
    Ag2 = Agent(Env2, {"dt": 0.1})
    for _ in range(5):
        Ag2.update()
    Ag2.import_trajectory(times=out["sar_times"], positions=out["sar_positions"])
    _record(out, "sar", Ag2, {}, 120)

    # ---- frc: forced positions with a NaN sample and a zero displacement, three populations
    Env3 = Environment()
    for w in BOX_WALLS:
        Env3.add_wall(w)
    Ag3 = Agent(Env3, {"dt": 0.05})
    pops3 = _pops(out, "frc", Ag3, rng)
    F = 0.5 + 0.3 * np.stack([np.cos(np.linspace(0, 2, 30)), np.sin(np.linspace(0, 3, 30))], axis=1)
    F[9] = F[8]                       # zero displacement: measured velocity = 1e-8 randn (Agent.py:460-461)
    F[15] = [np.nan, np.nan]          # a NaN sample: velocities NaN, distance unchanged, zero rates
    out["frc_forced"] = F
    _record(out, "frc", Ag3, pops3, len(F), lambda i: {"forced_next_position": F[i].copy()})
    out["frc_fallback"] = out["frc_measured_velocity"][9]

    # ---- per: forced positions crossing a periodic boundary
    Env4 = Environment({"boundary_conditions": "periodic"})
    Ag4 = Agent(Env4, {"dt": 0.05})
    P = np.array([[0.9, 0.5], [0.97, 0.52], [0.02, 0.55], [0.06, 0.97], [0.08, 0.03], [0.1, 0.08], [0.98, 0.1]])
    out["per_forced"] = P
    _record(out, "per", Ag4, {}, len(P), lambda i: {"forced_next_position": P[i].copy()})

    # ---- error cases of import_trajectory
    def err(f):
        try:
            f()
        except Exception as e:          # noqa: BLE001 -- the type name is the fixture
            return type(e).__name__
        return "none"

    # ---- prec: forced_next_position given to an Agent that imported a trajectory.  The branch order (Agent.py:219-232)
    # takes the imported branch, which passes **kwargs on to _update_position_along_imported_trajectory(self) (:230,
    # :255): the reference raises TypeError for ANY kwarg there.  Stored as such, with the state after an update()
    # without kwargs for comparison
    Env5 = Environment()
    Ag5 = Agent(Env5, {"dt": 0.05})
    Ag5.import_trajectory(times=times, positions=positions)
    out["err_precedence"] = np.array(err(lambda: Ag5.update(forced_next_position=np.array([0.1, 0.1]))))
    Ag5 = Agent(Env5, {"dt": 0.05})
    Ag5.import_trajectory(times=times, positions=positions)
    _record(out, "prec", Ag5, {}, 10)
    Ag6 = Agent(Environment(), {"dt": 0.05})
    out["err_interpolate_false"] = np.array(err(lambda: Ag6.import_trajectory(times=times, positions=positions,
                                                                                interpolate=False)))
    out["err_short"] = np.array(err(lambda: Agent(Environment(), {}).import_trajectory(times=times[:3],
                                                                                        positions=positions[:3])))
    tdup = times.copy()
    tdup[5] = tdup[4]
    out["err_duplicate"] = np.array(err(lambda: Agent(Environment(), {}).import_trajectory(times=tdup, positions=positions)))
    out["err_periodic"] = np.array(err(lambda: Agent(Environment({"boundary_conditions": "periodic"}), {})
                                       .import_trajectory(times=times, positions=positions)))
    np.savez_compressed(os.path.join(GOLD, "traj.npz"), **out)
    print("traj.npz", len(out), "arrays")


if __name__ == "__main__":
    main()

"""TEST INFRASTRUCTURE -- write tests/golden/td_pa.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): K independent single-agent ValueNeuron runs (contribs/ValueNeuron.py) along ONE shared trajectory,
the data a batch of K agents with per-agent weights must reproduce row by row.

    python oracle/gen_td_pa_golden.py

The trajectory is a seeded 200-step native run in the box with two walls (the setting of gen_td_golden.py).  Every run
k then replays it with Agent.update(forced_next_position=...) over the same PlaceCells(20, line_of_sight) and
GridCells(12) (the same seed builds them), with its own initial weights (seed 100 + k) and its own one-cell top_hat
reward at REWARD_CENTRES[k]; update_weights every step.

Contents: the shared "pos" (steps, 2), the cells' parameters, and per run k (leading axis K): the "biases", the input
rates "PC" / "GC", "reward", "fr", "prime", "td" and the traces "e_PC" / "e_GC" per step, and the weights every 10 steps
("W_PC", "W_GC": [k, c] after step 10 c, [k, 0] before step 1).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
BOX_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
VN_PARAMS = {"tau": 1.0, "eta": 0.05, "L2": 0.01}
REWARD_CENTRES = [[0.1, 0.1], [0.2, 0.3], [0.15, 0.55]]
STEPS = 200


def _env():
    from ratinabox.Environment import Environment
    Env = Environment()
    for w in BOX_WALLS:
        Env.add_wall(w)
    return Env


def _setup():
    """Agent, PlaceCells, GridCells, identical for every run."""
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import PlaceCells, GridCells
    np.random.seed(11)
    Ag = Agent(_env(), {"dt": 0.05})
    pc = PlaceCells(Ag, {"n": 20, "wall_geometry": "line_of_sight", "name": "PC"})
    gc = GridCells(Ag, {"n": 12, "name": "GC"})
    return Ag, pc, gc


def trajectory():
    Ag, _, _ = _setup()
    pos = []
    for _ in range(STEPS):
        Ag.update()
        pos.append(Ag.pos.copy())
    return np.array(pos)


def run(k, pos, out):
    from ratinabox.Neurons import PlaceCells
    from ratinabox.contribs.ValueNeuron import ValueNeuron
    Ag, pc, gc = _setup()
    rew = PlaceCells(Ag, {"n": 1, "description": "top_hat", "widths": 0.3,
                          "place_cell_centres": np.array([REWARD_CENTRES[k]]), "name": "Reward"})
    np.random.seed(100 + k)
    vn = ValueNeuron(Ag, dict(VN_PARAMS, input_layers=[pc, gc], biases=np.full(1, 0.3)))
    if k == 0:
        out["pc_centres"], out["pc_widths"] = pc.place_cell_centres, pc.place_cell_widths
        out["gc_gridscales"], out["gc_phase_offsets"], out["gc_w"] = gc.gridscales, gc.phase_offsets, gc.w
        out["tau_e"] = vn.tau_e
    rec = {key: [] for key in ["reward", "fr", "prime", "td", "e_PC", "e_GC", "PC", "GC"]}
    W = {"PC": [vn.inputs["PC"]["w"].copy()], "GC": [vn.inputs["GC"]["w"].copy()]}
    rec["biases"] = np.asarray(vn.biases, dtype=np.float64).copy()
    for t in range(STEPS):
        Ag.update(forced_next_position=pos[t].copy())
        for N in Ag.Neurons:
            N.update()
        vn.update_weights(rew.firingrate)
        assert np.array_equal(Ag.pos, pos[t])
        rec["reward"].append(rew.firingrate.copy())
        rec["PC"].append(pc.firingrate.copy())
        rec["GC"].append(gc.firingrate.copy())
        rec["fr"].append(vn.firingrate.copy())
        rec["prime"].append(np.asarray(vn.firingrate_prime, dtype=np.float64).copy())
        rec["td"].append(vn.td_error.copy())
        rec["e_PC"].append(vn.inputs["PC"]["eligibility_trace"].copy())
        rec["e_GC"].append(vn.inputs["GC"]["eligibility_trace"].copy())
        if (t + 1) % 10 == 0:
            for key in W:
                W[key].append(vn.inputs[key]["w"].copy())
    rec["W_PC"], rec["W_GC"] = np.array(W["PC"]), np.array(W["GC"])
    return {key: np.array(v) for key, v in rec.items()}


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    out = {}
    pos = trajectory()
    out["pos"] = pos
    runs = [run(k, pos, out) for k in range(len(REWARD_CENTRES))]
    for key in runs[0]:
        out[key] = np.stack([r[key] for r in runs])
    out["reward_centres"] = np.array(REWARD_CENTRES)
    np.savez_compressed(os.path.join(GOLD, "td_pa.npz"), **out)
    print("td_pa.npz", len(out), "arrays")


if __name__ == "__main__":
    main()

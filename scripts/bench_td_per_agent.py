"""Cost of per-agent TD learning (ValueNeuron(per_agent_weights=True)), modelled on scripts/bench_td.py:
  * vpa: the c2 setting (65 536 agents, box + 2 walls, 1024 line-of-sight PlaceCells) plus a per-agent ValueNeuron
    (n = 1) over the PlaceCells, rewarded by a device tensor;
  * sfpa: SuccessorFeatures (n = 64) of 64 PlaceCells at 16 384 agents, per agent.
For each: ms per stepped iteration (Ag.update, PlaceCells.update, the TD layer's update, update_weights), every TD
kernel's time over many launches (torch.profiler's CUDA kernel records), and the bytes of W each kernel must move,
8 A n n_in for the forward and 16 A n n_in for the learning step (plus the rows and traces), against 3.35 TB/s HBM3
(H100 SXM data sheet).  Prints one JSON line with the card's name and power limit, read in the same run.

    python scripts/bench_td_per_agent.py [--steps 30] [--launches 20]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
import bench_ffl  # noqa: E402
import bench_td  # noqa: E402
import ratinabox_b200 as rb  # noqa: E402
from ratinabox_b200.contribs import SuccessorFeatures, ValueNeuron  # noqa: E402

HBM_GBS = 3350.0


def build(kind):
    wl = bench.WORKLOADS["c2"]
    A = wl["agents"] if kind == "vpa" else 16384
    np.random.seed(1234)
    Env = rb.Environment()
    for w in wl["walls"]:
        Env.add_wall(w)
    Ag = rb.Agent(Env, {"dt": 0.01, "n_agents": A, "seed": 7})
    pos, vel = bench.synthetic_agents(A, wl["walls"], 100)
    Ag.pos, Ag.velocity = pos, vel
    Ag.measured_velocity = vel
    if kind == "vpa":
        pcs = bench.build_populations(rb, Ag, wl)[0]
        td = ValueNeuron(Ag, {"input_layers": [pcs], "name": "VN", "per_agent_weights": True})
        reward = torch.full((1,), 0.5, dtype=torch.float64, device="cuda")
        learn = lambda: td.update_weights(reward)           # noqa: E731
    else:
        pcs = rb.PlaceCells(Ag, {"n": 64, "name": "PC", "wall_geometry": "line_of_sight", "save_history": False})
        td = SuccessorFeatures(Ag, {"features": pcs, "input_layers": [pcs], "name": "SF", "save_history": False,
                                    "per_agent_weights": True})
        learn = td.update_weights
    return Ag, pcs, td, learn


def model(A, n, n_in):
    """Bytes of each per-agent kernel from the shapes (float32 rows with their padded strides, float64 W)."""
    ld, ld_in = (n + 3) // 4 * 4, (n_in + 3) // 4 * 4
    m = {
        "k_td_forward_pa": {"w_bytes": 8.0 * A * n * n_in, "bytes": 8.0 * A * n * n_in + 4.0 * A * (ld_in + 2 * ld)},
        "k_td_learn_pa": {"w_bytes": 16.0 * A * n * n_in, "bytes": 16.0 * A * n * n_in + 4.0 * A * (ld_in + 2 * ld)},
        "k_td_trace": {"bytes": 4.0 * A * (3 * ld_in + 3 * ld)},
        "k_td_g": {"bytes": 4.0 * A * 5 * ld},
    }
    for v in m.values():
        v["hbm_floor_us"] = v["bytes"] / (HBM_GBS * 1e9) * 1e6
    return m


def run(kind, steps, launches):
    Ag, pcs, td, learn = build(kind)
    A, n, n_in = Ag.n_agents, td.n, pcs.n
    r = {"ms_per_iteration": bench_td.ms_per_iteration(Ag, pcs, td, learn, steps)}
    times = bench_td.kernel_times(Ag, pcs, td, learn, launches)
    mod = model(A, n, n_in)
    for k, v in mod.items():
        if k in times:
            us = times[k]["us"]
            v["us"] = us
            v["gbs"] = v["bytes"] / (us * 1e-6) / 1e9
            v["frac_of_hbm_floor"] = v["hbm_floor_us"] / us
    r["kernels"] = mod
    r["A"], r["n"], r["n_in"] = A, n, n_in
    del Ag, pcs, td, learn
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--launches", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_td_per_agent.py measures on a CUDA device")
    res = {"card": bench_ffl.card(), "steps": args.steps, "launches": args.launches}
    for kind in ("vpa", "sfpa"):
        res[kind] = run(kind, args.steps, args.launches)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

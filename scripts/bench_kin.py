"""Cost of the kinematic populations (HeadDirectionCells, VelocityCells, SpeedCell) on top of the motion step: 65 536
agents in the c2 box (2 inner walls), dt 0.01, default history (rates and spike rings).  Prints one JSON line with, per
set-up, ms per step of Ag.run (CUDA events; the set-ups are timed twice in alternating order, both rounds reported):
  * motion alone (no population);
  * HeadDirectionCells(n=10);
  * HeadDirectionCells(10) + VelocityCells(10) + SpeedCell;
  * HeadDirectionCells(n=256);
each set-up's extra ms over motion alone, and its populations' row bytes per step (rates + spike words) over the
H100 SXM data sheet's 3.35 TB/s, the least time those writes can take; plus the card's name and power limit, read in
the same run.  Writes nothing.
  python scripts/bench_kin.py [--steps K] [--warmup W]"""
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
import ratinabox_b200 as rb  # noqa: E402

HBM_PEAK_GBS = 3350.0                                   # H100 SXM data sheet (HBM3)
SETUPS = {
    "motion": [],
    "hdc10": [("HeadDirectionCells", {"n": 10})],
    "hdc10_vel10_speed": [("HeadDirectionCells", {"n": 10}), ("VelocityCells", {"n": 10}), ("SpeedCell", {})],
    "hdc256": [("HeadDirectionCells", {"n": 256})],
}


def build(pops):
    wl = bench.WORKLOADS["c2"]
    A = wl["agents"]
    np.random.seed(1234)
    Env = rb.Environment()
    for w in wl["walls"]:
        Env.add_wall(w)
    Ag = rb.Agent(Env, {"dt": 0.01, "n_agents": A, "seed": 7})
    pos, vel = bench.synthetic_agents(A, wl["walls"], 100)
    Ag.pos, Ag.velocity = pos, vel
    Ag.measured_velocity = vel
    for cls, prm in pops:
        getattr(rb, cls)(Ag, prm)
    return Ag


def row_bytes(Ag):
    """Bytes one step writes to the populations' rings: float32 rates (ld floats per agent) and 4 spike words per 128 cells."""
    return sum(Ag.n_agents * (N._ld() + 4 * ((N.n + 127) // 128)) * 4 for N in Ag.Neurons)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_kin.py measures on a CUDA device")
    res = {"workload": "c2 box + 2 walls, 65536 agents, dt 0.01, Ag.run with history and spikes", "steps": args.steps,
           "card": bench_ffl.card()}
    times = {k: [] for k in SETUPS}
    for _ in range(2):
        for name, pops in SETUPS.items():
            Ag = build(pops)
            times[name].append(bench_ffl.ms_per_step(Ag, args.steps, args.warmup))
            nbytes = row_bytes(Ag)
            res[f"{name}_row_bytes"] = nbytes
            res[f"{name}_row_bytes_us_at_peak"] = nbytes / (HBM_PEAK_GBS * 1e9) * 1e6
            del Ag
            torch.cuda.empty_cache()
    base = min(times["motion"])
    for name, t in times.items():
        res[f"{name}_ms_per_step"] = t
        if name != "motion":
            res[f"{name}_extra_ms"] = min(t) - base
    res["hbm_peak_gbs"] = HBM_PEAK_GBS
    print(json.dumps(res))


if __name__ == "__main__":
    main()

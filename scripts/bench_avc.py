"""Cost of AgentVectorCells on top of the motion step: 65 536 agent pairs (two Agents of 65 536 rows, row i of Ag1 sees
row i of Ag2) in the c2 box (2 inner walls), dt 0.01, default history (rates and spike rings).  Prints one JSON line with
ms per step (CUDA events; every set-up is timed twice in alternating order, both rounds reported) of:
  * motion alone: Ag1.run(K) without populations;
  * avc10: Ag1.run(K) with AgentVectorCells(Ag1, Ag2, n=10) (line of sight);
  * fov58: Ag1.run(K) with FieldOfViewAVCs(Ag1, Ag2) (58 cells);
  * motion_both_stepped: the stepped two-Agent loop ``Ag1.update(); Ag2.update()`` without populations;
  * avc_both_stepped: the same loop with AgentVectorCells(n=10) both ways, each Agent's population updated after both moved;
each set-up's extra ms over its motion-only baseline, and its populations' row bytes per step (rates + spike words) over
the H100 SXM data sheet's 3.35 TB/s, the least time those writes can take; plus the card's name and power limit, read in
the same run.  Writes nothing.
  python scripts/bench_avc.py [--steps K] [--warmup W]"""
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
import bench_kin  # noqa: E402
import ratinabox_b200 as rb  # noqa: E402

HBM_PEAK_GBS = bench_kin.HBM_PEAK_GBS
RUN_SETUPS = {"motion": [], "avc10": [("AgentVectorCells", {"n": 10})], "fov58": [("FieldOfViewAVCs", {})]}
STEP_SETUPS = {"motion_both_stepped": False, "avc_both_stepped": True}


def build(pops, both=False):
    wl = bench.WORKLOADS["c2"]
    A = wl["agents"]
    np.random.seed(1234)
    Env = rb.Environment()
    for w in wl["walls"]:
        Env.add_wall(w)
    agents = []
    for seed in (7, 8):
        Ag = rb.Agent(Env, {"dt": 0.01, "n_agents": A, "seed": seed})
        pos, vel = bench.synthetic_agents(A, wl["walls"], 100 + seed)
        Ag.pos, Ag.velocity = pos, vel
        agents.append(Ag)
    Ag1, Ag2 = agents
    for cls, prm in pops:
        getattr(rb, cls)(Ag1, Ag2, dict(prm))
        if both:
            getattr(rb, cls)(Ag2, Ag1, dict(prm))
    return Ag1, Ag2


def stepped_ms_per_step(Ag1, Ag2, steps, warmup):
    def loop(k):
        for _ in range(k):
            Ag1.update()
            Ag2.update()
            for N in Ag1.Neurons + Ag2.Neurons:
                N.update()
    loop(warmup)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    loop(steps)
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_avc.py measures on a CUDA device")
    res = {"workload": "c2 box + 2 walls, 65536 agent pairs, dt 0.01, history and spikes", "steps": args.steps,
           "card": bench_ffl.card()}
    times = {k: [] for k in list(RUN_SETUPS) + list(STEP_SETUPS)}
    for _ in range(2):
        for name, pops in RUN_SETUPS.items():
            Ag1, Ag2 = build(pops)
            times[name].append(bench_ffl.ms_per_step(Ag1, args.steps, args.warmup))
            nbytes = bench_kin.row_bytes(Ag1)
            res[f"{name}_row_bytes"] = nbytes
            res[f"{name}_row_bytes_us_at_peak"] = nbytes / (HBM_PEAK_GBS * 1e9) * 1e6
            del Ag1, Ag2
            torch.cuda.empty_cache()
        for name, with_avc in STEP_SETUPS.items():
            Ag1, Ag2 = build([("AgentVectorCells", {"n": 10})] if with_avc else [], both=True)
            times[name].append(stepped_ms_per_step(Ag1, Ag2, args.steps, args.warmup))
            nbytes = bench_kin.row_bytes(Ag1) + bench_kin.row_bytes(Ag2)
            res[f"{name}_row_bytes"] = nbytes
            res[f"{name}_row_bytes_us_at_peak"] = nbytes / (HBM_PEAK_GBS * 1e9) * 1e6
            del Ag1, Ag2
            torch.cuda.empty_cache()
    for name, t in times.items():
        res[f"{name}_ms_per_step"] = t
    res["avc10_extra_ms"] = min(times["avc10"]) - min(times["motion"])
    res["fov58_extra_ms"] = min(times["fov58"]) - min(times["motion"])
    res["avc_both_stepped_extra_ms"] = min(times["avc_both_stepped"]) - min(times["motion_both_stepped"])
    res["hbm_peak_gbs"] = HBM_PEAK_GBS
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Per-step device time in environments with many walls: the unit box (4 walls), the README's circular arena (100), the
successor-features demo's loop track (200) and a 1024-wall maze (the box and 1020 random 2 cm walls).  Rows, each after
a warm-up, timed with CUDA events around --steps steps that end in a synchronise:
  * motion:  Ag.update() alone (k_agent_update), 65 536 agents;
  * run_pc:  Ag.run(steps) with 1 024 Euclidean PlaceCells, 65 536 agents (above 64 walls: the motion kernel, then the
             rate kernel, per step);
  * bvc:     BVCs.update() (k_bvc_rays + k_bvc_integrate) at fixed positions, 16 384 agents x 512 cells.
Beside each row its work per agent-step computed from W: the FP64 operations of the motion step's two per-wall loops
(wall repulsion: 20 per wall; one collision-test pass: 16 per wall; passes = 1 + bounces, counted here as 1), and the
(ray, wall) screens of the BVC rays (T x W).  Prints the card's name and power limit, read in the same run, and one JSON
line.  Writes nothing.  The library is the one ratinabox_b200 loads (RIAB_LIB selects another build, e.g. the parent
commit's, so that two builds can be run alternately in one job).
  python scripts/bench_curved.py [--steps K] [--warmup W] [--envs box,circle,annulus,maze1024] [--rows motion,run_pc,bvc]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ratinabox_b200 as rb  # noqa: E402

FP64_REPEL_PER_WALL, FP64_COLLIDE_PER_WALL = 20, 16
# H100 SXM data sheet, FP64 without tensor cores (a card allowed up to 700 W)
FP64_PEAK = 34e12


def circle(r, n=100):
    return [[r * np.cos(t), r * np.sin(t)] for t in np.linspace(0, 2 * np.pi, n)]


def make_env(name):
    if name == "box":
        return rb.Environment()
    if name == "circle":
        return rb.Environment({"boundary": circle(0.5)})
    if name == "annulus":
        return rb.Environment({"boundary": circle(0.5), "holes": [circle(0.4)]})
    if name == "maze1024":
        rs = np.random.RandomState(0)
        E = rb.Environment()
        c = rs.uniform(0.05, 0.95, size=(1020, 2))
        ang = rs.uniform(0, np.pi, size=1020)
        h = 0.01 * np.stack((np.cos(ang), np.sin(ang)), axis=1)
        for a, b in zip(c - h, c + h):
            E.add_wall([a, b])
        return E
    raise ValueError(name)


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def row(env_name, kind, steps, warmup):
    np.random.seed(1)
    E = make_env(env_name)
    W = len(E.walls)
    if kind == "motion":
        Ag = rb.Agent(E, {"n_agents": 65536, "dt": 0.01, "save_history": False, "seed": 3})
        ms = timed(Ag.update, steps, warmup)
        ops = W * (FP64_REPEL_PER_WALL + FP64_COLLIDE_PER_WALL)
        rate = ops * 65536 / (ms * 1e-3)
        return {"ms_per_step": ms, "fp64_ops_per_agent_step": ops, "fp64_ops_per_s": rate, "fp64_share_of_peak": rate / FP64_PEAK}
    if kind == "run_pc":
        Ag = rb.Agent(E, {"n_agents": 65536, "dt": 0.01, "save_history": False, "seed": 3})
        rb.PlaceCells(Ag, {"n": 1024, "wall_geometry": "euclidean", "save_history": False})
        Ag.run(warmup)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        Ag.run(steps)
        e1.record()
        torch.cuda.synchronize()
        return {"ms_per_step": e0.elapsed_time(e1) / steps,
                "fp64_ops_per_agent_step": W * (FP64_REPEL_PER_WALL + FP64_COLLIDE_PER_WALL)}
    if kind == "bvc":
        Ag = rb.Agent(E, {"n_agents": 16384, "dt": 0.01, "save_history": False, "seed": 3})
        BVCs = rb.BoundaryVectorCells(Ag, {"n": 512, "save_history": False})
        Ag.update()
        ms = timed(BVCs.update, steps, warmup)
        return {"ms_per_step": ms, "ray_wall_screens_per_agent_step": len(BVCs.test_angles) * W}
    raise ValueError(kind)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--envs", default="box,circle,annulus,maze1024")
    ap.add_argument("--rows", default="motion,run_pc,bvc")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_curved.py measures on a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    out = {"gpu": q[0] if q else torch.cuda.get_device_name(), "lib": os.environ.get("RIAB_LIB", "in-tree"),
           "steps": args.steps, "rows": {}}
    for env_name in args.envs.split(","):
        W = len(make_env(env_name).walls)
        for kind in args.rows.split(","):
            r = row(env_name, kind, args.steps, args.warmup)
            out["rows"][f"{env_name}/{kind}"] = dict(walls=W, **r)
            print(f"{env_name:9s} W={W:5d} {kind:7s} {r['ms_per_step']:.4f} ms/step", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

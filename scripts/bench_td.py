"""TD learning cost on the c2 workload (65 536 agents, box + 2 walls, 1024 line-of-sight PlaceCells):
  * c2v: c2 plus a ValueNeuron (n = 1) over the PlaceCells, rewarded by a device tensor;
  * c2s: SuccessorFeatures of the same PlaceCells (n = 1024), with the PlaceCells as the only input layer.
For each: ms per stepped iteration (Ag.update, PlaceCells.update, the TD layer's update, update_weights), every TD
kernel's time over many launches (torch.profiler's CUDA kernel records), and each kernel's bytes and FLOPs from the
shapes against 3.35 TB/s HBM3, 495 dense TF32 TFLOP/s and 67 FP32 CUDA-core TFLOP/s (H100 SXM data sheet), naming the
bound.  Prints one JSON line with the card's name and power limit, read in the same run.

    python scripts/bench_td.py [--steps 50] [--launches 30]
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
import ratinabox_b200 as rb  # noqa: E402
from ratinabox_b200.contribs import SuccessorFeatures, ValueNeuron  # noqa: E402

HBM_GBS, TF32_TFLOPS, FP32_TFLOPS = 3350.0, 495.0, 67.0


def build(kind):
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
    pcs = bench.build_populations(rb, Ag, wl)[0]
    if kind == "c2v":
        td = ValueNeuron(Ag, {"input_layers": [pcs], "name": "VN"})
        reward = torch.full((1,), 0.5, dtype=torch.float64, device="cuda")
        learn = lambda: td.update_weights(reward)           # noqa: E731
    else:
        td = SuccessorFeatures(Ag, {"features": pcs, "input_layers": [pcs], "name": "SF", "save_history": False})
        learn = td.update_weights
    return Ag, pcs, td, learn


def iteration(Ag, pcs, td, learn):
    Ag.update()
    pcs.update()
    td.update()
    learn()


def ms_per_iteration(Ag, pcs, td, learn, steps, warmup=5):
    for _ in range(warmup):
        iteration(Ag, pcs, td, learn)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(steps):
        iteration(Ag, pcs, td, learn)
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / steps


def kernel_times(Ag, pcs, td, learn, launches):
    """Mean CUDA time per launch of every k_td_* kernel over `launches` (td.update() + learn) pairs."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            td.update()
            learn()
        torch.cuda.synchronize()
    acc = {}
    for e in prof.events():
        name = e.name
        if "k_td_" not in name or e.device_type.name != "CUDA":
            continue
        key = name.split("k_td_")[1].split("<")[0].split("(")[0].split("I")[0]
        key = "k_td_" + key
        t, c = acc.get(key, (0.0, 0))
        acc[key] = (t + e.device_time_total if hasattr(e, "device_time_total") else t + e.cuda_time_total, c + 1)
    return {k: {"us": t / c, "launches": c} for k, (t, c) in acc.items()}


def model(A, n, n_in, splits):
    """Bytes / FLOPs of each kernel from the shapes (float32 rows with their padded strides; float64 master)."""
    ld, ld_in, ldg = (n + 3) // 4 * 4, (n_in + 3) // 4 * 4, (n + 7) // 8 * 8
    m = {
        "k_td_trace": {"bytes": 4.0 * A * (3 * ld_in + 3 * ld), "flop": 3.0 * A * n_in},
        "k_td_g": {"bytes": 4.0 * A * (5 * ld + ldg), "flop": 4.0 * A * n},
        "k_td_learn": {"bytes": 4.0 * A * (ld_in + ldg) + 8.0 * splits * n * n_in, "flop": 2.0 * A * n * n_in},
        "k_td_apply": {"bytes": 8.0 * n * n_in * (splits + 2) + 8.0 * n * n_in, "flop": 6.0 * n * n_in},
    }
    for name, v in m.items():
        v["hbm_floor_us"] = v["bytes"] / (HBM_GBS * 1e9) * 1e6
        passes = 3 if name == "k_td_learn" else 1            # 3xTF32: three tensor-core products per useful one
        v["tf32_floor_us"] = passes * v["flop"] / (TF32_TFLOPS * 1e12) * 1e6
        v["fp32_floor_us"] = v["flop"] / (FP32_TFLOPS * 1e12) * 1e6
    return m


def run(kind, steps, launches):
    Ag, pcs, td, learn = build(kind)
    A, n, n_in = Ag.n_agents, td.n, pcs.n
    r = {"ms_per_iteration": ms_per_iteration(Ag, pcs, td, learn, steps)}
    times = kernel_times(Ag, pcs, td, learn, launches)
    mod = model(A, n, n_in, rb._lib.load().riab_td_splits(n, n_in, A))      # riab_td_learn's own split
    for k, v in mod.items():
        kk = k + "_tc" if k + "_tc" in times else k            # n > 8: the wgmma learning kernel
        if kk in times:
            us = times[kk]["us"]
            v["kernel"] = kk
            v["us"] = us
            v["gbs"] = v["bytes"] / (us * 1e-6) / 1e9
            v["tflops"] = v["flop"] / (us * 1e-6) / 1e12
            v["frac_of_hbm_floor"] = v["hbm_floor_us"] / us
            v["binds_vs_tf32"] = "hbm" if v["hbm_floor_us"] >= v["tf32_floor_us"] else "tf32"
            v["binds_vs_fp32"] = "hbm" if v["hbm_floor_us"] >= v["fp32_floor_us"] else "fp32"
    r["kernels"] = mod
    r["A"], r["n"], r["n_in"] = A, n, n_in
    del Ag, pcs, td, learn
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--launches", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_td.py measures on a CUDA device")
    res = {"card": bench_ffl.card(), "steps": args.steps, "launches": args.launches}
    for kind in ("c2v", "c2s"):
        res[kind] = run(kind, args.steps, args.launches)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""FeedForwardLayer cost on the c2 workload ("c2f"): c2 (65 536 agents, box + 2 walls, 1024 line-of-sight PlaceCells)
plus a 256-unit linear FeedForwardLayer reading the PlaceCells' rows of the same step.  Prints one JSON line with
  * ms per step of Ag.run for c2 and c2f (same job, CUDA events);
  * the layer kernel's own device time (CUDA events around many riab_ffl_rates launches over the last step's rows),
    its useful 2 A K N rate, the tensor-core rate of its three TF32 passes against the data sheet's 495 TFLOP/s, its
    input bytes against 3.35 TB/s, and which of the two bounds binds;
  * the card's name and power limit, read in the same run.
Writes nothing.
  python scripts/bench_ffl.py [--steps K] [--warmup W] [--n N]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import ratinabox_b200 as rb  # noqa: E402
from ratinabox_b200 import _lib  # noqa: E402

TF32_PEAK_TFLOPS, HBM_PEAK_GBS = 495.0, 3350.0        # H100 SXM data sheet (dense TF32; HBM3)


def build(n_ffl):
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
    pops = bench.build_populations(rb, Ag, wl)
    if n_ffl:
        rng = np.random.default_rng(11)
        f = rb.FeedForwardLayer(Ag, {"n": n_ffl, "name": "FFL"})
        f.add_input(pops[0], w=rng.normal(0, 1 / np.sqrt(pops[0].n), (n_ffl, pops[0].n)))
        pops.append(f)
    return Env, Ag, pops


def ms_per_step(Ag, steps, warmup):
    Ag.run(warmup)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    Ag.run(steps)
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / steps


def kernel_timing(Ag, ffl, launches=50):
    lib = _lib.load()
    A, N = Ag.n_agents, ffl.n
    K = sum(e["layer"].n for e in ffl.inputs.values())
    cells = ffl._cells()                                 # rows: the inputs' last step
    out = torch.empty((A, ffl._ld()), dtype=torch.float32, device="cuda")
    ro = _lib.RatesOut()
    ro.rates_row, ro.ld = out.data_ptr(), ffl._ld()

    def launch():
        _lib.check(lib.riab_ffl_rates(C.byref(cells), A, None, None, C.byref(ro), Ag._stream()))

    for _ in range(5):
        launch()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(launches):
        launch()
    ev1.record()
    torch.cuda.synchronize()
    s = ev0.elapsed_time(ev1) * 1e-3 / launches
    flop, in_bytes = 2.0 * A * K * N, 4.0 * A * K
    t_tc, t_hbm = 3 * flop / (TF32_PEAK_TFLOPS * 1e12), in_bytes / (HBM_PEAK_GBS * 1e9)
    return {"kernel_us": s * 1e6, "launches": launches, "A": A, "K": K, "N": N,
            "useful_tflops": flop / s / 1e12, "tensor_tflops_3pass": 3 * flop / s / 1e12,
            "tensor_peak_tflops": TF32_PEAK_TFLOPS, "input_gbs": in_bytes / s / 1e9, "hbm_peak_gbs": HBM_PEAK_GBS,
            "bound": "tensor" if t_tc >= t_hbm else "hbm", "frac_of_bound": max(t_tc, t_hbm) / s}


def card():
    c = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        c["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--n", type=int, default=256, help="units of the FeedForwardLayer")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_ffl.py measures on a CUDA device")
    res = {"workload": f"c2f: c2 + a {args.n}-unit FeedForwardLayer on its 1024 PlaceCells", "steps": args.steps,
           "card": card()}
    Env, Ag, pops = build(0)
    res["c2_ms_per_step"] = ms_per_step(Ag, args.steps, args.warmup)
    del Env, Ag, pops
    torch.cuda.empty_cache()
    Env, Ag, pops = build(args.n)
    res["c2f_ms_per_step"] = ms_per_step(Ag, args.steps, args.warmup)
    res["ffl"] = kernel_timing(Ag, pops[-1])
    print(json.dumps(res))


if __name__ == "__main__":
    main()

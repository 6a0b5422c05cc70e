"""RandomSpatialNeurons cost on the c2 workload: 65 536 agents in the box with 2 inner walls, lengthscale 0.1
(|X| = 400 sample points, line_of_sight: the reference's geodesic default falls back to it with 2 inner walls).
Prints one JSON line with, per n:
  * ms per step of Ag.run with the RandomSpatialNeurons population alone (CUDA events);
  * the k_rsn device time (CUDA events around 50 riab_rsn_rates launches at the agents' positions);
  * its exp count A |X| n_tiles against the MUFU ex2 issue rate (16 / clk / SM at the boost clock), the rate of its three
    TF32 tensor-core passes against the data sheet's 495 TFLOP/s, its output bytes against 3.35 TB/s, which of the
    three bounds binds, and the (A, |X|) float32 scratch traffic (written once, read once) a two-kernel design would add;
  * the card's name and power limit, read in the same run.
Writes nothing.
  python scripts/bench_rsn.py [--steps K] [--warmup W]"""
import argparse
import ctypes as C
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
from ratinabox_b200 import _lib  # noqa: E402

TF32_PEAK_TFLOPS, HBM_PEAK_GBS = 495.0, 3350.0        # H100 SXM data sheet (dense TF32; HBM3)


def build(n):
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
    N = rb.RandomSpatialNeurons(Ag, {"n": n, "lengthscale": 0.1})
    return Ag, N


def kernel_timing(Ag, N, launches=50):
    lib = _lib.load()
    A, n, K = Ag.n_agents, N.n, N.X.shape[0]
    cells = N._cells()
    out = torch.empty((A, N._ld()), dtype=torch.float32, device="cuda")
    pos = Ag._s["pos"]

    def launch():
        _lib.check(lib.riab_rsn_rates(pos.data_ptr(), A, C.byref(Ag._env_struct()), C.byref(cells), out.data_ptr(),
                                      out.stride(0), Ag._stream()))

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
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    clock_hz = 1.98e9                                     # H100 SXM boost clock
    bn = 8 if n <= 8 else (32 if n <= 32 else 64)
    n_tiles = (n + bn - 1) // bn
    kp = (K + 31) // 32 * 32
    exps = float(A) * kp * n_tiles
    t_mufu = exps / (16.0 * sms * clock_hz)
    flop = 2.0 * A * kp * bn * n_tiles
    t_tc = 3 * flop / (TF32_PEAK_TFLOPS * 1e12)
    out_bytes = 4.0 * A * n
    t_hbm = out_bytes / (HBM_PEAK_GBS * 1e9)
    bounds = {"mufu_ex2": t_mufu, "tensor": t_tc, "hbm": t_hbm}
    bound = max(bounds, key=bounds.get)
    scratch = 2 * 4.0 * A * K
    return {"kernel_us": s * 1e6, "launches": launches, "A": A, "X": K, "n": n, "bn": bn, "n_tiles": n_tiles,
            "exp_count": exps, "ex2_rate_per_s": exps / s, "ex2_bound_us": t_mufu * 1e6,
            "tensor_tflops_3pass": 3 * flop / s / 1e12, "tensor_peak_tflops": TF32_PEAK_TFLOPS, "tensor_bound_us": t_tc * 1e6,
            "output_gbs": out_bytes / s / 1e9, "hbm_peak_gbs": HBM_PEAK_GBS, "hbm_bound_us": t_hbm * 1e6,
            "bound": bound, "frac_of_bound": bounds[bound] / s,
            "avoided_scratch_bytes": scratch, "avoided_scratch_us_at_peak": scratch / (HBM_PEAK_GBS * 1e9) * 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_rsn.py measures on a CUDA device")
    res = {"workload": "c2 box + 2 walls, 65536 agents, RandomSpatialNeurons lengthscale 0.1 (line_of_sight)",
           "steps": args.steps, "card": bench_ffl.card()}
    for n in (10, 256):
        Ag, N = build(n)
        res[f"n{n}_ms_per_step"] = bench_ffl.ms_per_step(Ag, args.steps, args.warmup)
        res[f"n{n}_rsn"] = kernel_timing(Ag, N)
        del Ag, N
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

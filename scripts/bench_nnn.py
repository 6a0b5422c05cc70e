"""NeuralNetworkNeurons cost: PlaceCells(256) + GridCells(128) -> a network, in the open unit box, dt 0.01, for 1 024,
16 384 and 65 536 agents, with the default MLP (hidden [20, 20], 10 outputs) and a 256-wide one (hidden [256, 256]).
Prints one JSON line with, per (agents, network):
  * ms per step of Ag.run with and without the network (same job, CUDA events);
  * the fused kernel's own device time (CUDA events around many riab_nnn_rates launches over the last step's rows)
    against torch's module(X) on the same gathered rows (float32, TF32 off, CUDA events);
  * the kernel's useful FLOP rate (2 A sum(widths[l-1] widths[l])) and its input bytes (4 A n_in) against the data sheet's
    67 TFLOP/s (FP32) and 3.35 TB/s, and which bound binds;
  * the card's name and power limit, read in the same run.
Writes nothing.
  python scripts/bench_nnn.py [--steps K] [--warmup W] [--agents A,A,...]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ratinabox_b200 as rb  # noqa: E402
from ratinabox_b200 import _lib  # noqa: E402
from ratinabox_b200.contribs import MultiLayerPerceptron, NeuralNetworkNeurons  # noqa: E402

FP32_PEAK_TFLOPS, HBM_PEAK_GBS = 67.0, 3350.0        # H100 SXM data sheet (dense FP32; HBM3)
NETS = {"default_mlp": [20, 20], "wide_256": [256, 256]}


def build(A, hidden):
    np.random.seed(1234)
    Ag = rb.Agent(rb.Environment(), {"dt": 0.01, "n_agents": A, "seed": 7})
    lim = {"history_bytes_limit": 64 << 20}
    pc = rb.PlaceCells(Ag, dict(lim, n=256))
    gc = rb.GridCells(Ag, dict(lim, n=128))
    N = None
    if hidden is not None:
        torch.manual_seed(0)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            N = NeuralNetworkNeurons(Ag, dict(lim, input_layers=[pc, gc],
                                              NeuralNetworkModule=MultiLayerPerceptron(384, 10, hidden)))
        assert N.fused
    return Ag, N


def ms_per_step(Ag, steps, warmup):
    Ag.run(warmup)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    Ag.run(steps)
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / steps


def timed(fn, launches):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(launches):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) * 1e-3 / launches


def kernel_timing(Ag, N, launches=100):
    lib = _lib.load()
    A = Ag.n_agents
    cells = N._cells()                                   # rows: the inputs' last step
    out = torch.empty((A, N._ld()), dtype=torch.float32, device="cuda")
    ro = _lib.RatesOut()
    ro.rates_row, ro.ld = out.data_ptr(), N._ld()
    s = timed(lambda: _lib.check(lib.riab_nnn_rates(C.byref(cells), A, None, None, C.byref(ro), Ag._stream())), launches)
    X = N._gather(N._input_rows(), A)
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        s_torch = timed(lambda: N.NeuralNetworkModule(X), launches)
        diff = float((N.NeuralNetworkModule(X) - out[:, : N.n]).abs().max())
    widths = [cells.widths[i] for i in range(cells.n_layers + 1)]
    flop = 2.0 * A * sum(widths[i] * widths[i + 1] for i in range(len(widths) - 1))
    in_bytes = 4.0 * A * widths[0]
    t_fp32, t_hbm = flop / (FP32_PEAK_TFLOPS * 1e12), in_bytes / (HBM_PEAK_GBS * 1e9)
    return {"kernel_us": s * 1e6, "torch_module_us": s_torch * 1e6, "kernel_over_torch": s / s_torch, "launches": launches,
            "widths": widths, "useful_tflops": flop / s / 1e12, "fp32_peak_tflops": FP32_PEAK_TFLOPS,
            "input_gbs": in_bytes / s / 1e9, "hbm_peak_gbs": HBM_PEAK_GBS,
            "bound": "fp32" if t_fp32 >= t_hbm else "hbm", "frac_of_bound": max(t_fp32, t_hbm) / s,
            "max_abs_diff_vs_torch": diff}


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
    ap.add_argument("--agents", default="1024,16384,65536")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_nnn.py measures on a CUDA device")
    res = {"workload": "PlaceCells(256) + GridCells(128) -> NeuralNetworkNeurons, unit box, dt 0.01", "steps": args.steps,
           "card": card(), "runs": []}
    for A in [int(a) for a in args.agents.split(",")]:
        Ag, _ = build(A, None)
        base = ms_per_step(Ag, args.steps, args.warmup)
        del Ag
        for name, hidden in NETS.items():
            Ag, N = build(A, hidden)
            r = {"agents": A, "network": name, "ms_per_step_without": base,
                 "ms_per_step_with": ms_per_step(Ag, args.steps, args.warmup)}
            r.update(kernel_timing(Ag, N))
            res["runs"].append(r)
            del Ag, N
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

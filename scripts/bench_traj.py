"""Cost of the motion sources on the c2 workload (65 536 agents, box + 2 walls, 1024 line-of-sight PlaceCells): Ag.run with
  1. the random motion (c2 itself),
  2. one imported trajectory shared by every agent (2 000 samples),
  3. one imported trajectory per agent (65 536 x 2 000 samples, 4.2 GB of positions and spline coefficients),
built once and measured in alternating rounds in the same job.  Prints one JSON line with
  * us per step of Ag.run (CUDA events; median and all rounds) and the kernel launches of one run() per source;
  * the spline build's device time (CUDA events around riab_trajectory_build, which includes the upload of the host's
    elimination factors) for the per-agent trajectories, and its modelled traffic (read y, write the swept right-hand
    side, read it back, write M: 64 B per sample and trajectory) against 3.35 TB/s;
  * the card's name and power limit, read in the same run.
Writes nothing.
  python scripts/bench_traj.py [--steps K] [--warmup W] [--rounds R]"""
import argparse
import contextlib
import ctypes as C
import gc
import io
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
import ratinabox_b200 as rb  # noqa: E402
from ratinabox_b200 import _lib  # noqa: E402
from bench_ffl import card  # noqa: E402

HBM_PEAK_GBS = 3350.0
T_SAMPLES = 2000


def trajectories(A):
    """2 000 samples at 20-60 ms spacing of a smooth loop inside the box, and per agent the same loop shifted and scaled."""
    rng = np.random.default_rng(3)
    times = np.cumsum(rng.uniform(0.02, 0.06, T_SAMPLES))
    u = np.linspace(0, 12 * np.pi, T_SAMPLES)
    base = np.stack([0.5 + 0.3 * np.cos(u) * np.cos(0.11 * u), 0.5 + 0.3 * np.sin(1.3 * u)], axis=1)
    off = rng.uniform(-0.1, 0.1, (A, 1, 2))
    per_agent = base[None] * rng.uniform(0.8, 1.0, (A, 1, 1)) + off
    return times, base, per_agent


def build(source, traj):
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
    times, base, per_agent = traj
    with contextlib.redirect_stdout(io.StringIO()):           # import_trajectory's messages: the output is one JSON line
        if source == "shared":
            Ag.import_trajectory(times=times, positions=base)
        elif source == "per_agent":
            Ag.import_trajectory(times=times, positions=per_agent)
    return Env, Ag, pops


def us_per_step(Ag, steps, warmup):
    lib = _lib.load()
    Ag.run(warmup)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    c0 = lib.riab_launch_count()
    ev0.record()
    Ag.run(steps)
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) * 1e3 / steps, lib.riab_launch_count() - c0


def build_timing(Ag, repeats=5):
    lib = _lib.load()
    tr = Ag._traj
    xs = tr["times"].cpu().numpy()
    c = tr["c"]

    def launch():
        _lib.check(lib.riab_trajectory_build(C.byref(c), xs.ctypes.data_as(_lib.c_double_p), Ag._stream()))

    launch()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(repeats):
        ev0.record()
        launch()
        ev1.record()
        torch.cuda.synchronize()
        ms.append(ev0.elapsed_time(ev1))
    s = statistics.median(ms) * 1e-3
    nbytes = 64.0 * c.T * c.n_traj
    return {"build_ms": s * 1e3, "T": int(c.T), "n_traj": int(c.n_traj), "model_bytes": nbytes,
            "gbs": nbytes / s / 1e9, "hbm_peak_gbs": HBM_PEAK_GBS, "frac_of_peak": nbytes / s / 1e9 / HBM_PEAK_GBS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_traj.py measures on a CUDA device")
    A = bench.WORKLOADS["c2"]["agents"]
    traj = trajectories(A)
    res = {"workload": "c2 (65 536 agents, 1024 line-of-sight PlaceCells) by motion source", "steps": args.steps,
           "trajectory_samples": T_SAMPLES, "card": card()}
    times = {s: [] for s in ("random", "shared", "per_agent")}
    launches = {}
    for r in range(args.rounds):
        for source in times:
            Env, Ag, pops = build(source, traj)
            us, n = us_per_step(Ag, args.steps, args.warmup)
            times[source].append(us)
            launches[source] = n
            if source == "per_agent" and r == 0:
                res["per_agent_build"] = build_timing(Ag)
            del Env, Ag, pops
            gc.collect()                # the Environment and its Agent reference each other
            torch.cuda.empty_cache()
    for s, v in times.items():
        res[f"{s}_us_per_step"] = statistics.median(v)
        res[f"{s}_us_per_step_rounds"] = v
        res[f"{s}_launches_per_run"] = launches[s]
    print(json.dumps(res))


if __name__ == "__main__":
    main()

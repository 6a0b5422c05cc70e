"""Time of the history analytics through the public API: ``Agent.get_position_heatmap`` and
``Neurons.get_history_rate_maps`` (riab_history_rate_maps), each call timed on the host clock from a device synchronise
to a device synchronise after the call returned (the call itself ends with the copy of the maps to the host).
Cases:
  * full: 65 536 agents in the unit box after Agent.run(1100): the default 1 024-row Agent ring (2^26 samples) and 64
    euclidean PlaceCells with a 256-row ring (2^24 samples);
  * c2:   bench.py's c2 set-up, 65 536 agents in the box with 2 walls and 1 024 line-of-sight PlaceCells with their
    default ring (32 rows at this size, 2^21 samples of 1 024 cells), after Agent.run(40);
each at dx 0.5 (4 bins in the unit box) and 0.05 (441).  Prints one JSON line with every call's time in ms, the medians,
and the card's name and power limit, read in the same run.  Writes nothing.
  python scripts/bench_history_maps.py [--repeats R] [--label NAME]"""
import argparse
import gc
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
import bench_ffl  # noqa: E402
import ratinabox_b200 as rb  # noqa: E402

A = 65536
DXS = (0.5, 0.05)


def setup(case):
    np.random.seed(1234)
    Env = rb.Environment()
    if case == "full":
        Ag = rb.Agent(Env, {"dt": 0.01, "n_agents": A, "seed": 7})
        Ns = rb.PlaceCells(Ag, {"n": 64, "wall_geometry": "euclidean", "history_bytes_limit": 256 * A * 64 * 4})
        Ag.run(1100)
    else:
        walls = bench.WORKLOADS["c2"]["walls"]
        for w in walls:
            Env.add_wall(w)
        Ag = rb.Agent(Env, {"dt": 0.01, "n_agents": A, "seed": 7})
        Ag.pos, Ag.velocity = bench.synthetic_agents(A, walls, 107)
        Ns = rb.PlaceCells(Ag, {"n": 1024, "wall_geometry": "line_of_sight"})
        Ag.run(40)
    torch.cuda.synchronize()
    return Ag, Ns


def timed(fn, repeats):
    fn()                                                   # warm-up: first launch, edge upload, host buffers
    out = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(1e3 * (time.perf_counter() - t0))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_history_maps.py measures on a CUDA device")
    res = {"label": args.label, "repeats": args.repeats, "card": bench_ffl.card(), "ms": {}}
    for case in ("full", "c2"):
        Ag, Ns = setup(case)
        for dx in DXS:
            res["ms"][f"{case}_heatmap_dx{dx}"] = timed(lambda: Ag.get_position_heatmap(dx=dx), args.repeats)
            res["ms"][f"{case}_rate_maps_dx{dx}"] = timed(lambda: Ns.get_history_rate_maps(dx=dx), args.repeats)
        del Ag, Ns
        gc.collect()                                       # the Agent and its populations reference each other
        torch.cuda.empty_cache()
    res["median_ms"] = {k: float(np.median(v)) for k, v in res["ms"].items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

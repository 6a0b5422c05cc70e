"""Cost of the theta modulation of PhasePrecessingPlaceCells: 65 536 agents x 1 024 cells, spikes on, dt 0.01, in the c2
box (2 inner walls, line_of_sight) and in the open box (euclidean).  Arms, all through Agent.run, alternated over
--rounds rounds in one process, timed with CUDA events (µs per step):
  * pppc:          PhasePrecessingPlaceCells (description "gaussian", widths 0.2): the per-step riab_run loop;
  * place_perstep: PlaceCells with the same parameters on the same per-step loop (RIAB_NO_WHOLE_RUN=1);
  * place_whole:   PlaceCells as riab_run's whole-run launch (the c2 headline's path).
Prints one JSON line with every round, the medians, pppc's extra µs over place_perstep, and the card's name and power
limit, read in the same run.  Writes nothing.
  python scripts/bench_pppc.py [--steps K] [--warmup W] [--rounds R]"""
import argparse
import gc
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
from ratinabox_b200.contribs import PhasePrecessingPlaceCells  # noqa: E402

BOXES = {"c2_line_of_sight": (bench.WORKLOADS["c2"]["walls"], "line_of_sight"), "open_euclidean": ([], "euclidean")}
ARMS = ("pppc", "place_perstep", "place_whole")


def build(walls, geom, arm, A=65536, n=1024):
    np.random.seed(1234)
    Env = rb.Environment()
    for w in walls:
        Env.add_wall(w)
    Ag = rb.Agent(Env, {"dt": 0.01, "n_agents": A, "seed": 7})
    pos, vel = bench.synthetic_agents(A, walls, 107)
    Ag.pos, Ag.velocity = pos, vel
    # rings of 4 rows (1 GiB of rates at this size): every arm writes the same rows, and they wrap
    prm = {"n": n, "description": "gaussian", "widths": 0.2, "wall_geometry": geom, "min_fr": 0.0, "max_fr": 1.0,
           "history_bytes_limit": 4 * A * n * 4}
    if arm == "pppc":
        PhasePrecessingPlaceCells(Ag, prm)
    else:
        rb.PlaceCells(Ag, prm)
    return Ag


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_pppc.py measures on a CUDA device")
    res = {"workload": "65536 agents x 1024 cells, gaussian widths 0.2, dt 0.01, history and spikes", "steps": args.steps,
           "rounds": args.rounds, "card": bench_ffl.card()}
    times = {(b, a): [] for b in BOXES for a in ARMS}
    for _ in range(args.rounds):
        for box, (walls, geom) in BOXES.items():
            for arm in ARMS:
                if arm == "place_perstep":
                    os.environ["RIAB_NO_WHOLE_RUN"] = "1"
                else:
                    os.environ.pop("RIAB_NO_WHOLE_RUN", None)
                Ag = build(walls, geom, arm)
                times[(box, arm)].append(1e3 * bench_ffl.ms_per_step(Ag, args.steps, args.warmup))
                del Ag
                gc.collect()                              # the Agent and its populations reference each other
                torch.cuda.empty_cache()
    os.environ.pop("RIAB_NO_WHOLE_RUN", None)
    for box in BOXES:
        med = {arm: float(np.median(times[(box, arm)])) for arm in ARMS}
        res[box] = {"us_per_step": {arm: times[(box, arm)] for arm in ARMS}, "median_us_per_step": med,
                    "pppc_extra_us_vs_place_perstep": med["pppc"] - med["place_perstep"]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

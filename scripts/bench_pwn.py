"""Cost of PlaneWaveNeurons: 65 536 agents x 1 024 cells in the open unit box, dt 0.01, history on, spikes on and off.
Arms, all through Agent.run, alternated over --rounds rounds in one process, timed with CUDA events (µs per step):
  * pwn_whole:         PlaneWaveNeurons (Rayleigh wavescales, scale 0.2: the compensated phase) as riab_run's whole-run
                       launch;
  * pwn_whole_radians: the same population with the radian phase form forced (what the compensated form costs);
  * pwn_whole_dense:   spikes on only: the whole run with RIAB_DENSE_SPIKES=1.  With PwnPolicy::THIN = false it equals
                       pwn_whole; built with THIN = true it is the dense stream against pwn_whole's thinned one (how
                       THIN was chosen, DESIGN.md §1);
  * pwn_perstep:       PlaneWaveNeurons on the per-step riab_run loop (RIAB_NO_WHOLE_RUN=1);
  * grid_whole:        GridCells with n = 1 024 as the whole-run launch.
Prints one JSON line with every round, the medians, and the card's name and power limit, read in the same run.  Writes
nothing.
  python scripts/bench_pwn.py [--steps K] [--warmup W] [--rounds R]"""
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
from ratinabox_b200.contribs import PlaneWaveNeurons  # noqa: E402

ARMS = ("pwn_whole", "pwn_whole_radians", "pwn_whole_dense", "pwn_perstep", "grid_whole")
ENV_OF = {"pwn_perstep": {"RIAB_NO_WHOLE_RUN": "1"}, "pwn_whole_dense": {"RIAB_DENSE_SPIKES": "1"}}


def build(arm, spikes, A=65536, n=1024):
    np.random.seed(1234)
    Ag = rb.Agent(rb.Environment(), {"dt": 0.01, "n_agents": A, "seed": 7})
    pos, vel = bench.synthetic_agents(A, [], 107)
    Ag.pos, Ag.velocity = pos, vel
    # rings of 4 rows (1 GiB of rates at this size): every arm writes the same rows, and they wrap
    prm = {"n": n, "min_fr": 0.0, "max_fr": 1.0, "save_spikes": spikes, "history_bytes_limit": 4 * A * n * 4}
    if arm == "grid_whole":
        rb.GridCells(Ag, prm)
    else:
        N = PlaneWaveNeurons(Ag, prm)
        if arm == "pwn_whole_radians":
            N._phase_form = 0
    return Ag


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_pwn.py measures on a CUDA device")
    res = {"workload": "65536 agents x 1024 cells, open unit box, dt 0.01, history", "steps": args.steps,
           "rounds": args.rounds, "card": bench_ffl.card()}
    cases = [(sp, arm) for sp in (True, False) for arm in ARMS if sp or arm != "pwn_whole_dense"]
    times = {c: [] for c in cases}
    for _ in range(args.rounds):
        for spikes, arm in cases:
            for k in ("RIAB_NO_WHOLE_RUN", "RIAB_DENSE_SPIKES"):
                os.environ.pop(k, None)
            os.environ.update(ENV_OF.get(arm, {}))
            Ag = build(arm, spikes)
            if arm == "pwn_whole":
                res["phase_turns"] = int(Ag.Neurons[0]._cells().phase_turns)
            times[(spikes, arm)].append(1e3 * bench_ffl.ms_per_step(Ag, args.steps, args.warmup))
            del Ag
            gc.collect()                              # the Agent and its populations reference each other
            torch.cuda.empty_cache()
    for k in ("RIAB_NO_WHOLE_RUN", "RIAB_DENSE_SPIKES"):
        os.environ.pop(k, None)
    for spikes in (True, False):
        key = "spikes_on" if spikes else "spikes_off"
        arms = [a for s, a in cases if s == spikes]
        res[key] = {"us_per_step": {a: times[(spikes, a)] for a in arms},
                    "median_us_per_step": {a: float(np.median(times[(spikes, a)])) for a in arms}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Cost of a ThetaSequenceAgent: a lead Agent of 65 536 agents in the open box, dt 0.01, a ThetaSequenceAgent over it and
1 024 PlaceCells(TSA), stepped with the per-step API (Lead.update(); TSA.update(); PCs.update()) over --cycles theta
cycles after --warmup-cycles.  CUDA events time, per step:
  * lead:    Lead.update() (the lead's motion kernel);
  * theta:   riab_theta_seq_step (k_theta_seq: look-behind ring append + sweep position, lazy forward rollouts);
  * forced:  the forced Agent.update that moves the ThetaSequenceAgent to the sweep position;
  * place:   PCs.update() on the ThetaSequenceAgent's positions;
and the whole step.  Reports the mean and median per phase, (theta + forced) / lead, and the card's name and power limit,
read in the same run, as one JSON line.  Writes nothing.
  python scripts/bench_theta_sequence.py [--cycles C] [--warmup-cycles W]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench_ffl  # noqa: E402
import ratinabox_b200 as rb  # noqa: E402
from ratinabox_b200.contribs import ThetaSequenceAgent  # noqa: E402

TIMED = {"riab_theta_seq_step": "theta", "riab_agent_update_src": "forced"}


class _TimedLib:
    """The library as the ThetaSequenceAgent calls it, with CUDA events around its two launches."""

    def __init__(self, lib, marks):
        self._lib, self._marks = lib, marks

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in TIMED:
            return fn

        def timed(*a):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*a)
            e1.record()
            self._marks.append((TIMED[name], e0, e1))
            return rc
        return timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cycles", type=int, default=20)
    ap.add_argument("--warmup-cycles", type=int, default=3)
    ap.add_argument("--agents", type=int, default=65536)
    ap.add_argument("--cells", type=int, default=1024)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_theta_sequence.py measures on a CUDA device")
    np.random.seed(1234)
    Lead = rb.Agent(rb.Environment(), {"dt": 0.01, "n_agents": args.agents, "seed": 7, "save_history": False})
    TSA = ThetaSequenceAgent(Lead, {"seed": 9, "save_history": False})
    PCs = rb.PlaceCells(TSA, {"n": args.cells, "widths": 0.2, "min_fr": 0.0, "max_fr": 1.0, "save_history": False})
    marks = []
    TSA._lib = _TimedLib(TSA._lib, marks)
    steps_per_cycle = int(round(0.1 / 0.01))
    for _ in range(args.warmup_cycles * steps_per_cycle):
        Lead.update(); TSA.update(); PCs.update()
    torch.cuda.synchronize()
    marks.clear()
    per = {k: [] for k in ("lead", "theta", "forced", "place", "step")}
    ev = []
    for _ in range(args.cycles * steps_per_cycle):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record(); Lead.update(); e[1].record(); TSA.update(); e[2].record(); PCs.update(); e[3].record()
        ev.append(e)
    torch.cuda.synchronize()
    for e in ev:
        per["lead"].append(1e3 * e[0].elapsed_time(e[1]))
        per["place"].append(1e3 * e[2].elapsed_time(e[3]))
        per["step"].append(1e3 * e[0].elapsed_time(e[3]))
    for name, e0, e1 in marks:
        per[name].append(1e3 * e0.elapsed_time(e1))
    res = {"workload": f"{args.agents} agents, lead + ThetaSequenceAgent + {args.cells} PlaceCells(TSA), open box, dt 0.01, "
                       "per-step API, no history", "steps": len(ev), "theta_cycles": args.cycles, "card": bench_ffl.card()}
    res["mean_us"] = {k: float(np.mean(v)) for k, v in per.items()}
    res["median_us"] = {k: float(np.median(v)) for k, v in per.items()}
    res["tsa_over_lead"] = (res["mean_us"]["theta"] + res["mean_us"]["forced"]) / res["mean_us"]["lead"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()

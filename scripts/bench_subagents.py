"""Cost of the SubAgents: a lead Agent of 65 536 agents in the open box, dt 0.01, with one DumbAgent, one ShiftAgent
and one ReplayAgent over it, stepped with the per-step API (Lead.update(); D.update(); S.update(); R.update()), no
history.  CUDA events time, per step:
  * lead:           Lead.update() (the lead's motion kernel);
  * shift / dumb:   riab_subagent_step of that kind (k_subagent);
  * replay:         riab_subagent_step of the ReplayAgent (k_subagent, with its lazy sham rollouts);
  * forced:         the forced Agent.update that moves a SubAgent to its position (mean over the three SubAgents).
The ReplayAgent runs at replay_freq 0.3 (the default) and at 5: one agent per thread diverges whenever a warp holds a
replaying lane, and the two rates show what that costs.  Reports the mean and median per phase and the card's name and
power limit, read in the same run, as one JSON line.  Writes nothing.
  python scripts/bench_subagents.py [--steps N] [--warmup W]"""
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
from ratinabox_b200.contribs import DumbAgent, ReplayAgent, ShiftAgent  # noqa: E402

KINDS = {0: "shift", 1: "dumb", 2: "replay"}


class _TimedLib:
    """The library as a SubAgent calls it, with CUDA events around its two launches."""

    def __init__(self, lib, marks):
        self._lib, self._marks = lib, marks

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in ("riab_subagent_step", "riab_agent_update_src"):
            return fn

        def timed(*a):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*a)
            e1.record()
            tag = KINDS[a[0]._obj.kind] if name == "riab_subagent_step" else "forced"
            self._marks.append((tag, e0, e1))
            return rc
        return timed


def run(replay_freq, args):
    np.random.seed(1234)
    Lead = rb.Agent(rb.Environment(), {"dt": 0.01, "n_agents": args.agents, "seed": 7, "save_history": False})
    subs = [DumbAgent(Lead, {"seed": 8, "save_history": False}), ShiftAgent(Lead, {"save_history": False}),
            ReplayAgent(Lead, {"seed": 9, "replay_freq": replay_freq, "save_history": False})]
    marks = []
    for s in subs:
        s._lib = _TimedLib(s._lib, marks)
    for _ in range(args.warmup):
        Lead.update()
        for s in subs:
            s.update()
    torch.cuda.synchronize()
    marks.clear()
    per = {k: [] for k in ("lead", "shift", "dumb", "replay", "forced", "step")}
    ev = []
    replaying = []
    for i in range(args.steps):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record(); Lead.update(); e[1].record()
        for s in subs:
            s.update()
        e[2].record()
        ev.append(e)
        if i % 50 == 0:
            replaying.append(float(subs[2]._replaying.float().mean()))
    torch.cuda.synchronize()
    for e in ev:
        per["lead"].append(1e3 * e[0].elapsed_time(e[1]))
        per["step"].append(1e3 * e[0].elapsed_time(e[2]))
    for name, e0, e1 in marks:
        per[name].append(1e3 * e0.elapsed_time(e1))
    return {"replay_freq": replay_freq, "replaying_share": float(np.mean(replaying)),
            "mean_us": {k: float(np.mean(v)) for k, v in per.items()},
            "median_us": {k: float(np.median(v)) for k, v in per.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--agents", type=int, default=65536)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts/bench_subagents.py measures on a CUDA device")
    res = {"workload": f"{args.agents} agents, lead + DumbAgent + ShiftAgent + ReplayAgent, open box, dt 0.01, per-step "
                       "API, no history", "steps": args.steps, "card": bench_ffl.card(),
           "runs": [run(f, args) for f in (0.3, 5.0)]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""TEST INFRASTRUCTURE -- write tests/golden/nnn.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): ratinabox/contribs/NeuralNetworkNeurons.py.

    python oracle/gen_nnn_golden.py

Records: the default MultiLayerPerceptron built under torch.manual_seed(0) (its state_dict) and the warning text; a user
Sequential Linear-Tanh-Linear-Sigmoid and one whose first Linear has no bias; a seeded native run (Agent + PlaceCells +
GridCells -> NeuralNetworkNeurons, dt 0.05 s) with the positions, the inputs' firing rates and the network's firing rate
per step; get_state at 384 positions and at "all" (every 37th point) with the inputs' rates there; the three ValueError
texts.  The reference's size probe (:66-70) cannot fail after the call that sets n (:52-53) succeeded, so its text is
recorded with a module that refuses its second call; a plain mismatched module raises torch's own error there, whose
type is recorded too.

Neurons.__init__ (ratinabox/Neurons.py:120) calls np.zeros(self.n) while n is still None on the user-module path; NumPy 1.x
read a None shape as (), NumPy 2 raises.  The reference's Neurons module is given that NumPy 1.x reading here, nothing else.
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")


def state(out, key, module):
    sd = module.state_dict()
    out[f"{key}_keys"] = np.array(list(sd.keys()))
    for k, v in sd.items():
        out[f"{key}_sd_{k}"] = v.detach().numpy().copy()


def inputs(out, key, PC, GC):
    out[f"{key}_pc_centres"] = np.array(PC.place_cell_centres, dtype=float)
    out[f"{key}_pc_widths"] = np.array(PC.place_cell_widths, dtype=float)
    out[f"{key}_gc_gridscales"] = np.array(GC.gridscales, dtype=float)
    out[f"{key}_gc_phase_offsets"] = np.array(GC.phase_offsets, dtype=float)
    out[f"{key}_gc_w"] = np.array(GC.w, dtype=float)


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    import torch
    import torch.nn as nn
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import PlaceCells, GridCells
    from ratinabox.contribs.NeuralNetworkNeurons import NeuralNetworkNeurons
    RN = sys.modules["ratinabox.Neurons"]

    class NumPy1Zeros:
        def __getattr__(self, name):
            return getattr(np, name)

        @staticmethod
        def zeros(shape, *args, **kwargs):
            return np.zeros(() if shape is None else shape, *args, **kwargs)
    RN.np = NumPy1Zeros()
    out = {}
    out["default_params_json"] = np.array(json.dumps(NeuralNetworkNeurons.default_params, sort_keys=True, default=str))

    # ---- the native run: PlaceCells(30) + GridCells(12) -> the default MLP with 5 outputs
    np.random.seed(0)
    Env = Environment()
    Ag = Agent(Env, {"dt": 0.05})
    PC = PlaceCells(Ag, {"n": 30})
    GC = GridCells(Ag, {"n": 12})
    torch.manual_seed(0)
    with warnings.catch_warnings(record=True) as ws:
        warnings.simplefilter("always")
        N = NeuralNetworkNeurons(Ag, {"input_layers": [PC, GC], "n": 5})
    out["default_warning"] = np.array([str(w.message) for w in ws if "default MLP" in str(w.message)][0])
    out["mlp_n_in"] = np.array(N.n_in)
    state(out, "mlp", N.NeuralNetworkModule)
    inputs(out, "run", PC, GC)
    rec = {k: [] for k in ("pos", "pc", "gc", "fr", "fr_torch")}
    for _ in range(30):
        Ag.update()
        PC.update()
        GC.update()
        N.update()
        rec["pos"].append(np.array(Ag.pos, dtype=float))
        rec["pc"].append(np.array(PC.firingrate, dtype=float))
        rec["gc"].append(np.array(GC.firingrate, dtype=float))
        rec["fr"].append(np.array(N.firingrate, dtype=float))
        rec["fr_torch"].append(N.firingrate_torch.detach().numpy()[0].astype(float))
    for k, v in rec.items():
        out[f"run_{k}"] = np.array(v)

    # ---- get_state at 384 positions and at "all"
    X = np.random.RandomState(3).uniform(0.0, 1.0, size=(384, 2))
    out["pos_P"] = X
    out["pos_pc"] = PC.get_state(evaluate_at=None, pos=X)
    out["pos_gc"] = GC.get_state(evaluate_at=None, pos=X)
    out["pos_state"] = N.get_state(evaluate_at=None, pos=X)
    out["all_pc"] = PC.get_state(evaluate_at="all")[:, ::37]
    out["all_gc"] = GC.get_state(evaluate_at="all")[:, ::37]
    out["all_state"] = N.get_state(evaluate_at="all")[:, ::37]
    out["all_coords"] = np.array(Env.flattened_discrete_coords, dtype=float)[::37]

    # ---- user Sequentials: Linear-Tanh-Linear-Sigmoid, and a bias-free first Linear
    torch.manual_seed(1)
    seq = nn.Sequential(nn.Linear(42, 16), nn.Tanh(), nn.Linear(16, 3), nn.Sigmoid())
    S = NeuralNetworkNeurons(Ag, {"input_layers": [PC, GC], "NeuralNetworkModule": seq})
    state(out, "seq", seq)
    out["seq_n"] = np.array(S.n)
    out["seq_state"] = S.get_state(evaluate_at=None, pos=X)
    torch.manual_seed(2)
    nob = nn.Sequential(nn.Linear(42, 8, bias=False), nn.ReLU(), nn.Linear(8, 4))
    B = NeuralNetworkNeurons(Ag, {"input_layers": [PC, GC], "NeuralNetworkModule": nob})
    state(out, "nobias", nob)
    out["nobias_state"] = B.get_state(evaluate_at=None, pos=X)

    # ---- the errors
    def text(params):
        try:
            NeuralNetworkNeurons(Ag, params)
        except Exception as e:                       # noqa: BLE001
            return type(e).__name__, str(e)
        raise AssertionError("no error")
    t, out["err_both"] = text({"input_layers": [PC], "n": 3, "NeuralNetworkModule": nn.Linear(30, 3)})
    assert t == "ValueError"
    t, out["err_neither"] = text({"input_layers": [PC]})
    assert t == "ValueError"

    class SecondCallFails(nn.Module):
        calls = 0

        def forward(self, X):
            SecondCallFails.calls += 1
            if SecondCallFails.calls > 1:
                raise RuntimeError("refused")
            return torch.zeros(X.shape[0], 2)
    t, out["err_probe"] = text({"input_layers": [PC], "NeuralNetworkModule": SecondCallFails()})
    assert t == "ValueError"
    t, _ = text({"input_layers": [PC], "NeuralNetworkModule": nn.Linear(31, 2)})
    out["mismatch_error_type"] = np.array(t)
    np.savez_compressed(os.path.join(GOLD, "nnn.npz"), **out)
    print("nnn.npz", os.path.getsize(os.path.join(GOLD, "nnn.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()

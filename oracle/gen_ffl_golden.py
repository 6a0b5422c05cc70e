"""TEST INFRASTRUCTURE -- write tests/golden/ffl.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): FeedForwardLayer (ratinabox/Neurons.py:2654-2847) and utils.activate (utils.py:919-1026).

    python oracle/gen_ffl_golden.py

Contents
  * a native seeded run (box + 2 walls, PlaceCells + GridCells) feeding a two-input layer (F1), a layer stacked on it
    (F2), a self-recurrent layer (R) and a layer registered before its input (Late): every step's rates and primes of
    every population, the weights and biases;
  * get_state(evaluate_at=None, pos=P) of those layers at 384 positions (R with max_recurrence=1);
  * every premade activation with non-default parameters, values and derivatives;
  * an add_input weight draw under a fixed seed;
  * FeedForwardLayer.default_params (JSON).
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
BOX_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
ACTS = {"linear": {}, "sigmoid": {"max_fr": 2.0, "min_fr": 0.5, "mid_x": 0.3, "width_x": 1.5},
        "relu": {"gain": 1.5, "threshold": 0.1}, "tanh": {"gain": 0.8, "threshold": 0.2},
        "retanh": {"gain": 1.3, "threshold": -0.1}, "softmax": {"gain": 1.2, "threshold": -0.3}}
STEPS = 30


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import PlaceCells, GridCells, FeedForwardLayer
    out = {}
    np.random.seed(0)
    Env = Environment()
    for w in BOX_WALLS:
        Env.add_wall(w)
    Ag = Agent(Env, {"dt": 0.05})
    late = FeedForwardLayer(Ag, {"n": 7, "name": "Late", "activation_function": dict(ACTS["relu"], activation="relu")})
    pc = PlaceCells(Ag, {"n": 20, "wall_geometry": "line_of_sight", "name": "PC"})
    gc = GridCells(Ag, {"n": 12, "name": "GC"})
    late.add_input(pc)
    f1 = FeedForwardLayer(Ag, {"n": 10, "name": "F1", "input_layers": [pc, gc],
                               "activation_function": dict(ACTS["sigmoid"], activation="sigmoid"),
                               "biases": np.random.normal(0, 0.3, 10)})
    f2 = FeedForwardLayer(Ag, {"n": 6, "name": "F2", "input_layers": [f1],
                               "activation_function": dict(ACTS["tanh"], activation="tanh")})
    rec = FeedForwardLayer(Ag, {"n": 5, "name": "R", "input_layers": [pc],
                                "activation_function": dict(ACTS["softmax"], activation="softmax")})
    rec.add_input(rec, recurrent=True, w_init_scale=0.5)
    ffls = {"Late": late, "F1": f1, "F2": f2, "R": rec}
    out["pc_centres"], out["pc_widths"] = pc.place_cell_centres, pc.place_cell_widths
    out["gc_gridscales"], out["gc_phase_offsets"], out["gc_w"] = gc.gridscales, gc.phase_offsets, gc.w
    for name, f in ffls.items():
        out[f"{name}_biases"] = np.asarray(f.biases, dtype=np.float64)
        for iname, e in f.inputs.items():
            out[f"{name}_w_{iname}"] = e["w"]
    rates = {k: [] for k in ["PC", "GC"] + list(ffls)}
    primes = {k: [] for k in ffls}
    for _ in range(STEPS):
        Ag.update()
        for N in Ag.Neurons:
            N.update()
        for k, N in zip(["PC", "GC"], [pc, gc]):
            rates[k].append(N.firingrate.copy())
        for k, f in ffls.items():
            rates[k].append(f.firingrate.copy())
            primes[k].append(np.asarray(f.firingrate_prime, dtype=np.float64).copy())
    for k, v in rates.items():
        out[f"run_{k}"] = np.array(v)
    for k, v in primes.items():
        out[f"run_{k}_prime"] = np.array(v)
    P = Env.sample_positions(n=384, method="uniform_jitter")
    out["P"] = P
    for k, f in ffls.items():
        out[f"gs_{k}"] = f.get_state(evaluate_at=None, pos=P, max_recurrence=1)
    out["gs_PC"] = pc.get_state(evaluate_at=None, pos=P)
    out["gs_GC"] = gc.get_state(evaluate_at=None, pos=P)
    # activations
    from ratinabox import utils
    x = np.linspace(-6, 6, 241)
    out["act_x"] = x
    for name, args in ACTS.items():
        a = dict(args, activation=name)
        out[f"act_{name}"] = utils.activate(x, name, False, a)
        out[f"act_{name}_deriv"] = utils.activate(x, name, True, a)
    # add_input draw
    np.random.seed(11)
    f1.add_input(gc, w_init_scale=0.7, name_tag="extra")
    out["draw_seed"], out["draw_n"], out["draw_n_in"], out["draw_scale"] = 11, 10, 12, 0.7
    out["draw_w"] = f1.inputs["GC"]["w"]
    d = {}
    for k, v in FeedForwardLayer.default_params.items():
        try:
            json.dumps(v)
        except TypeError:
            v = repr(v)
        d[k] = v
    out["default_params_json"] = np.array(json.dumps(d, sort_keys=True))
    np.savez_compressed(os.path.join(GOLD, "ffl.npz"), **out)
    print("ffl.npz", len(out), "arrays")


if __name__ == "__main__":
    main()

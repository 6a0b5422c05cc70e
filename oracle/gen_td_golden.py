"""TEST INFRASTRUCTURE -- write tests/golden/td.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py): contribs/ValueNeuron.py and contribs/SuccessorFeatures.py.

    python oracle/gen_td_golden.py

Contents
  * "v_": a seeded 200-step native run in the box with two walls: a ValueNeuron over PlaceCells(20, line_of_sight) and
    GridCells(12), rewarded by a one-cell top_hat PlaceCells, update_weights every step.  Per step: position, the input
    and reward rates, firingrate, firingrate_prime, firingrate_deriv, both traces, td_error; the weights every 10 steps
    (and before the first step); the cells' parameters;
  * "s_": an n = 2 sigmoid ValueNeuron with an explicit tau_e and a self-recurrent input, reset() after step 30 of 60;
  * "f_": SuccessorFeatures of PlaceCells(6) with input_layers=[features, GridCells], 60 steps;
  * the error cases' exception types and texts, and the printed assertion message;
  * both classes' default params (JSON).
"""
import contextlib
import io
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
BOX_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
VN_PARAMS = {"tau": 1.0, "eta": 0.05, "L2": 0.01, "biases": None}
STEPS = 200


def _env():
    from ratinabox.Environment import Environment
    Env = Environment()
    for w in BOX_WALLS:
        Env.add_wall(w)
    return Env


def _record(out, key, rows):
    out[key] = np.array(rows)


def value_run(out):
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import PlaceCells, GridCells
    from ratinabox.contribs.ValueNeuron import ValueNeuron
    np.random.seed(3)
    Ag = Agent(_env(), {"dt": 0.05})
    rew = PlaceCells(Ag, {"n": 1, "description": "top_hat", "widths": 0.3, "place_cell_centres": np.array([[0.5, 0.5]]),
                          "name": "Reward"})
    pc = PlaceCells(Ag, {"n": 20, "wall_geometry": "line_of_sight", "name": "PC"})
    gc = GridCells(Ag, {"n": 12, "name": "GC"})
    vn = ValueNeuron(Ag, dict(VN_PARAMS, input_layers=[pc, gc], biases=np.full(1, 0.5)))
    out["v_pc_centres"], out["v_pc_widths"] = pc.place_cell_centres, pc.place_cell_widths
    out["v_gc_gridscales"], out["v_gc_phase_offsets"], out["v_gc_w"] = gc.gridscales, gc.phase_offsets, gc.w
    out["v_biases"] = np.asarray(vn.biases, dtype=np.float64)
    out["v_pos0"] = Ag.pos.copy()
    rec = {k: [] for k in ["pos", "reward", "PC", "GC", "fr", "prime", "deriv", "e_PC", "e_GC", "td"]}
    W = {"PC": [vn.inputs["PC"]["w"].copy()], "GC": [vn.inputs["GC"]["w"].copy()]}
    for t in range(STEPS):
        Ag.update()
        for N in Ag.Neurons:
            N.update()
        vn.update_weights(rew.firingrate)
        rec["pos"].append(Ag.pos.copy())
        rec["reward"].append(rew.firingrate.copy())
        rec["PC"].append(pc.firingrate.copy())
        rec["GC"].append(gc.firingrate.copy())
        rec["fr"].append(vn.firingrate.copy())
        rec["prime"].append(np.asarray(vn.firingrate_prime, dtype=np.float64).copy())
        rec["deriv"].append(vn.firingrate_deriv.copy())
        rec["e_PC"].append(vn.inputs["PC"]["eligibility_trace"].copy())
        rec["e_GC"].append(vn.inputs["GC"]["eligibility_trace"].copy())
        rec["td"].append(vn.td_error.copy())
        if (t + 1) % 10 == 0:
            for k in W:
                W[k].append(vn.inputs[k]["w"].copy())
    for k, v in rec.items():
        _record(out, f"v_{k}", v)
    for k, v in W.items():
        out[f"v_W_{k}"] = np.array(v)                      # [0] before step 1, [c] after step 10 c
    out["v_tau_e"] = vn.tau_e


def recurrent_run(out):
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import PlaceCells
    from ratinabox.contribs.ValueNeuron import ValueNeuron
    np.random.seed(5)
    Ag = Agent(_env(), {"dt": 0.05})
    pc = PlaceCells(Ag, {"n": 9, "name": "PC"})
    act = {"activation": "sigmoid", "max_fr": 2.0, "min_fr": 0.5, "mid_x": 0.3, "width_x": 1.5}
    vn = ValueNeuron(Ag, {"n": 2, "tau": 0.8, "tau_e": 0.3, "eta": 0.2, "L2": 0.05, "input_layers": [pc],
                          "activation_function": act, "name": "VN"})
    vn.add_input(vn, recurrent=True, w_init_scale=0.5)
    dict.__setitem__(vn.inputs["VN"], "eligibility_trace", np.zeros(2))   # the reference's trace for a late input
    out["s_pc_centres"], out["s_pc_widths"] = pc.place_cell_centres, pc.place_cell_widths
    out["s_W0_PC"], out["s_W0_VN"] = vn.inputs["PC"]["w"].copy(), vn.inputs["VN"]["w"].copy()
    rec = {k: [] for k in ["pos", "PC", "fr", "prime", "deriv", "e_PC", "e_VN", "td", "reward"]}
    for t in range(60):
        Ag.update()
        pc.update()
        vn.update()
        r = np.array([pc.firingrate[0], 0.5])
        vn.update_weights(r)
        rec["reward"].append(r)
        rec["pos"].append(Ag.pos.copy())
        rec["PC"].append(pc.firingrate.copy())
        rec["fr"].append(vn.firingrate.copy())
        rec["prime"].append(np.asarray(vn.firingrate_prime, dtype=np.float64).copy())
        rec["deriv"].append(vn.firingrate_deriv.copy())
        rec["e_PC"].append(vn.inputs["PC"]["eligibility_trace"].copy())
        rec["e_VN"].append(vn.inputs["VN"]["eligibility_trace"].copy())
        rec["td"].append(vn.td_error.copy())
        if t == 29:
            vn.reset()
    for k, v in rec.items():
        _record(out, f"s_{k}", v)
    out["s_W_PC"], out["s_W_VN"] = vn.inputs["PC"]["w"].copy(), vn.inputs["VN"]["w"].copy()


def sf_run(out):
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import PlaceCells, GridCells
    from ratinabox.contribs.SuccessorFeatures import SuccessorFeatures
    np.random.seed(7)
    Ag = Agent(_env(), {"dt": 0.05})
    feat = PlaceCells(Ag, {"n": 6, "name": "Feat", "widths": 0.25})
    gc = GridCells(Ag, {"n": 12, "name": "GC"})
    sf = SuccessorFeatures(Ag, {"features": feat, "input_layers": [feat, gc], "eta": 0.3, "tau_e": 0.2})
    sf.inputs["Feat"]["w"] *= 0.1                                      # the successor-features demo's scaling
    out["f_feat_centres"], out["f_feat_widths"] = feat.place_cell_centres, feat.place_cell_widths
    out["f_gc_gridscales"], out["f_gc_phase_offsets"], out["f_gc_w"] = gc.gridscales, gc.phase_offsets, gc.w
    out["f_W0_Feat"], out["f_W0_GC"] = sf.inputs["Feat"]["w"].copy(), sf.inputs["GC"]["w"].copy()
    out["f_n"] = sf.n
    rec = {k: [] for k in ["pos", "Feat", "GC", "fr", "prime", "deriv", "e_Feat", "e_GC", "td"]}
    for _ in range(60):
        Ag.update()
        feat.update()
        gc.update()
        sf.update()
        sf.update_weights()
        rec["pos"].append(Ag.pos.copy())
        rec["Feat"].append(feat.firingrate.copy())
        rec["GC"].append(gc.firingrate.copy())
        rec["fr"].append(sf.firingrate.copy())
        rec["prime"].append(np.asarray(sf.firingrate_prime, dtype=np.float64).copy())
        rec["deriv"].append(sf.firingrate_deriv.copy())
        rec["e_Feat"].append(sf.inputs["Feat"]["eligibility_trace"].copy())
        rec["e_GC"].append(sf.inputs["GC"]["eligibility_trace"].copy())
        rec["td"].append(sf.td_error.copy())
    for k, v in rec.items():
        _record(out, f"f_{k}", v)
    out["f_W_Feat"], out["f_W_GC"] = sf.inputs["Feat"]["w"].copy(), sf.inputs["GC"]["w"].copy()


def errors(out):
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import PlaceCells
    from ratinabox.contribs.ValueNeuron import ValueNeuron
    from ratinabox.contribs.SuccessorFeatures import SuccessorFeatures
    np.random.seed(9)
    Ag = Agent(_env(), {"dt": 0.05})
    pc = PlaceCells(Ag, {"n": 5, "name": "PC"})
    cases = {}

    def catch(name, fn):
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf):
                fn()
        except Exception as e:      # noqa: BLE001 -- the reference's exception types are the point
            cases[name] = [type(e).__name__, str(e), buf.getvalue()]
        else:
            raise AssertionError(f"{name} did not raise")

    catch("sf_no_features", lambda: SuccessorFeatures(Ag, {"input_layers": [pc]}))
    vz = ValueNeuron(Ag, {"input_layers": [pc], "tau_e": 0, "name": "VZ"})
    Ag.update()
    pc.update()
    catch("tau_e_zero", vz.update)
    vl = ValueNeuron(Ag, {"input_layers": [pc], "name": "VL"})
    vl.add_input(PlaceCells(Ag, {"n": 3, "name": "Late"}))
    catch("late_input", vl.update)
    vr = ValueNeuron(Ag, {"n": 2, "input_layers": [pc], "name": "VR"})
    catch("reward_length", lambda: vr.update_weights(np.zeros(3)))
    out["errors_json"] = np.array(json.dumps(cases, sort_keys=True))


def defaults(out):
    from ratinabox.contribs.ValueNeuron import ValueNeuron
    from ratinabox.contribs.SuccessorFeatures import SuccessorFeatures
    d = {}
    for cls in (ValueNeuron, SuccessorFeatures):
        p = {}
        for k, v in cls.default_params.items():
            try:
                json.dumps(v)
            except TypeError:
                v = repr(v)
            p[k] = v
        d[cls.__name__] = p
    out["default_params_json"] = np.array(json.dumps(d, sort_keys=True))


def main():
    assert ref_shim.import_reference() is not None, "reference not present"
    out = {}
    value_run(out)
    recurrent_run(out)
    sf_run(out)
    errors(out)
    defaults(out)
    np.savez_compressed(os.path.join(GOLD, "td.npz"), **out)
    print("td.npz", len(out), "arrays")


if __name__ == "__main__":
    main()

"""The schedules riab_run picks for Agents with several populations, against the stepped loop.

Each set-up is built four times from the same seeds and stepped four ways after one stepped step:

    run         Ag.run(n)
    run_fused   Ag.run(n) on an Agent with fused_step=True
    step        for: Ag.update(); [N.update() for N in Ag.Neurons]
    step_fused  the same loop with fused_step=True (riab_step_fused for the first population updated)

The four must agree bit for bit on the agent state, every population's rates, both history rings (times included) and
the spike rows.  The launch counter pins which kernels each way runs, per set-up, as a formula in the number of steps n.
GPU only."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

A = 257
STATE = ("pos", "velocity", "rotational_velocity", "measured_velocity", "measured_rotational_velocity",
         "head_direction", "distance_travelled", "distance_to_closest_wall")
WAYS = ("run", "run_fused", "step", "step_fused")


def _agent(rb, fused, walls=True, objects=False):
    np.random.seed(9)
    E = rb.Environment()
    if walls:
        E.add_wall([[0.3, 0.0], [0.3, 0.5]])
        E.add_wall([[0.7, 1.0], [0.7, 0.5]])
    if objects:
        E.add_object([0.15, 0.2])
        E.add_object([0.5, 0.8])
    return rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": 5, "fused_step": fused})


def skewed(rb, fused):
    # population 0 is a Place population: motion(0), then per step Grid, OVC and the skewed Place launch (rates of step s,
    # motion of step s+1); the last step's Place launch is rates only
    Ag = _agent(rb, fused, objects=True)
    rb.PlaceCells(Ag, {"n": 200, "wall_geometry": "line_of_sight"})
    rb.GridCells(Ag, {"n": 64})
    rb.ObjectVectorCells(Ag, {"n": 20})
    return Ag


def bvc_pipelined(rb, fused):
    # every population an allocentric BVC one with a ring of 2 rows: rays(s+1) overlap the integral of step s
    Ag = _agent(rb, fused)
    for name in ("B0", "B1"):
        rb.BoundaryVectorCells(Ag, {"n": 40, "name": name, "history_bytes_limit": 2 * A * 40 * 4})
    return Ag


def bvc_egocentric(rb, fused):
    Ag = _agent(rb, fused)
    rb.FieldOfViewBVCs(Ag, {})
    return Ag


def one_hot_first(rb, fused):
    Ag = _agent(rb, fused)
    rb.PlaceCells(Ag, {"n": 40, "description": "one_hot"})
    rb.GridCells(Ag, {"n": 64})
    return Ag


def feedforward(rb, fused):
    # F0 is population 0 and reads PC (registered after it) one step late; F1 reads PC of the same step
    Ag = _agent(rb, fused)
    with pytest.warns(UserWarning, match="No input layers"):
        f0 = rb.FeedForwardLayer(Ag, {"n": 6, "name": "F0", "input_layers": []})
    pc = rb.PlaceCells(Ag, {"n": 64, "name": "PC"})
    rb.FeedForwardLayer(Ag, {"n": 10, "name": "F1", "input_layers": [pc],
                             "activation_function": {"activation": "sigmoid"}})
    f0.add_input(pc)
    return Ag


def imported(rb, fused):
    Ag = _agent(rb, fused)
    rng = np.random.default_rng(8)
    times = np.cumsum(rng.uniform(0.05, 0.2, 20))
    Ag.import_trajectory(times=times, positions=rng.uniform(0.05, 0.95, (20, 2)))
    rb.PlaceCells(Ag, {"n": 128, "wall_geometry": "line_of_sight"})
    rb.GridCells(Ag, {"n": 64})
    return Ag


def no_populations(rb, fused):
    return _agent(rb, fused)


# set-up: launches of n steps for each way
SETUPS = {
    "skewed": (skewed, lambda n: {"run": 1 + 3 * n, "run_fused": 1 + 3 * n, "step": 4 * n, "step_fused": 3 * n}),
    # per step: motion, then per population the ray and integration kernels (spikes folded into the integral)
    "bvc_pipelined": (bvc_pipelined, lambda n: dict.fromkeys(WAYS, 5 * n)),
    "bvc_egocentric": (bvc_egocentric, lambda n: dict.fromkeys(WAYS, 3 * n)),
    # motion, one_hot and its spike post-pass, Grid
    "one_hot_first": (one_hot_first, lambda n: dict.fromkeys(WAYS, 4 * n)),
    # motion, PC, then per layer the GEMM and its spike post-pass
    "feedforward": (feedforward, lambda n: dict.fromkeys(WAYS, 6 * n)),
    "imported": (imported, lambda n: dict.fromkeys(WAYS, 3 * n)),
    # with fused_step=True no population takes the queued motion step: the first step's runs in the window too
    "no_populations": (no_populations, lambda n: {"run": n, "run_fused": n + 1, "step": n, "step_fused": n + 1}),
}


def _step(Ag):
    Ag.update()
    for N in Ag.Neurons:
        N.update()


def _collect(Ag):
    out = {k: np.asarray(getattr(Ag, k)).copy() for k in STATE}
    out["t"] = Ag.t
    for k, v in Ag.get_history_arrays().items():
        out["agent." + k] = np.asarray(v)
    for i, N in enumerate(Ag.Neurons):
        out[f"{i}.firingrate"] = np.asarray(N.firingrate).copy()
        for k, v in N.get_history_arrays().items():
            out[f"{i}.{k}"] = np.asarray(v)
    return out


@pytest.mark.parametrize("n", [4])
@pytest.mark.parametrize("name", list(SETUPS))
def test_run_equals_the_stepped_loop(name, n):
    import ratinabox_b200 as rb
    from ratinabox_b200 import _lib
    lib = _lib.load()
    build, launches = SETUPS[name]
    res, counts = {}, {}
    for way in WAYS:
        Ag = build(rb, fused=way.endswith("fused"))
        _step(Ag)
        c0 = lib.riab_launch_count()
        if way.startswith("run"):
            Ag.run(n)
        else:
            for _ in range(n):
                _step(Ag)
        res[way] = _collect(Ag)                         # (reading the state runs a queued motion step)
        counts[way] = lib.riab_launch_count() - c0
        if name == "bvc_pipelined":
            assert all(N.history_dropped > 0 for N in Ag.Neurons)      # the 2-row rings wrapped
    assert counts == launches(n), counts
    ref = res["step"]
    for way in WAYS:
        assert res[way].keys() == ref.keys(), way
        for k in ref:
            x, y = np.asarray(res[way][k]), np.asarray(ref[k])
            assert x.shape == y.shape and x.dtype == y.dtype, (way, k, x.shape, y.shape)
            assert np.array_equal(x, y), f"{name}: {way} vs step: {k} differs at {int((x != y).sum())} entries"
    assert any(np.asarray(v).any() for k, v in ref.items() if k.endswith(".spikes")) or name == "no_populations"


def test_refused_fused_step_launches_nothing():
    """riab_step_fused validates everything before the motion kernel: a refused call runs nothing, so the queued motion
    step that Neurons.update() puts back runs once, on the next call."""
    import torch
    import ratinabox_b200 as rb
    from ratinabox_b200 import _lib
    lib = _lib.load()
    Ags = []
    for _ in range(2):
        Ag = _agent(rb, fused=True)
        pc = rb.PlaceCells(Ag, {"n": 64, "name": "PC"})
        f = rb.FeedForwardLayer(Ag, {"n": 10, "name": "F", "input_layers": [pc]})
        _step(Ag)
        Ags.append((Ag, pc, f))
    (Ag, pc, f), (twin, tpc, tf) = Ags
    Ag.update()                                          # queued: the layer's update fuses it
    f._cells().activation = 99
    p0 = Ag._s["pos"].clone()
    c0 = lib.riab_launch_count()
    with pytest.raises(_lib.RiabError, match="activation"):
        f.update()
    torch.cuda.synchronize()
    assert lib.riab_launch_count() == c0
    assert torch.equal(Ag._s["pos"], p0)
    f._cells().activation = _lib.ACTIVATIONS["linear"]
    f.update()
    pc.update()
    twin.update(); tf.update(); tpc.update()
    assert np.array_equal(Ag.pos, twin.pos)
    assert np.array_equal(f.firingrate, tf.firingrate) and np.array_equal(pc.firingrate, tpc.firingrate)

"""Whole-run step kernel (k_step MODE 3, one launch for all of Ag.run(n)) against the per-step paths, the NumPy mirror of
the spike streams and the oracle.  Each case builds the same seeded Environment, Agent and single Place / Grid population
four times and runs the compared steps four ways:

    W  Ag.run(n)                                   whole run: ONE k_step MODE 3 launch where riab_run allows it
    R  Ag.run(n) with RIAB_NO_WHOLE_RUN=1          motion(0), then one skewed MODE 2 launch per step
    S  for: Ag.update(); Ns.update()               k_agent_update + k_step MODE 0 per step
    F  the same loop with fused_step=True          riab_step_fused: k_step MODE 1 per step

Every case states the path W must take and the launch counter checks it.  The four ways must agree bit for bit on the
agent state, the last rates and both history rings; every retained spike row equals the NumPy mirror of its stream, and
the final positions and rates of a sample of agents agree with the float64 oracle.  Batch sizes derive from the device's
SM count so that each case lands in the tile regime it names (small batches get shrunk tiles, see launch_tile).  GPU only.
"""
import numpy as np
import pytest

import riab_oracle as O
from philox_np import agent_normals, expected_spikes_of

pytestmark = pytest.mark.gpu

SEED = 11
# final positions against the oracle fed with the NumPy mirror of the Philox normals (m): the mirror's float32 Box-Muller
# agrees with the GPU's to a few ulps (philox_np.agent_normals); measured up to 1.7e-9 m after 10 steps of 50 ms
POS_TOL = 1e-8
RATE_TOL = 1e-5         # rates against the oracle, relative to max_fr - min_fr
BOX_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
WALLS = {
    0: [],
    1: [[[0.5, 0.0], [0.5, 0.7]]],
    2: BOX_WALLS,
    3: BOX_WALLS + [[[0.0, 0.75], [0.2, 0.75]]],
    7: [[[k / 8, 0.0], [k / 8, 0.6]] if k % 2 else [[k / 8, 1.0], [k / 8, 0.4]] for k in range(1, 8)],
    "aspect2": [[[0.6, 0.0], [0.6, 0.5]], [[1.4, 1.0], [1.4, 0.5]]],
    "free": [[[0.5, 0.2], [0.5, 0.8]]],             # both ends inside the box
}


def lean_groups(n_cells):
    """Consumer groups per CTA of the lean slot loop for n_cells (riab_b200.cu: lean_groups over the padded cells)."""
    ct = -(-n_cells // 128) * 128 // 4
    g = min(4, 512 // ct)
    while 4 % g:
        g -= 1
    return g


def batch(kind, n_cells):
    """Agent counts of the tile regimes (launch_tile: fewer than 4 full slots per (CTA, consumer group) shrink the tiles)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    slots = 32 * sms * lean_groups(n_cells)         # agents of one full 32-agent slot per (CTA, group)
    return {"two": 2, "odd": 37,
            "one_slot": slots // 2,                 # shrunk tiles, one slot per group: one tile per producer warp and step
            "rounds": int(2.5 * slots) | 1,         # shrunk tiles over 3 rounds per group, odd batch
            "full": 4 * slots + 33}[kind]           # full 32-agent tiles and an odd remainder


# name: (kind, n_cells, batch, W's path, extra parameters)
#   walls / geom / aspect / desc / widths / min_fr / max_fr / dt: the set-up (geom: the place cells' wall_geometry,
#   line_of_sight unless given);  steps, pre: compared steps after `pre` stepped ones;
#   rows / agent_rows: history_bytes_limit of the population / Agent in rows (default: the library's limits);
#   off: id_offset;  spikes / history: save_spikes / save_history
CASES = {
    # ---- PlaceCells: every wall template and exponent form of the lean consumers
    "place_euclid_fold_dense": ("place", 512, "one_slot", "whole", dict(walls=0, steps=12)),
    "place_euclid_fold_nospikes": ("place", 512, "odd", "whole", dict(walls=0, spikes=False, steps=12, pre=1)),
    "place_1wall_expanded": ("place", 512, "two", "whole", dict(walls=1, min_fr=0.1, steps=20)),
    "place_2walls_direct_388": ("place", 388, "rounds", "whole", dict(walls=2, widths="per_cell", steps=6)),
    "place_aspect2_direct_wraps": ("place", 1024, "one_slot", "whole", dict(walls="aspect2", steps=10, pre=2, rows=3)),
    "place_3walls_threshold": ("place", 768, "odd", "whole", dict(walls=3, desc="gaussian_threshold", max_fr=3.0,
                                                                  steps=12, pre=2, rows=3, agent_rows=5)),
    "place_7walls_dog": ("place", 512, "one_slot", "whole", dict(walls=7, desc="diff_of_gaussians", widths=0.15, steps=8)),
    "place_2walls_top_hat": ("place", 512, "odd", "whole", dict(walls=2, desc="top_hat", widths=0.3, steps=10)),
    "place_384_idle_warps": ("place", 384, "one_slot", "whole", dict(walls=0, steps=10, rows=2)),
    "place_2048_one_group": ("place", 2048, "rounds", "whole", dict(walls=2, steps=4)),
    "place_even_offset": ("place", 512, "odd", "whole", dict(walls=2, off=64, steps=10)),
    "place_odd_offset": ("place", 512, "odd", "step", dict(walls=2, off=33, steps=10)),
    # geodesic (one inner wall): the compensated direct form with the wall-end block of the agent record
    "place_geodesic_end_on_boundary": ("place", 512, "odd", "whole", dict(walls=1, geom="geodesic", steps=10, pre=2,
                                                                          rows=3)),
    "place_geodesic_free_wall_dog": ("place", 512, "one_slot", "whole", dict(walls="free", geom="geodesic",
                                                                            desc="diff_of_gaussians", steps=8)),
    "place_geodesic_top_hat": ("place", 512, "odd", "whole", dict(walls="free", geom="geodesic", desc="top_hat",
                                                                  widths=0.3, steps=10)),
    "place_geodesic_rounds": ("place", 388, "rounds", "whole", dict(walls=1, geom="geodesic", widths="per_cell",
                                                                    min_fr=0.1, steps=6)),
    "place_no_history": ("place", 512, "one_slot", "whole", dict(walls=2, history=False, steps=10)),
    "place_256_cells": ("place", 256, "odd", "step", dict(walls=2, steps=8)),
    "place_390_cells": ("place", 390, "odd", "step", dict(walls=0, steps=8)),
    "place_one_row_spikes": ("place", 512, "one_slot", "step", dict(walls=0, steps=8, rows=1)),
    # ---- GridCells: thinned stream (dt * max_fr <= 1/16), dense stream by the rate bound, no spikes
    "grid_512_thin_one_row": ("grid", 512, 4096, "step", dict(steps=50, rows=1)),
    "grid_512_thin": ("grid", 512, "one_slot", "whole", dict(steps=30)),
    "grid_1024_thin_wraps": ("grid", 1024, "rounds", "whole", dict(steps=10, pre=2, rows=3)),
    "grid_2048_thin_full_tiles": ("grid", 2048, "full", "whole", dict(steps=3)),
    "grid_1024_dense_by_bound": ("grid", 1024, "odd", "whole", dict(dt=0.05, max_fr=2.0, steps=10)),
    "grid_512_shifted_nospikes": ("grid", 512, "two", "whole", dict(desc="shifted_cosines", spikes=False, steps=20)),
    "grid_512_shifted_two_rows": ("grid", 512, "one_slot", "whole", dict(desc="shifted_cosines", steps=9, pre=1, rows=2)),
    "grid_512_one_row_nospikes": ("grid", 512, "one_slot", "whole", dict(spikes=False, steps=10, rows=1)),
    "grid_768_rings_differ": ("grid", 768, "odd", "whole", dict(steps=12, pre=2, rows=3, agent_rows=5)),
    "grid_even_offset": ("grid", 512, "rounds", "whole", dict(off=128, steps=6)),
    "grid_odd_offset": ("grid", 512, "odd", "step", dict(off=33, steps=10)),
    "grid_256_cells": ("grid", 256, "odd", "step", dict(steps=8)),
    "grid_thin_one_row_two_agents": ("grid", 512, "two", "step", dict(steps=10, rows=1)),
}


def _cell_params(kind, n, p):
    rs = np.random.RandomState(1000 + n)
    if kind == "place":
        aspect = 2.0 if p.get("walls") == "aspect2" else 1.0
        widths = p.get("widths", 0.2)
        if isinstance(widths, str):
            widths = rs.uniform(0.1, 0.25, n)
        return {"n": n, "place_cell_centres": np.stack((rs.uniform(0, aspect, n), rs.uniform(0, 1, n)), axis=1),
                "widths": widths, "description": p.get("desc", "gaussian"), "wall_geometry": p.get("geom", "line_of_sight"),
                "min_fr": p.get("min_fr", 0.0), "max_fr": p.get("max_fr", 1.0)}
    return {"gridscale": rs.uniform(0.2, 1.0, n), "orientation": rs.uniform(0, np.pi / 3, n),
            "phase_offset": rs.uniform(0, 2 * np.pi, (n, 2)), "description": p.get("desc", "rectified_cosines"),
            "min_fr": p.get("min_fr", 0.0), "max_fr": p.get("max_fr", 1.0)}


def build(rb, kind, n, A, p, fused=False, state=None):
    """The case's Environment, Agent and population (identical for every way: seeded, explicit cell parameters).
    `state`: the agents' initial state arrays (a shard of another batch)."""
    np.random.seed(5)
    E = rb.Environment({"aspect": 2.0} if p.get("walls") == "aspect2" else {})
    for w in WALLS[p.get("walls", 0)]:
        E.add_wall(w)
    dt = p.get("dt", 0.01)
    ld = -(-n // 4) * 4
    agent = {"dt": dt, "n_agents": A, "seed": SEED, "id_offset": p.get("off", 0), "fused_step": fused,
             "save_history": p.get("history", True)}
    if "agent_rows" in p:
        agent["history_bytes_limit"] = p["agent_rows"] * A * 32
    Ag = rb.Agent(E, agent)
    if state is not None:
        for k, v in state.items():
            setattr(Ag, k, v)
    cells = dict(_cell_params(kind, n, p), save_spikes=p.get("spikes", True), save_history=p.get("history", True))
    if "rows" in p:
        cells["history_bytes_limit"] = p["rows"] * A * ld * 4
    Ns = (rb.PlaceCells if kind == "place" else rb.GridCells)(Ag, cells)
    return E, Ag, Ns


STATE = ("pos", "velocity", "rotational_velocity", "measured_velocity", "measured_rotational_velocity",
         "head_direction", "distance_travelled", "distance_to_closest_wall")


def run_way(rb, monkeypatch, way, kind, n, A, p, state=None):
    """Runs `pre` stepped steps and then the case's steps the given way; returns (results, launches of the compared steps)."""
    from ratinabox_b200 import _lib
    lib = _lib.load()
    E, Ag, Ns = build(rb, kind, n, A, p, fused=(way == "F"), state=state)
    init = {k: np.asarray(getattr(Ag, k)).copy() for k in STATE}
    for _ in range(p.get("pre", 0)):
        Ag.update(); Ns.update()
    steps = p["steps"]
    c0 = lib.riab_launch_count()
    if way in ("W", "R"):
        with monkeypatch.context() as m:
            if way == "R":
                m.setenv("RIAB_NO_WHOLE_RUN", "1")
            else:
                m.delenv("RIAB_NO_WHOLE_RUN", raising=False)
            Ag.run(steps)
    else:
        for _ in range(steps):
            Ag.update(); Ns.update()
    launches = lib.riab_launch_count() - c0
    out = {k: np.asarray(getattr(Ag, k)).copy() for k in STATE}
    out["firingrate"] = Ns.firingrate
    out["t"] = Ag.t
    for k, v in Ag.get_history_arrays().items():
        out["agent." + k] = v
    out["agent.dropped"] = Ag.history_dropped
    for k, v in Ns.get_history_arrays().items():
        out["pop." + k] = v
    out["pop.dropped"] = Ns.history_dropped
    return out, launches, (E, Ag, Ns, init)


def assert_same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.shape == y.shape and x.dtype == y.dtype, (what, k, x.shape, y.shape)
        if not np.array_equal(x, y):
            bad = np.argwhere(x != y)
            pytest.fail(f"{what}: {k} differs at {len(bad)} entries, first {bad[:3].tolist()}")


def check_spikes(out, Ns, p, A, total, what):
    """Every retained spike row against the NumPy mirror of its stream (row r holds population update total - rows + r)."""
    sp = out["pop.spikes"]
    if not (p.get("spikes", True) and p.get("history", True)):
        assert not sp.any(), what
        return
    dt = p.get("dt", 0.01)
    bound = max(p.get("min_fr", 0.0), p.get("max_fr", 1.0))
    ids = np.arange(A) if A * Ns.n <= (1 << 23) else np.unique(np.linspace(0, A - 1, 512).astype(np.int64))
    rows = sp.shape[0]
    for r in range(rows):
        step = total - rows + r
        want = expected_spikes_of(Ns, SEED, step, p.get("off", 0) + ids, out["pop.firingrate"][r][ids], dt, pop=0,
                                  fr_bound=bound)
        got = sp[r][ids]
        if not np.array_equal(got, want):
            bad = np.argwhere(got != want)
            pytest.fail(f"{what}: spike row of step {step}: {int((got & ~want).sum())} extra, {int((want & ~got).sum())} "
                        f"missing bits, first (agent, cell) {[(int(ids[a]), int(c)) for a, c in bad[:3]]}")
    p_sp = np.clip(dt * out["pop.firingrate"][:, ids].astype(np.float64), 0.0, 1.0)     # (difference of Gaussians dips below 0)
    n_sp, mu, var = sp[:, ids].sum(), p_sp.sum(), (p_sp * (1 - p_sp)).sum()
    assert abs(n_sp - mu) < 6 * np.sqrt(var) + 1, (what, n_sp, mu)


def expected_launches(way, path, steps):
    if way == "W":
        return 1 if path == "whole" else steps + 1     # the per-step loop: motion(0) + one skewed launch per step
    return {"R": steps + 1, "S": 2 * steps, "F": steps}[way]


@pytest.mark.parametrize("name", list(CASES))
def test_whole_run_equals_per_step_paths(name, monkeypatch):
    import ratinabox_b200 as rb
    kind, n, A, path, p = CASES[name]
    A = batch(A, n) if isinstance(A, str) else A
    steps, pre, off = p["steps"], p.get("pre", 0), p.get("off", 0)
    full = state = None
    if off % 2:
        # the same agents as part of an unsharded batch (id_offset 0: even, so a whole run)
        full, launches, objs = run_way(rb, monkeypatch, "W", kind, n, off + A, dict(p, off=0))
        assert launches == 1
        state = {k: v[off:] for k, v in objs[3].items()}
        del objs
    total = pre + steps
    W = None
    for way in ("W", "R", "S", "F"):
        out, launches, objs = run_way(rb, monkeypatch, way, kind, n, A, p, state=state)
        assert launches == expected_launches(way, path, steps), (way, path, launches)
        check_spikes(out, objs[2], p, A, total, way)
        if way == "W":
            E, Ag, Ns, init = objs
            W = out
        else:
            assert_same(W, out, f"W vs {way}")
        del out, objs

    # ---- history bookkeeping: what the rings hold after pre + steps rows
    if p.get("history", True):
        pop_rows = min(total, p.get("rows", total))
        agent_rows = min(total, p.get("agent_rows", total))
        assert W["pop.firingrate"].shape == (pop_rows, A, n) and W["pop.dropped"] == total - pop_rows
        assert W["agent.pos"].shape == (agent_rows, A, 2) and W["agent.dropped"] == total - agent_rows
        assert np.array_equal(W["pop.firingrate"][-1], W["firingrate"])
        assert np.array_equal(W["agent.pos"][-1], W["pos"].astype(np.float32).astype(np.float64))
        assert len(W["pop.t"]) == pop_rows and W["pop.t"][-1] == W["t"] and W["agent.t"][-1] == W["t"]
    else:
        assert W["pop.firingrate"].shape[0] == 0 and W["agent.pos"].shape[0] == 0

    # ---- odd id_offset: the shard (per-step fallback) equals those agents' rows of the unsharded whole run
    if full is not None:
        for k in STATE + ("firingrate",):
            assert np.array_equal(W[k], full[k][off:]), k
        for k in W:
            if k.startswith(("agent.", "pop.")) and k not in ("agent.t", "pop.t", "agent.dropped", "pop.dropped"):
                assert np.array_equal(W[k], full[k][:, off:]), k

    # ---- oracle: final positions of a sample of agents and the rates there
    sample = np.unique(np.linspace(0, A - 1, min(A, 32)).astype(np.int64))     # includes the last (odd) agent
    env = O.OracleEnvironment(aspect=2.0 if p.get("walls") == "aspect2" else 1.0, walls=WALLS[p.get("walls", 0)])
    dt = p.get("dt", 0.01)
    ref_pos = np.zeros((len(sample), 2))
    for k, a in enumerate(sample):
        oa = O.OracleAgent(env, init["pos"][a], init["velocity"][a], {"dt": dt})
        for s in range(total):
            oa.update(O.TapeRNG(agent_xi=agent_normals(SEED, s, np.array([off + a]))[0]))
        ref_pos[k] = oa.pos
    pos = W["pos"][sample]
    worst = np.abs(pos - ref_pos).max()
    assert worst <= POS_TOL, f"positions vs oracle: {worst:.3e} m"
    fr = W["firingrate"][sample]
    span = p.get("max_fr", 1.0) - p.get("min_fr", 0.0)
    if kind == "place":
        geom = "euclidean" if p.get("walls", 0) == 0 else p.get("geom", "line_of_sight")
        assert Ns._effective_geometry() == geom
        desc = p.get("desc", "gaussian")
        scalar = Ns.widths if np.isscalar(Ns.widths) else None
        ref = O.place_cells_get_state(env, Ns.place_cell_centres, Ns.place_cell_widths, pos, O.TapeRNG(), desc, geom,
                                      p.get("min_fr", 0.0), p.get("max_fr", 1.0), scalar_width=scalar).T
        if geom != "euclidean":
            blocked = O.distances_accounting_for_environment(env, Ns.place_cell_centres, pos, "line_of_sight",
                                                             O.TapeRNG()).T == 1000
            assert blocked.mean() > 0.02, blocked.mean()        # the wall shadows are exercised
    else:
        ref = O.grid_cells_get_state(Ns.gridscales, Ns.phase_offsets, Ns.w, pos, p.get("desc", "rectified_cosines"),
                                     min_fr=p.get("min_fr", 0.0), max_fr=p.get("max_fr", 1.0)).T
    err = np.abs(fr - ref)
    assert err.max() <= RATE_TOL * span, f"rates vs oracle: {err.max():.3e}"
    if kind == "place" and p.get("desc", "gaussian") == "gaussian":
        big = np.abs(ref) > 1e-3 * span
        assert big.any()
        rel = (err[big] / np.abs(ref[big])).max()
        assert rel <= RATE_TOL, f"rates vs oracle: max rel err {rel:.3e}"

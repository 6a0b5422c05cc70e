"""Parity at BASELINE.json's full sizes (configs[1..3]): the CUDA path stepped with its production
Philox stream, checked against the oracle on a sample of agents (all cells) plus size-independent
properties on the whole batch.  GPU only."""
import numpy as np
import pytest

import riab_oracle as O
from philox_np import agent_normals, expected_spikes_of

pytestmark = pytest.mark.gpu

BOX_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]


def maze_walls(n=8, length=0.6):
    out = []
    for k in range(1, n + 1):
        x = k / (n + 1)
        out.append([[x, 0.0], [x, length]] if k % 2 else [[x, 1.0], [x, 1.0 - length]])
    return out


def _pure_relative(got, ref, scale, what):
    """north_star's "<= 1e-5 relative" leg: entries above 1e-3 of the rate scale also agree to 1e-5 of their own value
    (below that, float32 differences of O(1) terms have no meaningful relative error)."""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    big = np.abs(ref) > 1e-3 * scale
    assert big.any(), what
    rel = (np.abs(got - ref)[big] / np.abs(ref[big])).max()
    assert rel <= 1e-5, f"{what}: max rel err {rel:.3e}"


def _setup(rb, A, walls, seed=21):
    np.random.seed(seed)
    E = rb.Environment()
    for w in walls:
        E.add_wall(w)
    Ag = rb.Agent(E, {"dt": 0.01, "n_agents": A, "seed": 5})
    return E, Ag


def _oracle_positions(walls, pos0, vel0, sample, steps, seed=5):
    env = O.OracleEnvironment(walls=walls)
    out = np.zeros((len(sample), 2))
    for k, a in enumerate(sample):
        oa = O.OracleAgent(env, pos0[a], vel0[a], {"dt": 0.01})
        for s in range(steps):
            oa.update(O.TapeRNG(agent_xi=agent_normals(seed, s, np.array([a]))[0]))
        out[k] = oa.pos
    return env, out


def test_config2_65536_agents_1024_place_cells_line_of_sight():
    import ratinabox_b200 as rb
    A, N, steps = 65536, 1024, 4
    E, Ag = _setup(rb, A, BOX_WALLS)
    pos0, vel0 = Ag.pos.copy(), Ag.velocity.copy()
    PCs = rb.PlaceCells(Ag, {"n": N})
    assert PCs.wall_geometry == "line_of_sight"            # reference default for a 6-wall box (Neurons.py:922-928)
    Ag.run(steps)
    pos, fr = Ag.pos, PCs.firingrate
    assert fr.shape == (A, N)
    # ---- whole-batch properties
    assert np.isfinite(pos).all() and (pos > 0).all() and (pos < 1).all()
    assert np.isfinite(fr).all() and fr.min() >= 0.0 and fr.max() <= 1.0 + 1e-6
    h = PCs.get_history_arrays()
    assert np.array_equal(h["firingrate"][-1], fr)         # the last history row IS the step's output
    p_spike = 0.01 * h["firingrate"][-1].astype(np.float64)
    n_sp, mu, var = h["spikes"][-1].sum(), p_spike.sum(), (p_spike * (1 - p_spike)).sum()
    assert abs(n_sp - mu) < 6 * np.sqrt(var), (n_sp, mu)    # Bernoulli(dt*rate) spikes (Neurons.py:682-684)
    # ---- sample of agents, every cell, against the oracle
    sample = np.random.RandomState(0).choice(A, 768, replace=False)
    env, ref_pos = _oracle_positions(BOX_WALLS, pos0, vel0, sample, steps)
    assert np.abs(pos[sample] - ref_pos).max() <= 1e-6
    ref = O.place_cells_get_state(env, PCs.place_cell_centres, PCs.place_cell_widths, pos[sample], O.TapeRNG(),
                                  "gaussian", "line_of_sight").T
    err = np.abs(fr[sample] - ref)
    assert err.max() <= 1e-5, err.max()
    _pure_relative(fr[sample], ref, 1.0, "config 2 PlaceCells")
    blocked = O.distances_accounting_for_environment(env, PCs.place_cell_centres, pos[sample], "line_of_sight",
                                                     O.TapeRNG()).T == 1000
    assert blocked.mean() > 0.05                            # the wall shadows are exercised
    assert np.array_equal(fr[sample][blocked] < 1e-30, np.ones(blocked.sum(), dtype=bool))


def test_config3_65536_agents_1024_grid_cells():
    import ratinabox_b200 as rb
    A, N, steps = 65536, 1024, 3
    E, Ag = _setup(rb, A, [])
    pos0, vel0 = Ag.pos.copy(), Ag.velocity.copy()
    rs = np.random.RandomState(3)
    GCs = rb.GridCells(Ag, {"gridscale": rs.uniform(0.2, 1.0, N), "orientation": rs.uniform(0, np.pi / 3, N),
                            "phase_offset": rs.uniform(0, 2 * np.pi, (N, 2))})
    Ag.run(steps)
    pos, fr = Ag.pos, GCs.firingrate
    assert fr.shape == (A, N) and np.isfinite(fr).all() and fr.min() >= 0 and fr.max() <= 1 + 1e-6
    sample = np.random.RandomState(1).choice(A, 512, replace=False)
    env, ref_pos = _oracle_positions([], pos0, vel0, sample, steps)
    assert np.abs(pos[sample] - ref_pos).max() <= 1e-6
    ref = O.grid_cells_get_state(GCs.gridscales, GCs.phase_offsets, GCs.w, pos[sample]).T
    assert np.abs(fr[sample] - ref).max() <= 1e-5
    # the whole run's thinned spike stream (dt * max_fr = 0.01): the last row bit for bit against the NumPy mirror
    h = GCs.get_history_arrays()
    assert np.array_equal(h["firingrate"][-1], fr)
    want = expected_spikes_of(GCs, 5, steps - 1, sample, fr[sample], 0.01, fr_bound=1.0)
    assert np.array_equal(h["spikes"][-1][sample], want)
    assert want.any()


def _ring_spikes(ns, slot, agents):
    """Spike bits of ring row `slot` for some agents (get_history_arrays' unpacking: bit L of word 4B+i = cell 128B+4L+i)."""
    import torch
    words = ns._spk[slot][torch.as_tensor(agents, device=ns._spk.device)].cpu().numpy().view(np.uint32)
    bits = np.unpackbits(words.view(np.uint8), axis=-1, bitorder="little")
    return bits.reshape(len(agents), -1, 4, 32).transpose(0, 1, 3, 2).reshape(len(agents), -1)[:, : ns.n].astype(bool)


def test_config3_whole_run_wraps_the_default_ring():
    """configs[2]'s population at full size, 40 steps of Ag.run after 3 stepped ones: a 65 536 x 1 024 rate row is 256 MiB,
    so the default 8 GiB history_bytes_limit holds 32 rows and the whole run (one launch) wraps its rings in the middle.
    The last row is the step's output and the last two retained rows carry the thinned spikes of their steps."""
    import torch
    import ratinabox_b200 as rb
    from ratinabox_b200 import _lib
    lib = _lib.load()
    A, N, pre, steps = 65536, 1024, 3, 40
    E, Ag = _setup(rb, A, [])
    pos0, vel0 = Ag.pos.copy(), Ag.velocity.copy()
    rs = np.random.RandomState(3)
    GCs = rb.GridCells(Ag, {"gridscale": rs.uniform(0.2, 1.0, N), "orientation": rs.uniform(0, np.pi / 3, N),
                            "phase_offset": rs.uniform(0, 2 * np.pi, (N, 2))})
    for _ in range(pre):
        Ag.update(); GCs.update()
    c0 = lib.riab_launch_count()
    Ag.run(steps)
    assert lib.riab_launch_count() - c0 == 1                 # k_step MODE 3
    total = pre + steps
    cap = GCs._hist_cap
    assert cap == (8 << 30) // (A * N * 4) == 32 and GCs._hist_rows == total
    ha = Ag.get_history_arrays()
    assert Ag.history_dropped == 0 and ha["pos"].shape == (total, A, 2)
    last = (total - 1) % cap
    fr = GCs.firingrate
    assert np.array_equal(GCs._hist[last][:, :N].cpu().numpy().astype(np.float64), fr)
    sample = np.random.RandomState(6).choice(A, 256, replace=False)
    for k in (1, 2):
        slot = (total - k) % cap
        rates = GCs._hist[slot][torch.as_tensor(sample, device=GCs._hist.device), :N].cpu().numpy()
        want = expected_spikes_of(GCs, 5, total - k, sample, rates, 0.01, fr_bound=1.0)
        assert np.array_equal(_ring_spikes(GCs, slot, sample), want), k
    torch.cuda.synchronize()
    env, ref_pos = _oracle_positions([], pos0, vel0, sample[:64], total)
    assert np.abs(Ag.pos[sample[:64]] - ref_pos).max() <= 1e-6
    ref = O.grid_cells_get_state(GCs.gridscales, GCs.phase_offsets, GCs.w, Ag.pos[sample]).T
    assert np.abs(fr[sample] - ref).max() <= 1e-5


def test_config4_16384_agents_512_bvcs_maze():
    import ratinabox_b200 as rb
    A, N, steps = 16384, 512, 2
    walls = maze_walls()
    E, Ag = _setup(rb, A, walls)
    pos0, vel0 = Ag.pos.copy(), Ag.velocity.copy()
    BVCs = rb.BoundaryVectorCells(Ag, {"n": N})
    Ag.run(steps)
    pos, fr = Ag.pos, BVCs.firingrate
    assert fr.shape == (A, N) and np.isfinite(fr).all() and fr.min() >= 0
    sample = np.random.RandomState(2).choice(A, 192, replace=False)
    env, ref_pos = _oracle_positions(walls, pos0, vel0, sample, steps)
    assert np.abs(pos[sample] - ref_pos).max() <= 1e-6
    ref = O.bvc_get_state(env, BVCs.tuning_distances, BVCs.tuning_angles, BVCs.sigma_distances, BVCs.sigma_angles,
                          pos[sample], O.TapeRNG()).T
    assert np.abs(fr[sample] - ref).max() <= 1e-5
    _pure_relative(fr[sample], ref, 1.0, "config 4 BVCs")
    # spikes are drawn in the integration kernel's epilogue: Bernoulli(dt * rate) (Neurons.py:682-684)
    h = BVCs.get_history_arrays()
    p_spike = 0.01 * h["firingrate"][-1].astype(np.float64)
    n_sp, mu, var = h["spikes"][-1].sum(), p_spike.sum(), (p_spike * (1 - p_spike)).sum()
    assert abs(n_sp - mu) < 6 * np.sqrt(var), (n_sp, mu)


def test_config5_shard_32768_agents_three_populations():
    """configs[4] (262 144 agents over 8 GPUs) as one GPU sees it: a 32 768-agent shard with global ids
    32768..65535 and 512 Place (line_of_sight) + 512 Grid + 256 BVC populations on one Agent."""
    import ratinabox_b200 as rb
    A, steps, off = 32768, 3, 32768
    np.random.seed(8)
    E = rb.Environment()
    for w in BOX_WALLS:
        E.add_wall(w)
    Ag = rb.Agent(E, {"dt": 0.01, "n_agents": A, "seed": 5, "id_offset": off})
    pos0, vel0 = Ag.pos.copy(), Ag.velocity.copy()
    PCs = rb.PlaceCells(Ag, {"n": 512})
    GCs = rb.GridCells(Ag, {"n": 512})
    BVCs = rb.BoundaryVectorCells(Ag, {"n": 256})
    Ag.run(steps)
    pos = Ag.pos
    sample = np.random.RandomState(4).choice(A, 160, replace=False)
    env = O.OracleEnvironment(walls=BOX_WALLS)
    ref_pos = np.zeros((len(sample), 2))
    for k, a in enumerate(sample):                         # Philox streams are keyed on the GLOBAL agent id
        oa = O.OracleAgent(env, pos0[a], vel0[a], {"dt": 0.01})
        for s in range(steps):
            oa.update(O.TapeRNG(agent_xi=agent_normals(5, s, np.array([off + a]))[0]))
        ref_pos[k] = oa.pos
    assert np.abs(pos[sample] - ref_pos).max() <= 1e-6
    rng = O.TapeRNG()
    ps = pos[sample]
    assert np.abs(PCs.firingrate[sample] - O.place_cells_get_state(env, PCs.place_cell_centres, PCs.place_cell_widths, ps, rng,
                                                                   "gaussian", "line_of_sight").T).max() <= 1e-5
    assert np.abs(GCs.firingrate[sample] - O.grid_cells_get_state(GCs.gridscales, GCs.phase_offsets, GCs.w, ps).T).max() <= 1e-5
    assert np.abs(BVCs.firingrate[sample] - O.bvc_get_state(env, BVCs.tuning_distances, BVCs.tuning_angles,
                                                            BVCs.sigma_distances, BVCs.sigma_angles, ps, rng).T).max() <= 1e-5
    for ns in (PCs, GCs, BVCs):
        h = ns.get_history_arrays()
        assert h["firingrate"].shape == (steps, A, ns.n) and h["spikes"].shape == (steps, A, ns.n)
        assert np.array_equal(h["firingrate"][-1], ns.firingrate)

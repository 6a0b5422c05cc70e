"""End-to-end behaviour of the engine through the reference-shaped Python API
(fused step, riab_run, Philox streams, spikes, history, attribute mutability) checked
against the CPU oracle.  GPU only."""
import numpy as np
import pytest

import riab_oracle as O
from philox_np import agent_normals, expected_spikes, expected_spikes_of

pytestmark = pytest.mark.gpu

BOX_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]


def make(rb, A, walls=BOX_WALLS, seed=3, **agent_params):
    np.random.seed(seed)
    E = rb.Environment()
    for w in walls:
        E.add_wall(w)
    Ag = rb.Agent(E, dict({"dt": 0.01, "n_agents": A, "seed": 11}, **agent_params))
    return E, Ag


def oracle_step(env, pos, vel, xi, dt=0.01, **state):
    oa = O.OracleAgent(env, pos, vel, {"dt": dt})
    for k, v in state.items():
        setattr(oa, k, v)
    info = oa.update(O.TapeRNG(agent_xi=xi))
    return oa, info


@pytest.mark.parametrize("fused", [True, False])
def test_fused_step_all_cell_types(fused):
    """Ag.update(); Ns.update() -> fused_step=True: one fused kernel per (motion, cell type) (riab_step_fused);
    False (default): the motion kernel is launched by update() and the populations' rate kernels follow.  Either way
    every population of the same Agent sees the same new positions."""
    import ratinabox_b200 as rb
    A = 200
    E, Ag = make(rb, A, fused_step=fused)
    pos0, vel0 = Ag.pos.copy(), Ag.velocity.copy()
    PCs = rb.PlaceCells(Ag, {"n": 150, "wall_geometry": "line_of_sight"})
    GCs = rb.GridCells(Ag, {"n": 60})
    BVCs = rb.BoundaryVectorCells(Ag, {"n": 40})
    xi = np.random.RandomState(5).normal(size=(A, 2))
    Ag.update(_xi=xi)
    PCs.update(); GCs.update(); BVCs.update()
    pos1 = Ag.pos
    env = O.OracleEnvironment(walls=BOX_WALLS)
    ref_pos = np.zeros((A, 2))
    for a in range(A):
        oa, _ = oracle_step(env, pos0[a], vel0[a], xi[a])
        ref_pos[a] = oa.pos
    assert np.abs(pos1 - ref_pos).max() <= 1e-12
    rng = O.TapeRNG()
    ref_pc = O.place_cells_get_state(env, PCs.place_cell_centres, PCs.place_cell_widths, ref_pos, rng, "gaussian", "line_of_sight")
    ref_gc = O.grid_cells_get_state(GCs.gridscales, GCs.phase_offsets, GCs.w, ref_pos)
    ref_bvc = O.bvc_get_state(env, BVCs.tuning_distances, BVCs.tuning_angles, BVCs.sigma_distances, BVCs.sigma_angles, ref_pos, rng)
    assert np.abs(PCs.firingrate - ref_pc.T).max() <= 1e-5
    assert np.abs(GCs.firingrate - ref_gc.T).max() <= 1e-5
    assert np.abs(BVCs.firingrate - ref_bvc.T).max() <= 1e-5
    assert PCs.firingrate.shape == (A, 150)


def test_philox_stream_and_run_equals_stepping():
    """Production RNG: Philox4x32-10 keyed on (seed, step, global agent id).  The GPU draws
    equal the NumPy mirror's, so the oracle fed with them tracks the GPU; riab_run (C loop)
    equals per-step Python calls bit for bit; results do not depend on how agents are sharded."""
    import ratinabox_b200 as rb
    A, steps = 96, 25
    E, Ag = make(rb, A)
    pos0, vel0 = Ag.pos.copy(), Ag.velocity.copy()
    PCs = rb.PlaceCells(Ag, {"n": 64})
    Ag.run(steps)
    pos_run, fr_run = Ag.pos, PCs.firingrate
    hist_run = Ag.get_history_arrays()["pos"]

    E2, Ag2 = make(rb, A)
    Ag2.pos, Ag2.velocity, Ag2.measured_velocity = pos0, vel0, vel0
    PCs2 = rb.PlaceCells(Ag2, {"place_cell_centres": PCs.place_cell_centres})
    for _ in range(steps):
        Ag2.update(); PCs2.update()
    assert np.array_equal(Ag2.pos, pos_run)
    assert np.array_equal(PCs2.firingrate, fr_run)
    assert np.array_equal(Ag2.get_history_arrays()["pos"], hist_run)
    assert np.array_equal(PCs2.get_history_arrays()["spikes"], PCs.get_history_arrays()["spikes"])

    # sharding invariance: the second half of the agents as its own shard (id_offset = A/2)
    E3, Ag3 = make(rb, A // 2, id_offset=A // 2)
    Ag3.pos, Ag3.velocity, Ag3.measured_velocity = pos0[A // 2:], vel0[A // 2:], vel0[A // 2:]
    Ag3.run(steps)
    assert np.array_equal(Ag3.pos, pos_run[A // 2:])

    # oracle driven by the NumPy mirror of the Philox stream
    env = O.OracleEnvironment(walls=BOX_WALLS)
    worst = 0.0
    for a in range(0, A, 7):
        oa = O.OracleAgent(env, pos0[a], vel0[a], {"dt": 0.01})
        for s in range(steps):
            oa.update(O.TapeRNG(agent_xi=agent_normals(11, s, np.array([a]))[0]))
        worst = max(worst, np.abs(oa.pos - pos_run[a]).max())
    # the GPU's float32 Box-Muller and the NumPy mirror agree to a few float32 ulps of the normals
    assert worst <= 1e-7, worst


def test_spikes_match_numpy_philox():
    """Neurons.save_to_history spikes: uniform < dt*firingrate (Neurons.py:682-684) with the
    Philox4x32-7 spike stream; bit-packed on the device, unpacked by get_history_arrays."""
    import ratinabox_b200 as rb
    A, N = 40, 100
    E, Ag = make(rb, A, dt=0.05)
    PCs = rb.PlaceCells(Ag, {"n": N, "max_fr": 15.0, "widths": 0.3})
    for _ in range(3):
        Ag.update(); PCs.update()
    h = PCs.get_history_arrays()
    assert h["firingrate"].shape == (3, A, N) and h["spikes"].shape == (3, A, N) and h["spikes"].dtype == bool
    for s in range(3):
        want = expected_spikes_of(PCs, 11, s, np.arange(A), h["firingrate"][s], 0.05, pop=0, fr_bound=15.0)
        assert np.array_equal(h["spikes"][s], want), s
    assert 0.02 < h["spikes"].mean() < 0.6


@pytest.mark.parametrize("A,N,stepped", [(131, 300, False), (64, 1024, False), (70, 128, True), (33, 2304, False)])
def test_thinned_spikes_match_numpy_mirror(A, N, stepped):
    """GridCells without OU noise and dt * max_fr <= 1/16 (here 0.01 * 3 Hz) use the thinned spike stream
    (Binomial(128, dt*max_fr) candidates per (agent, 128-cell block) at uniformly drawn distinct cells, accepted with
    rate/max_fr; riab_b200.cu: thin_block); the PlaceCells next to them keep the dense stream.  Both bit-equal to their NumPy
    mirrors for odd agent counts, ragged cell counts, several cell chunks (N > 2048), riab_run and the stepped API; both
    Bernoulli(dt * rate) (Neurons.py:682-684)."""
    import ratinabox_b200 as rb
    E, Ag = make(rb, A)
    PCs = rb.PlaceCells(Ag, {"n": N, "wall_geometry": "line_of_sight"})
    GCs = rb.GridCells(Ag, {"n": N, "max_fr": 3.0})
    steps = 3
    if stepped:
        for _ in range(steps):
            Ag.update(); PCs.update(); GCs.update()
    else:
        Ag.run(steps)
    for pop, (Ns, bound) in enumerate(((PCs, 1.0), (GCs, 3.0))):
        h = Ns.get_history_arrays()
        for s in range(steps):
            want = expected_spikes_of(Ns, 11, s, np.arange(A), h["firingrate"][s].reshape(A, Ns.n), 0.01, pop=pop, fr_bound=bound)
            assert np.array_equal(h["spikes"][s].reshape(A, Ns.n), want), (pop, s)
        p = 0.01 * h["firingrate"].astype(np.float64)
        n_sp, mu, var = h["spikes"].sum(), p.sum(), (p * (1 - p)).sum()
        assert abs(n_sp - mu) < 6 * np.sqrt(var) + 1, (n_sp, mu)


def test_dense_spike_stream_on_request(monkeypatch):
    """RIAB_DENSE_SPIKES=1 keeps the dense stream (one threshold test per rate in the pair loop) for GridCells too:
    bit-equal to its NumPy mirror through the lean consumers and riab_run."""
    import ratinabox_b200 as rb
    monkeypatch.setenv("RIAB_DENSE_SPIKES", "1")
    A = 96
    E, Ag = make(rb, A)
    GCs = rb.GridCells(Ag, {"n": 512})
    Ag.run(2)
    h = GCs.get_history_arrays()
    for s in range(2):
        want = expected_spikes_of(GCs, 11, s, np.arange(A), h["firingrate"][s], 0.01, pop=0, fr_bound=1.0)
        assert np.array_equal(h["spikes"][s], want), s


def test_multistep_tracking_config1():
    """Config 1 (1 agent, default box, 100 Gaussian PlaceCells, dt = 10 ms), 3000 steps with the
    same injected normals: the float64 GPU trajectory tracks the oracle to <= 1e-6 m throughout."""
    import ratinabox_b200 as rb
    np.random.seed(0)
    E = rb.Environment()
    Ag = rb.Agent(E, {"dt": 0.01})
    PCs = rb.PlaceCells(Ag, {"n": 100})
    assert PCs.wall_geometry == "geodesic"
    pos0, vel0 = Ag.pos.copy(), Ag.velocity.copy()
    assert pos0.shape == (2,)
    steps = 3000
    xi = np.random.RandomState(9).normal(size=(steps, 2))
    for s in range(steps):
        Ag.update(_xi=xi[s])
        PCs.update()
    h = Ag.get_history_arrays()
    assert h["pos"].shape == (steps, 2) and h["t"].shape == (steps,)
    env = O.OracleEnvironment()
    oa = O.OracleAgent(env, pos0, vel0, {"dt": 0.01})
    on = O.OracleNeurons(oa, 100, lambda p, r: O.place_cells_get_state(env, PCs.place_cell_centres, PCs.place_cell_widths, p, r))
    for s in range(steps):
        oa.update(O.TapeRNG(agent_xi=xi[s]))
        on.update(O.TapeRNG())
    ref = np.array(oa.history["pos"])
    assert np.abs(Ag.pos - oa.pos).max() <= 1e-9
    assert np.abs(h["pos"] - ref).max() <= 1e-6            # history rows are float32
    assert np.abs(h["rot_vel"] - np.array(oa.history["rot_vel"])).max() <= 2e-4 * np.abs(oa.history["rot_vel"]).max()
    assert np.abs(h["head_direction"] - np.array(oa.history["head_direction"])).max() <= 1e-6
    assert np.abs(h["distance_travelled"] - np.array(oa.history["distance_travelled"])).max() <= 1e-5
    assert np.allclose(h["t"], np.array(oa.history["t"]))
    fr = PCs.get_history_arrays()["firingrate"]
    assert fr.shape == (steps, 100)
    assert np.abs(fr - np.array(on.history["firingrate"])).max() <= 1e-5


def test_attribute_mutation_and_post_init_writes():
    """tests/test_advanced.py:35-72 pokes Ag.pos, Ag.speed_mean and PCs.place_cell_centres[-1]
    after construction, and calls update(dt=...): all must take effect."""
    import ratinabox_b200 as rb
    np.random.seed(2)
    Env = rb.Environment(params={"aspect": 2, "scale": 1})
    Env.add_wall([[1, 0], [1, 0.35]])
    Env.add_wall([[1, 0.65], [1, 1]])
    Ag = rb.Agent(Env)
    Ag.pos = np.array([0.5, 0.5])
    Ag.speed_mean = 0.2
    PCs = rb.PlaceCells(Ag, params={"n": 20, "description": "gaussian_threshold", "widths": 0.40,
                                    "wall_geometry": "line_of_sight", "max_fr": 10, "min_fr": 0.1, "color": "C1"})
    PCs.place_cell_centres[-1] = np.array([1.1, 0.5])
    BVCs = rb.BoundaryVectorCells(Ag, params={"n": 10, "color": "C2"})
    for i in range(200):
        Ag.update(dt=50e-3)
        PCs.update()
        BVCs.update()
    assert Ag.dt == 50e-3 and abs(Ag.t - 200 * 50e-3) < 1e-9
    p = Ag.pos
    assert p.shape == (2,) and 0 < p[0] < 2 and 0 < p[1] < 1
    env = O.OracleEnvironment(scale=1, aspect=2, walls=[[[1, 0], [1, 0.35]], [[1, 0.65], [1, 1]]])
    ref = O.place_cells_get_state(env, PCs.place_cell_centres, PCs.place_cell_widths, p, O.TapeRNG(),
                                  "gaussian_threshold", "line_of_sight", 0.1, 10)[:, 0]
    assert np.abs(PCs.firingrate - ref).max() <= 1e-4          # scale 9.9 -> 1e-5 relative
    assert PCs.get_history_arrays()["firingrate"].shape == (200, 20)
    # in-place mutation of a state array that was read
    q = Ag.pos
    q[0] = 0.25
    Ag.update(dt=50e-3)
    assert abs(Ag.get_history_arrays()["pos"][-1][0] - 0.25) < 0.05
    # unknown parameters warn like the reference (utils.check_params)
    with pytest.warns(UserWarning):
        rb.PlaceCells(Ag, {"n": 4, "not_a_param": 1})


def test_get_state_all_and_errors():
    import ratinabox_b200 as rb
    from ratinabox_b200._lib import RiabError
    E, Ag = make(rb, 1)
    PCs = rb.PlaceCells(Ag, {"n": 30, "wall_geometry": "line_of_sight"})
    m = PCs.get_state(evaluate_at="all")
    assert m.shape == (30, E.flattened_discrete_coords.shape[0]) and m.dtype == np.float64
    env = O.OracleEnvironment(walls=BOX_WALLS)
    ref = O.place_cells_get_state(env, PCs.place_cell_centres, PCs.place_cell_widths, E.flattened_discrete_coords,
                                  O.TapeRNG(), "gaussian", "line_of_sight")
    assert np.abs(m - ref).max() <= 1e-5
    # empty and ragged inputs
    assert PCs.get_state(evaluate_at=None, pos=np.zeros((0, 2))).shape == (30, 0)
    assert PCs.get_state(evaluate_at=None, pos=np.array([0.4, 0.6])).shape == (30, 1)
    # one_hot (arg-min across cells, np.argmin first-index ties) incl. the fused update path
    one_hot = rb.PlaceCells(Ag, {"n": 40, "description": "one_hot", "wall_geometry": "line_of_sight"})
    oh = one_hot.get_state(evaluate_at="all")
    ref_oh = O.place_cells_get_state(env, one_hot.place_cell_centres, one_hot.place_cell_widths,
                                     E.flattened_discrete_coords, O.TapeRNG(), "one_hot", "line_of_sight")
    assert np.array_equal(oh, ref_oh)
    Ag.update(); one_hot.update()
    assert one_hot.firingrate.sum() == 1.0 and one_hot.firingrate.max() == 1.0
    # more inner walls than the line-of-sight kernels hold in registers -> refused loudly, not silently wrong
    E9 = rb.Environment()
    for k in range(9):
        E9.add_wall([[0.1 * (k + 1), 0.0], [0.1 * (k + 1), 0.3]])
    Ag9 = rb.Agent(E9, {"dt": 0.01})
    with pytest.raises(RiabError):
        rb.PlaceCells(Ag9, {"n": 8, "wall_geometry": "line_of_sight"}).get_state(evaluate_at="all")
    with pytest.raises(NotImplementedError):
        rb.Environment({"dimensionality": "1D"})
    with pytest.raises(AssertionError):          # boundary cells only possible with solid boundary conditions
        rb.BoundaryVectorCells(rb.Agent(rb.Environment({"boundary_conditions": "periodic"})), {"n": 4})


def test_mode_b_statistics_of_the_production_stream(golden):
    """SURVEY section 8(c) mode B: the Philox-driven GPU motion is compared STATISTICALLY with the reference's
    process (config 1: default box, defaults, dt = 10 ms): Rayleigh speeds with scale speed_mean, an
    Ornstein-Uhlenbeck rotational velocity with std 120 deg/s and coherence 0.08 s, the speed process's coherence
    0.7 s, uniform-ish occupancy; the live reference's own 600-step run (native_c1.npz) lies within the batch's spread."""
    import ratinabox_b200 as rb
    np.random.seed(2)
    A, steps = 2048, 1500
    E = rb.Environment()
    Ag = rb.Agent(E, {"dt": 0.01, "n_agents": A, "seed": 77})
    Ag.run(steps)
    h = Ag.get_history_arrays()
    vel, rot, pos = h["vel"][300:], h["rot_vel"][300:], h["pos"][300:]
    speed = np.linalg.norm(vel, axis=-1)
    far = (np.minimum(pos, 1 - pos).min(axis=-1) > 0.15)               # away from walls: no repulsion / bounce effects
    # Rayleigh(sigma = speed_mean = 0.08) away from the walls: mean sigma*sqrt(pi/2), second moment 2 sigma^2 (Agent.py:298-312)
    assert abs(speed[far].mean() - 0.08 * np.sqrt(np.pi / 2)) < 0.002
    assert abs(np.sqrt((speed[far] ** 2).mean() / 2) - 0.08) < 0.002
    # over the whole box the walls slow the agents (repulsion, bounces at half speed): the NumPy port of the reference
    # measures 0.0937 +- 0.003 (12 agents x 2200 steps); the batch 0.0917
    assert 0.088 < speed.mean() < 0.098
    # OU rotational velocity: std sigma = 120 deg/s, autocorrelation exp(-lag/tau), tau = 0.08 s   (Agent.py:287-296)
    r = rot[:-8][far[:-8] & far[8:]]
    r8 = rot[8:][far[:-8] & far[8:]]
    assert abs(r.std() - np.radians(120)) < 0.05 * np.radians(120)
    assert abs(np.mean(r * r8) / r.var() - np.exp(-0.08 / 0.08)) < 0.05
    # speed coherence 0.7 s: correlation of the underlying normal at lag 0.7 s is exp(-1); the Rayleigh transform
    # keeps it close to that
    s0, s1 = speed[:-70], speed[70:]
    c = np.mean((s0 - s0.mean()) * (s1 - s1.mean())) / speed.var()
    assert 0.25 < c < 0.45
    # occupancy: inside, thigmotaxis 0.5 keeps a bias to the walls but no cell of a 5 x 5 grid is empty or dominant
    assert (pos > 0).all() and (pos < 1).all()
    H, _, _ = np.histogram2d(pos[..., 0].ravel(), pos[..., 1].ravel(), bins=5, range=[[0, 1], [0, 1]])
    H = H / H.sum()
    assert H.min() > 0.02 and H.max() < 0.08
    # the live reference's own run (600 steps of ONE agent): its mean speed lies within the spread of the batch's agents
    g = golden("native_c1.npz")
    ref_speed = np.linalg.norm(g["vel"], axis=-1).mean()
    per_agent = speed[:600].mean(axis=0)
    assert per_agent.min() < ref_speed < per_agent.max()


def test_zero_copy_host_io_equals_staged_copies():
    """Page-locked host buffers: a pinned drift_velocity tensor is read by the motion kernel directly and, for batches
    above the shadow limit, the new positions are posted into the pinned buffer `Ag.pos` hands out
    (riab_step_io.pos_mirror).  Both must equal the staged-copy path bit for bit, step after step."""
    import torch
    import ratinabox_b200 as rb
    A = 5000                                      # > Agent._SHADOW_MAX: pinned read-only views
    outs = []
    for pinned in (False, True):
        np.random.seed(12)
        E = rb.Environment()
        E.add_wall([[0.5, 0.0], [0.5, 0.6]])
        Ag = rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": 4})
        PCs = rb.PlaceCells(Ag, {"n": 32})
        rs = np.random.RandomState(0)
        traj = []
        for s in range(6):
            cmd = 0.2 * rs.standard_normal((A, 2))
            d = torch.as_tensor(cmd).pin_memory() if pinned else cmd
            Ag.update(drift_velocity=d, drift_to_random_strength_ratio=2.0)
            PCs.update()
            p = Ag.pos
            assert np.array_equal(p, Ag._s["pos"].cpu().numpy())        # the mirror IS the device state
            traj.append(p.copy())
        Ag.pos = traj[0]                                                  # a user write invalidates the mirror
        assert np.array_equal(Ag.pos, traj[0])
        Ag.update(); PCs.update()
        traj.append(Ag.pos.copy())
        outs.append((np.array(traj), PCs.firingrate.copy()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])


def test_history_rate_maps_on_the_device():
    """riab_history_rate_maps: occupancy and rate maps binned from the device history rings equal
    utils.bin_data_for_histogramming (utils.py:544-589) applied to the same history on the host -- counts exactly
    (same np.histogram2d edge semantics), rate sums to float32 accuracy (test_gpu_history_maps.py bounds them by float64 sums)."""
    import ratinabox_b200 as rb
    A, steps = 300, 40
    E, Ag = make(rb, A, dt=0.05)
    PCs = rb.PlaceCells(Ag, {"n": 20, "widths": 0.3})
    GCs = rb.GridCells(Ag, {"n": 6})
    Ag.run(steps)
    hp = Ag.get_history_arrays()["pos"].reshape(-1, 2)                # (steps*A, 2), float32-rounded positions
    dx = 0.1
    heat = Ag.get_position_heatmap(dx=dx)
    ref = O.bin_data_for_histogramming(hp, list(E.extent), dx)
    assert heat.shape == ref.shape and np.array_equal(heat, ref) and heat.sum() == steps * A
    for Ns in (PCs, GCs):
        fr = Ns.get_history_arrays()["firingrate"].reshape(-1, Ns.n)
        maps, zero = Ns.get_history_rate_maps(dx=dx, return_zero_bins=True)
        assert maps.shape == (Ns.n,) + ref.shape
        for c in range(Ns.n):
            m, zb = O.bin_data_for_histogramming(hp, list(E.extent), dx, weights=fr[:, c], norm_by_bincount=True,
                                                 return_zero_bins=True)
            assert np.array_equal(zero, zb)
            assert np.abs(maps[c] - m).max() <= 1e-5 * max(1.0, np.abs(m).max())
    # the default bin width is 5 x Environment.dx like the reference's plots
    assert Ag.get_position_heatmap().shape == (20, 20)


def test_history_rate_maps_after_the_rings_wrapped():
    """The same maps after the Agent ring (30 rows) and the population rings (17 and 23 rows) all wrapped inside one
    Ag.run: the heat-map bins the Agent's last 30 rows, each rate map the last min(30, population rows) rows of both
    rings -- equal to utils.bin_data_for_histogramming of the host get_history_arrays() of those steps."""
    import ratinabox_b200 as rb
    A, pre, steps = 300, 3, 40
    E, Ag = make(rb, A, dt=0.05, history_bytes_limit=30 * A * 32)
    PCs = rb.PlaceCells(Ag, {"n": 20, "widths": 0.3, "history_bytes_limit": 17 * A * 20 * 4})
    GCs = rb.GridCells(Ag, {"n": 6, "history_bytes_limit": 23 * A * 8 * 4})
    for _ in range(pre):
        Ag.update(); PCs.update(); GCs.update()
    Ag.run(steps)
    hp = Ag.get_history_arrays()["pos"]
    assert hp.shape == (30, A, 2) and Ag.history_dropped == pre + steps - 30
    dx = 0.1
    heat = Ag.get_position_heatmap(dx=dx)
    ref = O.bin_data_for_histogramming(hp.reshape(-1, 2), list(E.extent), dx)
    assert np.array_equal(heat, ref) and heat.sum() == 30 * A
    for Ns, rows in ((PCs, 17), (GCs, 23)):
        h = Ns.get_history_arrays()
        assert h["firingrate"].shape == (rows, A, Ns.n) and Ns.history_dropped == pre + steps - rows
        pos = hp[-rows:].reshape(-1, 2)
        fr = h["firingrate"].reshape(-1, Ns.n)
        maps, zero = Ns.get_history_rate_maps(dx=dx, return_zero_bins=True)
        for c in range(Ns.n):
            m, zb = O.bin_data_for_histogramming(pos, list(E.extent), dx, weights=fr[:, c], norm_by_bincount=True,
                                                 return_zero_bins=True)
            assert np.array_equal(zero, zb)
            assert np.abs(maps[c] - m).max() <= 1e-5 * max(1.0, np.abs(m).max())


def test_step_fused_host_entry_point():
    """riab_step_fused_host (the C-ABI e2e entry: HOST drift in, fused step, HOST positions out) equals the Python
    API's own step bit for bit."""
    import ctypes as C
    import torch
    import ratinabox_b200 as rb
    from ratinabox_b200 import _lib
    lib = _lib.load()
    A = 200
    res = []
    for use_host_entry in (False, True):
        E, Ag = make(rb, A, fused_step=True)          # (the host entry wraps the FUSED step: keep update() queueing)
        PCs = rb.PlaceCells(Ag, {"n": 48})
        rs = np.random.RandomState(5)
        for s in range(3):
            cmd = 0.1 * rs.standard_normal((A, 2))
            if not use_host_entry:
                Ag.update(drift_velocity=cmd); PCs.update()
                pos = Ag.pos.copy()
            else:
                Ag.update()                                   # stages params / io exactly like a normal step
                assert Ag._take_pending()
                cells = PCs._cells()
                row, spk = PCs._row_buffers()
                out, nz = PCs._fill_out_structs(row, spk)
                drift_host = torch.as_tensor(cmd).pin_memory()
                staging = torch.empty((A, 2), dtype=torch.float64, device=Ag.device)
                pos_host = torch.empty((A, 2), dtype=torch.float64).pin_memory()
                _lib.check(lib.riab_step_fused_host(C.byref(Ag._agents_c), C.byref(Ag._env_struct()), C.byref(Ag._mp),
                                                    C.byref(Ag._io), PCs._cells_kind, C.byref(cells), C.byref(nz), C.byref(out),
                                                    drift_host.data_ptr(), staging.data_ptr(), pos_host.data_ptr(), Ag._stream()))
                torch.cuda.synchronize()
                PCs._t_hist.append(Ag.t)
                pos = pos_host.numpy().copy()
                assert np.array_equal(pos, Ag.pos)
        res.append((pos, PCs.firingrate.copy()))
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])

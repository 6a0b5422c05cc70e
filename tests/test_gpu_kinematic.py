"""HeadDirectionCells, VelocityCells and SpeedCell on the GPU (csrc/riab_kin.cuh, k_step<KinPolicy>): rates against the
float64 oracle (oracle/riab_oracle_kin.py) at the agents and away from them for every cell tile and batch size, bit
equality of the stepped API, the fused stepped API and Agent.run (the kinematic population first, behind a PlaceCells
population, under an imported trajectory; launch counts pinned), NaN positions, spikes against the Philox mirror, the
OU noise, a FeedForwardLayer fed by velocity and head direction cells, the reference's raises and prints,
get_head_direction_averaged_state against the live reference's fixture (tests/golden/kin.npz), and the staged live
reference."""
import json
import warnings

import numpy as np
import pytest

import philox_np as PX
import riab_oracle_kin as K

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                      # noqa: E402

STATE = ("pos", "velocity", "rotational_velocity", "measured_velocity", "measured_rotational_velocity",
         "head_direction", "distance_travelled", "distance_to_closest_wall")
WAYS = ("run", "run_fused", "step", "step_fused")


def _bound(N, scale=1.0):
    return 1e-5 * abs(N.max_fr - N.min_fr) * np.maximum(1.0, scale)


def _vec(Ag, name):
    return np.asarray(getattr(Ag, name), dtype=float).reshape(Ag.n_agents, 2)


def _close(got, want, bound):
    assert got.shape == want.shape, (got.shape, want.shape)
    err = np.abs(got - want)
    assert np.all(err <= bound), float(np.max(err - bound))


def _populations(A, n, seed=4):
    np.random.seed(seed)
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05, "n_agents": A, "seed": seed})
    H = rb.HeadDirectionCells(Ag, {"n": n, "angular_spread_degrees": 30, "min_fr": 0.2, "max_fr": 1.5})
    V = rb.VelocityCells(Ag, {"n": n, "min_fr": 0.5, "max_fr": 0.1})
    S = rb.SpeedCell(Ag, {"min_fr": 0.1, "max_fr": 2.0})
    H.preferred_angles = np.random.RandomState(n).uniform(0, 2 * np.pi, n)            # editable: re-packed
    H.angular_tunings = np.random.RandomState(n + 1).uniform(0.05, 1.2, n)
    return Ag, H, V, S


@pytest.mark.parametrize("A", [1, 33, 4099])
@pytest.mark.parametrize("n", [1, 4, 10, 63, 64, 300])
def test_rates_match_the_oracle(n, A):
    Ag, H, V, S = _populations(A, n)
    for _ in range(3):
        Ag.update()
        for N in (H, V, S):
            N.update()
    hd, vel, mv = _vec(Ag, "head_direction"), _vec(Ag, "velocity"), _vec(Ag, "measured_velocity")
    pa, tu, oss = H.preferred_angles, H.angular_tunings, V.one_sigma_speed
    # at the agents: the rows of update() and get_state()
    want_h = K.head_direction_rows(hd, pa, tu, H.min_fr, H.max_fr)
    _close(H.get_state(), want_h, _bound(H))
    _close(H.get_history_arrays()["firingrate"][-1].reshape(A, n).T, want_h, _bound(H))
    _close(H.get_state(use_velocity=True), K.head_direction_rows(vel, pa, tu, H.min_fr, H.max_fr, use_velocity=True), _bound(H))
    vp, vt = V.preferred_angles, V.angular_tunings
    scale = np.linalg.norm(vel, axis=1) / oss
    want_v = K.velocity_rows(vel, oss, vp, vt, V.min_fr, V.max_fr)
    _close(V.get_state(), want_v, _bound(V, scale))
    _close(V.get_history_arrays()["firingrate"][-1].reshape(A, n).T, want_v, _bound(V, scale))
    want_s = K.speed_rows(mv, oss, S.min_fr, S.max_fr)
    _close(S.get_state(), want_s, _bound(S, np.linalg.norm(mv, axis=1) / oss))
    _close(S.get_history_arrays()["firingrate"][-1].reshape(A, 1).T, want_s, _bound(S, np.linalg.norm(mv, axis=1) / oss))
    # away from the agents: one vector for every position, and one per position
    rs = np.random.RandomState(A)
    P = rs.uniform(0.05, 0.95, (257, 2))
    D = rs.normal(size=(257, 2))
    d0 = np.array([-0.4, 0.25])
    _close(H.get_state(evaluate_at=None, pos=P, head_direction=d0), K.head_direction_rates(d0, pa, tu, H.min_fr, H.max_fr, 257),
           _bound(H))
    _close(H.get_state(evaluate_at=None, pos=P, head_direction=D), K.head_direction_rows(D, pa, tu, H.min_fr, H.max_fr), _bound(H))
    _close(H.get_state(evaluate_at=None, use_velocity=True, velocity=D),
           K.head_direction_rows(D, pa, tu, H.min_fr, H.max_fr, use_velocity=True), _bound(H))
    _close(S.get_state(evaluate_at="all", vel=d0),
           np.tile(K.speed_rate(d0, oss, S.min_fr, S.max_fr), (1, Ag.Environment.flattened_discrete_coords.shape[0])),
           _bound(S, np.linalg.norm(d0) / oss))
    _close(S.get_state(evaluate_at=None, vel=D), K.speed_rows(D, oss, S.min_fr, S.max_fr), _bound(S, np.linalg.norm(D, axis=1) / oss))
    if A == 1:
        av = vel[0]
        sc = np.linalg.norm(av) / oss
        _close(V.get_state(evaluate_at=None, pos=P, velocity=d0),
               K.velocity_rates(d0, av, oss, vp, vt, V.min_fr, V.max_fr, 257), _bound(V, sc))
        _close(V.get_state(evaluate_at=None, velocity=D), K.velocity_rows(D, oss, vp, vt, V.min_fr, V.max_fr, scale_by=av),
               _bound(V, sc))
    else:
        with pytest.raises(ValueError, match="n_agents"):
            V.get_state(evaluate_at="all", velocity=d0)
    t = H.get_state(evaluate_at=None, head_direction=torch.as_tensor(D, device="cuda"), return_tensor=True)
    assert t.shape == (257, n) and t.dtype == torch.float32


def test_the_reference_fixture(golden):
    """The fixture's cases through the device: the native run's states, the kwargs, the rate ranges, kappa = 700 and the
    zero velocity's NaN."""
    g = golden("kin.npz")
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05})
    H = rb.HeadDirectionCells(Ag)
    V = rb.VelocityCells(Ag)
    assert np.array_equal(H.preferred_angles, g["hdc_preferred_angles"]) and np.array_equal(H.angular_tunings, g["hdc_angular_tunings"])
    assert V.one_sigma_speed == float(g["vel_one_sigma_speed"])
    for t in range(0, g["run_hd"].shape[0], 7):
        Ag.head_direction, Ag.velocity = g["run_hd"][t], g["run_vel"][t]
        sc = np.linalg.norm(g["run_vel"][t]) / V.one_sigma_speed
        _close(H.get_state(), g["run_hdc"][t], _bound(H))
        _close(H.get_state(use_velocity=True), g["run_hdc_usevel"][t], _bound(H))
        _close(V.get_state(), g["run_velc"][t], _bound(V, sc))
    hd, P = g["kw_hd"], g["kw_P"]
    _close(H.get_state(evaluate_at=None, head_direction=hd), g["kw_head_direction"], _bound(H))
    _close(H.get_state(evaluate_at="all", head_direction=hd), g["kw_head_direction_all"], _bound(H))
    _close(H.get_state(evaluate_at=None, pos=P, head_direction=hd), g["kw_head_direction_pos"], _bound(H))
    _close(H.get_state(evaluate_at=None, use_velocity=True, velocity=hd), g["kw_velocity_usevel"], _bound(H))
    Ag.velocity = g["kw_agent_velocity"]
    sc = np.linalg.norm(g["kw_agent_velocity"]) / V.one_sigma_speed
    _close(V.get_state(evaluate_at=None, velocity=hd), g["kw_velc_velocity"], _bound(V, sc))
    _close(V.get_state(evaluate_at=None, pos=P, velocity=hd), g["kw_velc_velocity_pos"], _bound(V, sc))
    for case in ("lo", "inv"):
        prm = json.loads(str(g[f"fr_{case}_params"]))
        Ag.head_direction, Ag.velocity, Ag.measured_velocity = g["fr_agent_hd"], g["fr_agent_vel"], g["fr_agent_mvel"]
        Vc = rb.VelocityCells(Ag, dict(prm, n=13, angular_spread_degrees=30))
        Hc = rb.HeadDirectionCells(Ag, dict(prm, n=13, angular_spread_degrees=30))
        Sc = rb.SpeedCell(Ag, dict(prm))
        sc = np.linalg.norm(g["fr_agent_vel"]) / 0.16
        _close(Vc.get_state(), g[f"fr_{case}_velc"], _bound(Vc, sc))
        _close(Vc.get_state(evaluate_at=None, velocity=g["fr_vel"]), g[f"fr_{case}_velc_kw"], _bound(Vc, sc))
        _close(Hc.get_state(), g[f"fr_{case}_hdc"], _bound(Hc))
        _close(Sc.get_state()[:, 0], g[f"fr_{case}_speed_agent"], _bound(Sc, np.linalg.norm(g["fr_agent_mvel"]) / 0.16))
        _close(Sc.get_state(evaluate_at=None, vel=g["fr_vel"])[:, 0], g[f"fr_{case}_speed_kw"], _bound(Sc, 1.0))
    Hn = rb.HeadDirectionCells(Ag, {"n": 36, "angular_spread_degrees": float(g["narrow_deg"])})
    th = g["narrow_theta"]
    _close(Hn.get_state(evaluate_at=None, head_direction=np.stack((np.cos(th), np.sin(th)), axis=1)), g["narrow"], _bound(Hn))
    Ag.velocity = np.array([0.0, 0.0])
    assert np.all(np.isnan(V.get_state())) and np.all(np.isnan(H.get_state(use_velocity=True)))
    assert np.all(np.isnan(g["zero_velc"]))


def test_raises_warns_and_prints(capsys):
    with pytest.raises(NotImplementedError):
        rb.Environment({"dimensionality": "1D"})
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05, "n_agents": 3})
    H = rb.HeadDirectionCells(Ag, {"n": 6})
    V = rb.VelocityCells(Ag, {"n": 6})
    with pytest.raises(ValueError, match="n_agents"):
        V.get_state(evaluate_at="all")
    assert V.get_state().shape == (6, 3)
    capsys.readouterr()
    r = H.get_state(evaluate_at=None)
    assert capsys.readouterr().out == ("HeadDirection cells need a head direction but you didn't pass one. Taking [1,0] as "
                                       "defaultRecommended to pass one in the 'head_direction' argument of get_state()\n")
    _close(r, K.head_direction_rates([1, 0], H.preferred_angles, H.angular_tunings), _bound(H))
    H.get_state(evaluate_at=None, use_velocity=True)
    assert "need a velocity" in capsys.readouterr().out
    with pytest.warns(UserWarning, match="'vel' kwarg deprecated"):
        r2 = H.get_state(evaluate_at=None, vel=[0.0, 1.0])
    _close(r2, K.head_direction_rates([0.0, 1.0], H.preferred_angles, H.angular_tunings), _bound(H))
    with pytest.warns(UserWarning, match=r"Ignoring 'n' parameter value \(4\) that was passed for SpeedCell"):
        S = rb.SpeedCell(Ag, {"n": 4})
    assert S.n == 1 and S.get_state().shape == (1, 3)
    with pytest.raises(ValueError, match="vectors for 5 positions"):
        H.get_state(evaluate_at=None, pos=np.zeros((5, 2)), head_direction=np.ones((4, 2)))


def test_nan_positions_give_zero_rates():
    A = 40
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05, "n_agents": A, "seed": 2})
    pops = (rb.HeadDirectionCells(Ag, {"n": 10}), rb.VelocityCells(Ag, {"n": 10}), rb.SpeedCell(Ag))
    Ag.update()
    pos = _vec(Ag, "pos")
    pos[[3, 17, 39]] = np.nan
    Ag.pos = pos
    for N in pops:
        N.update()
        fr = N.firingrate
        assert np.all(fr[[3, 17, 39]] == 0) and np.all(np.isfinite(fr)) and np.all(fr[0] != 0)


# ---- stepped / fused / run
def _agent(fused, A=257):
    np.random.seed(9)
    E = rb.Environment()
    E.add_wall([[0.3, 0.0], [0.3, 0.5]])
    return rb.Agent(E, {"dt": 0.02, "n_agents": A, "seed": 5, "fused_step": fused})


def kin_first(fused):
    Ag = _agent(fused)
    rb.HeadDirectionCells(Ag, {"n": 10})
    rb.VelocityCells(Ag, {"n": 12, "max_fr": 2.0})
    rb.SpeedCell(Ag, {"max_fr": 3.0})
    return Ag


def behind_place(fused):
    Ag = _agent(fused)
    rb.PlaceCells(Ag, {"n": 64, "wall_geometry": "line_of_sight"})
    rb.HeadDirectionCells(Ag, {"n": 70, "noise_std": 0.05})
    return Ag


def imported(fused):
    Ag = _agent(fused)
    rng = np.random.default_rng(8)
    Ag.import_trajectory(times=np.cumsum(rng.uniform(0.05, 0.2, 20)), positions=rng.uniform(0.05, 0.95, (20, 2)))
    rb.HeadDirectionCells(Ag, {"n": 10})
    rb.VelocityCells(Ag, {"n": 10})
    return Ag


SETUPS = {
    # skewed: motion(0), then per step populations 1.. and the skewed launch of population 0
    "kin_first": (kin_first, lambda n: {"run": 1 + 3 * n, "run_fused": 1 + 3 * n, "step": 4 * n, "step_fused": 3 * n}),
    "behind_place": (behind_place, lambda n: {"run": 1 + 2 * n, "run_fused": 1 + 2 * n, "step": 3 * n, "step_fused": 2 * n}),
    # a motion source: the motion kernel, then every population
    "imported": (imported, lambda n: dict.fromkeys(WAYS, 3 * n)),
}


def _collect(Ag):
    out = {k: np.asarray(getattr(Ag, k)).copy() for k in STATE}
    for k, v in Ag.get_history_arrays().items():
        out["agent." + k] = np.asarray(v)
    for i, N in enumerate(Ag.Neurons):
        for k, v in N.get_history_arrays().items():
            out[f"{i}.{k}"] = np.asarray(v)
    return out


@pytest.mark.parametrize("name", list(SETUPS))
def test_run_fused_and_stepped_are_bit_identical(name):
    from ratinabox_b200 import _lib
    lib = _lib.load()
    build, launches = SETUPS[name]
    n = 5
    res, counts = {}, {}
    for way in WAYS:
        Ag = build(way.endswith("fused"))
        Ag.update()
        for N in Ag.Neurons:
            N.update()
        c0 = lib.riab_launch_count()
        if way.startswith("run"):
            Ag.run(n)
        else:
            for _ in range(n):
                Ag.update()
                for N in Ag.Neurons:
                    N.update()
        res[way] = _collect(Ag)
        counts[way] = lib.riab_launch_count() - c0
        if way == "step":
            # the last step's rows against the oracle and the Philox mirror of the dense spike stream
            hd, vel, mv = _vec(Ag, "head_direction"), _vec(Ag, "velocity"), _vec(Ag, "measured_velocity")
            for N in Ag.Neurons:
                h = N.get_history_arrays()
                fr = h["firingrate"][-1].reshape(Ag.n_agents, N.n)
                if N.noise_std == 0:
                    want = N.get_state().T
                    assert np.array_equal(fr, want.astype(np.float32).astype(np.float64)), type(N).__name__
                    sp = PX.expected_spikes(5, N._upd - 1, np.arange(Ag.n_agents), fr.astype(np.float32), 0.02,
                                            pop=N._population_id)
                    assert np.array_equal(h["spikes"][-1].reshape(Ag.n_agents, N.n), sp), type(N).__name__
                if isinstance(N, rb.VelocityCells):
                    w = K.velocity_rows(vel, N.one_sigma_speed, N.preferred_angles, N.angular_tunings, N.min_fr, N.max_fr).T
                    _close(fr, w, _bound(N, np.linalg.norm(vel, axis=1)[:, None] / N.one_sigma_speed))
                elif isinstance(N, rb.HeadDirectionCells) and N.noise_std == 0:
                    _close(fr, K.head_direction_rows(hd, N.preferred_angles, N.angular_tunings, N.min_fr, N.max_fr).T, _bound(N))
                elif isinstance(N, rb.SpeedCell):
                    _close(fr, K.speed_rows(mv, N.one_sigma_speed, N.min_fr, N.max_fr).T,
                           _bound(N, np.linalg.norm(mv, axis=1)[:, None] / N.one_sigma_speed))
    assert counts == launches(n), counts
    ref = res["step"]
    for way in WAYS:
        for k in ref:
            x, y = np.asarray(res[way][k]), np.asarray(ref[k])
            assert x.shape == y.shape and np.array_equal(x, y), f"{name}: {way} vs step: {k}"
    assert any(np.asarray(v).any() for k, v in ref.items() if k.endswith(".spikes"))


def test_ou_noise_is_an_ornstein_uhlenbeck_process():
    """noise_std 0.1, coherence time 0.5 s, dt 0.02 s: after 300 steps (12 coherence times) the noise across 4099 x 16
    cells has mean 0 and std 0.1, and the rows are the clean rates plus the noise state."""
    A, n = 4099, 16
    Ag = rb.Agent(rb.Environment(), {"dt": 0.02, "n_agents": A, "seed": 3})
    H = rb.HeadDirectionCells(Ag, {"n": n, "noise_std": 0.1, "noise_coherence_time": 0.5, "save_history": False})
    Ag.run(299)
    prev = H._noise[:, :n].double().cpu().numpy().copy()
    Ag.run(1)
    noise = H._noise[:, :n].double().cpu().numpy()
    fr = H.firingrate
    _close(fr - H.get_state().T, noise, 1e-5 + 1e-6 * np.abs(noise))
    assert abs(noise.mean()) < 0.004 and abs(noise.std() - 0.1) < 0.004, (noise.mean(), noise.std())
    rho = np.corrcoef(prev.ravel(), noise.ravel())[0, 1]               # exp(-dt/tau) = 0.961
    assert abs(rho - np.exp(-0.02 / 0.5)) < 0.01, rho


def test_path_integration_feedforward():
    """VelocityCells + HeadDirectionCells -> FeedForwardLayer (the reference's path-integration input layer): run and the
    stepped loop give the same rows, and the layer's rows are W . I + b of its inputs' rows."""
    A = 300
    res = []
    for way in ("run", "step"):
        np.random.seed(2)
        Ag = rb.Agent(rb.Environment(), {"dt": 0.05, "n_agents": A, "seed": 1})
        V = rb.VelocityCells(Ag, {"n": 16})
        H = rb.HeadDirectionCells(Ag, {"n": 12})
        F = rb.FeedForwardLayer(Ag, {"n": 20, "input_layers": [V, H], "name": "PI"})
        if way == "run":
            Ag.run(6)
        else:
            for _ in range(6):
                Ag.update()
                for N in Ag.Neurons:
                    N.update()
        res.append([N.get_history_arrays()["firingrate"] for N in (V, H, F)])
        v, h, f = (N.get_history_arrays()["firingrate"][-1].reshape(A, N.n) for N in (V, H, F))
        want = v @ F.inputs[V.name]["w"].T + h @ F.inputs[H.name]["w"].T + F.biases
        scale = np.abs(v) @ np.abs(F.inputs[V.name]["w"]).T + np.abs(h) @ np.abs(F.inputs[H.name]["w"]).T
        assert np.all(np.abs(f - want) <= 1e-5 * scale.max()), float(np.abs(f - want).max())
    for a, b in zip(*res):
        assert np.array_equal(a, b)


def test_head_direction_averaged_state(golden):
    g = golden("kin.npz")
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05})
    H = rb.HeadDirectionCells(Ag, {"n": 8, "angular_spread_degrees": 30, "min_fr": 0.1, "max_fr": 1.7})
    _close(H.get_head_direction_averaged_state(evaluate_at="all"), g["avg_hdc_all"], _bound(H))
    _close(H.get_head_direction_averaged_state(evaluate_at="all", angular_resolution_degrees=30), g["avg_hdc_all_res30"], _bound(H))
    Ag.head_direction = g["avg_agent_hd"]
    _close(H.get_head_direction_averaged_state(), g["avg_hdc_agent"], _bound(H))
    E = rb.Environment()
    E.add_wall([[0.3, 0.0], [0.3, 0.5]])
    F = rb.FieldOfViewBVCs(rb.Agent(E, {"dt": 0.05}), {"min_fr": 0.0, "max_fr": 2.0})
    got = F.get_head_direction_averaged_state(evaluate_at=None, pos=g["avg_fov_P"], angular_resolution_degrees=30)
    _close(got, g["avg_fov"], 2e-5)


def test_matches_the_staged_live_reference():
    import ref_shim
    if ref_shim.import_reference() is None:
        pytest.skip("the reference is not staged under oracle/_ref")
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import HeadDirectionCells, VelocityCells, SpeedCell
    np.random.seed(21)
    RA = Agent(Environment(), {"dt": 0.05})
    RH = HeadDirectionCells(RA, {"n": 17, "angular_spread_degrees": 20, "min_fr": 0.3, "max_fr": 1.1})
    RV = VelocityCells(RA, {"n": 9})
    RS = SpeedCell(RA, {"n": 1})
    Ag = rb.Agent(rb.Environment(), {"dt": 0.05})
    H = rb.HeadDirectionCells(Ag, {"n": 17, "angular_spread_degrees": 20, "min_fr": 0.3, "max_fr": 1.1})
    V = rb.VelocityCells(Ag, {"n": 9})
    S = rb.SpeedCell(Ag)
    for _ in range(25):
        RA.update()
        for N in (RH, RV, RS):
            N.update()
        Ag.head_direction, Ag.velocity = RA.head_direction, RA.velocity
        Ag.measured_velocity = RA.history["vel"][-1]
        sc = np.linalg.norm(RA.velocity) / RV.one_sigma_speed
        _close(H.get_state(), RH.get_state(), _bound(H))
        _close(V.get_state(), RV.get_state(), _bound(V, sc))
        _close(S.get_state()[:, 0], RS.get_state(), _bound(S, sc + 1))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            hd = np.random.RandomState(1).normal(size=2)
            _close(H.get_state(evaluate_at="all", head_direction=hd), RH.get_state(evaluate_at="all", head_direction=hd), _bound(H))

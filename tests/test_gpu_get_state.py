"""get_state's evaluation points for every population class: at the agents it equals, bit for bit, the evaluation at
their positions passed as ``pos`` (NumPy, a CUDA tensor or a CPU tensor) with the agents' head directions, partner
positions or kinematic vectors passed as kwargs; ``return_tensor=True`` is the NumPy result transposed; no positions give
(n, 0).  Egocentric vector cells at the agents read in-place edits of ``Ag.pos`` / ``Ag.head_direction``, and take
``pos`` and ``head_direction`` as CUDA tensors."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                      # noqa: E402

WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
OBJECTS = [([0.2, 0.8], 0), ([0.5, 0.9], 0), ([0.8, 0.2], 1)]


def _env():
    E = rb.Environment()
    for w in WALLS:
        E.add_wall(w)
    for xy, t in OBJECTS:
        E.add_object(xy, type=t)
    return E


def _hd(Ag, Ag2, Ag3):
    return {"head_direction": Ag.head_direction}


# name: (build(Ag, Ag2, Ag3), the kwargs that restate the agents' own inputs, position-based)
POPULATIONS = {
    "place": (lambda Ag, Ag2, Ag3: rb.PlaceCells(Ag, {"n": 20, "wall_geometry": "line_of_sight"}), None, True),
    "grid": (lambda Ag, Ag2, Ag3: rb.GridCells(Ag, {"n": 12}), None, True),
    "bvc": (lambda Ag, Ag2, Ag3: rb.BoundaryVectorCells(Ag, {"n": 16}), None, True),
    "bvc_ego": (lambda Ag, Ag2, Ag3: rb.BoundaryVectorCells(Ag, {"n": 16, "reference_frame": "egocentric"}), _hd, True),
    "fov_bvc": (lambda Ag, Ag2, Ag3: rb.FieldOfViewBVCs(Ag), _hd, True),
    "ovc": (lambda Ag, Ag2, Ag3: rb.ObjectVectorCells(Ag, {"n": 10}), None, True),
    "fov_ovc": (lambda Ag, Ag2, Ag3: rb.FieldOfViewOVCs(Ag, {"object_tuning_type": 0}), _hd, True),
    "avc_batched": (lambda Ag, Ag2, Ag3: rb.AgentVectorCells(Ag, Ag2, {"n": 9}),
                    lambda Ag, Ag2, Ag3: {"other_pos": Ag2.pos}, True),
    "avc_one": (lambda Ag, Ag2, Ag3: rb.AgentVectorCells(Ag, Ag3, {"n": 9, "reference_frame": "egocentric"}), _hd, True),
    "fov_avc": (lambda Ag, Ag2, Ag3: rb.FieldOfViewAVCs(Ag, Ag2),
                lambda Ag, Ag2, Ag3: {"other_pos": Ag2.pos, "head_direction": Ag.head_direction}, True),
    "rsn": (lambda Ag, Ag2, Ag3: rb.RandomSpatialNeurons(Ag, {"n": 8, "wall_geometry": "line_of_sight"}), None, True),
    "hdc": (lambda Ag, Ag2, Ag3: rb.HeadDirectionCells(Ag, {"n": 10}), _hd, False),
    "speed": (lambda Ag, Ag2, Ag3: rb.SpeedCell(Ag), lambda Ag, Ag2, Ag3: {"vel": Ag.measured_velocity}, False),
    "ffl": (lambda Ag, Ag2, Ag3: rb.FeedForwardLayer(Ag, {"n": 7, "input_layers": [rb.PlaceCells(Ag, {"n": 20})]}),
            None, False),
}


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("name", list(POPULATIONS))
def test_at_the_agents_equals_the_explicit_positions(name):
    build, restate, position_based = POPULATIONS[name]
    np.random.seed(7)
    E = _env()
    Ag = rb.Agent(E, {"dt": 0.02, "n_agents": 33, "seed": 3})
    Ag2 = rb.Agent(E, {"dt": 0.02, "n_agents": 33, "seed": 4})
    Ag3 = rb.Agent(E, {"dt": 0.02, "seed": 5})
    N = build(Ag, Ag2, Ag3)
    for _ in range(3):
        Ag.update()
        Ag2.update()
        Ag3.update()
        N.update()
    at_agents = N.get_state("agent")
    assert at_agents.shape == (N.n, 33) and at_agents.dtype == np.float64
    assert np.any(at_agents != 0), name
    kw = {} if restate is None else restate(Ag, Ag2, Ag3)
    P = Ag.pos
    for form in (np.asarray, lambda x: torch.as_tensor(x, device="cuda"), torch.as_tensor):
        got = N.get_state(None, pos=form(P), **{k: form(v) for k, v in kw.items()})
        assert _same_bits(got, at_agents), (name, form)
    t = N.get_state("agent", return_tensor=True)
    assert t.dtype == torch.float32 and t.shape == (33, N.n)
    assert _same_bits(t.cpu().numpy().T, at_agents)
    if position_based:
        none = {k: np.zeros((0, 2)) for k in kw}
        assert N.get_state(None, pos=np.zeros((0, 2)), **none).shape == (N.n, 0)


@pytest.mark.parametrize("cls", [rb.FieldOfViewBVCs, rb.FieldOfViewOVCs])
def test_egocentric_cells_read_in_place_edits_of_the_agent(cls):
    np.random.seed(1)
    Ag = rb.Agent(_env(), {"dt": 0.02, "seed": 2})
    N = cls(Ag, {"object_tuning_type": 0} if cls is rb.FieldOfViewOVCs else {})
    for _ in range(3):
        Ag.update()
        N.update()
    before = N.get_state()
    hd = Ag.head_direction
    hd[:] = [0.0, 1.0]
    pos = Ag.pos
    pos[:] = [0.5, 0.75]                       # a wall 0.25 ahead, an object 0.15 ahead
    after = N.get_state()
    assert _same_bits(after, N.get_state(evaluate_at=None, pos=[0.5, 0.75], head_direction=[0.0, 1.0]))
    assert not np.array_equal(after, before)
    assert np.array_equal(Ag.pos, [0.5, 0.75]) and np.array_equal(Ag.head_direction, [0.0, 1.0])


@pytest.mark.parametrize("name", ["bvc_ego", "fov_bvc", "fov_ovc", "avc_one"])
def test_egocentric_cells_take_cuda_tensors(name):
    np.random.seed(11)
    E = _env()
    Ag = rb.Agent(E, {"dt": 0.02, "n_agents": 4, "seed": 3})
    N = POPULATIONS[name][0](Ag, None, rb.Agent(E, {"dt": 0.02, "seed": 5}))
    X = np.random.uniform(0.05, 0.95, (40, 2))
    H = np.random.normal(size=(40, 2))
    for hd in (H, H[3]):                       # one direction per position, or one for all
        want = N.get_state(evaluate_at=None, pos=X, head_direction=hd)
        got = N.get_state(evaluate_at=None, pos=torch.as_tensor(X, device="cuda"),
                          head_direction=torch.as_tensor(hd, device="cuda"))
        assert _same_bits(got, want), name

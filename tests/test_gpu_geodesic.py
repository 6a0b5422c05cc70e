"""Geodesic PlaceCells (the default wall_geometry with exactly one added wall) on the device, at what the at-scale,
launch-path and fuzz suites do not reach: the float64 reference fixture of every description, which wall ends count as
inside the box, agents on the wall's line and at its ends, and walls with no end inside the box, where the reference's
np.amin over an empty list of detours raises (Environment.py:769-773).  GPU only."""
import os

import numpy as np
import pytest

import riab_oracle as O
import riab_oracle_pppc as PP

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                                  # noqa: E402
from ratinabox_b200 import _lib                               # noqa: E402
from ratinabox_b200.contribs import PhasePrecessingPlaceCells as PPPC   # noqa: E402

TOL = 1e-5
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "geodesic.npz")
DESCS = ("gaussian", "gaussian_threshold", "diff_of_gaussians", "top_hat", "one_hot")


def _setup(wall, aspect=1.0):
    E = rb.Environment({"aspect": aspect})
    E.add_wall(wall)
    return E, O.OracleEnvironment(aspect=aspect, walls=[wall]), rb.Agent(E, {"n_agents": 1})


def _check(got, want, lo, hi, desc, what):
    if desc in ("top_hat", "one_hot"):
        bad = got != want
        assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} classifications differ"
        return
    span = abs(hi - lo)
    err = np.abs(got - want)
    assert err.max() <= TOL * span, f"{what}: max |err| {err.max():.3e}"
    if desc == "gaussian":
        big = np.abs(want - lo) > 1e-3 * span
        rel = (err[big] / np.abs(want[big])).max()
        assert rel <= TOL, f"{what}: max relative err {rel:.3e}"


# ------------------------------------------------------------------------------------------- the reference's fixture
def test_device_against_the_reference_fixture():
    """Every description and wall case of tests/golden/geodesic.npz (oracle/gen_geodesic_golden.py)."""
    g = np.load(GOLDEN)
    for case in [str(c) for c in g["cases"]]:
        wall, aspect = g[f"{case}_wall"], float(g[f"{case}_aspect"])
        E, env, Ag = _setup(wall.tolist(), aspect)
        P, centres = g[f"{case}_pos"], g[f"{case}_centres"]
        lo, hi, w = float(g["min_fr"]), float(g["max_fr"]), float(g["width"])
        for desc in DESCS:
            N = rb.PlaceCells(Ag, {"place_cell_centres": centres, "widths": w, "description": desc, "min_fr": lo,
                                   "max_fr": hi})
            assert N._cells().ep_valid == int(g[f"{case}_ep_valid"]), case
            _check(N.get_state(evaluate_at=None, pos=P), g[f"{case}_{desc}"], lo, hi, desc, f"{case} {desc}")
            Ag.Neurons.remove(N)


# ------------------------------------------------------------------------------------------------- end validity
@pytest.mark.parametrize("y0,valid", [(0.0, 2), (1e-12, 3), (-1e-12, 2)])
def test_wall_end_validity(y0, valid):
    """An end exactly on the boundary (or outside it) is not a detour corner; 1e-12 inside it is -- the strict compares of
    Environment.check_if_position_is_in_environment.  With the bottom end valid, pairs under the wall's far end take the
    shorter detour around the bottom."""
    wall = [[0.5, y0], [0.5, 0.6]]
    E, env, Ag = _setup(wall)
    rs = np.random.RandomState(3)
    centres = np.concatenate([np.stack([rs.uniform(0.3, 0.49, 30), rs.uniform(0.0, 0.2, 30)], 1),
                              rs.uniform(0.05, 0.95, (20, 2))])
    P = np.concatenate([np.stack([rs.uniform(0.51, 0.7, 300), rs.uniform(0.0, 0.2, 300)], 1), rs.uniform(0, 1, (300, 2))])
    for desc in ("gaussian", "top_hat"):
        N = rb.PlaceCells(Ag, {"place_cell_centres": centres, "widths": 0.2, "description": desc})
        assert N._cells().ep_valid == valid
        want = O.place_cells_get_state(env, centres, N.place_cell_widths, P, O.TapeRNG(), desc, "geodesic",
                                       scalar_width=0.2)
        _check(N.get_state(evaluate_at=None, pos=P), want, 0.0, 1.0, desc, f"y0 {y0} {desc}")
        Ag.Neurons.remove(N)


# -------------------------------------------------------------------------------------------- line-of-sight band
def test_agents_on_the_wall_line_and_at_its_ends():
    """Agents within 1e-9 of the wall's line, on its ends and 1e-9 around them: the float32 crossing test is unsure
    there and the float64 test decides which pairs take the detour."""
    wall = [[0.5, 0.2], [0.5, 0.8]]
    E, env, Ag = _setup(wall)
    rs = np.random.RandomState(5)
    ys = rs.uniform(0.05, 0.95, 40)
    P = [np.stack([0.5 + d + 0 * ys, ys], 1) for d in (-1e-9, -1e-10, 0.0, 1e-10, 1e-9)]
    for e in ([0.5, 0.2], [0.5, 0.8]):
        for dx in (-1e-9, 0.0, 1e-9):
            for dy in (-1e-9, 0.0, 1e-9):
                P.append(np.array([[e[0] + dx, e[1] + dy]]))
    P = np.concatenate(P)
    centres = np.concatenate([rs.uniform(0.05, 0.95, (40, 2)), [[0.4, 0.5], [0.6, 0.5], [0.5 - 1e-9, 0.5]]])
    for desc in ("gaussian", "top_hat", "one_hot"):
        N = rb.PlaceCells(Ag, {"place_cell_centres": centres, "widths": 0.3, "description": desc})
        want = O.place_cells_get_state(env, centres, N.place_cell_widths, P, O.TapeRNG(), desc, "geodesic",
                                       scalar_width=0.3)
        _check(N.get_state(evaluate_at=None, pos=P), want, 0.0, 1.0, desc, desc)
        Ag.Neurons.remove(N)
    blocked = O.distances_accounting_for_environment(env, centres, P, "line_of_sight", O.TapeRNG()) == 1000
    assert blocked.any() and not blocked.all()


# ------------------------------------------------------------------------------------------ walls with no end inside
NO_END_INSIDE = {"boundary_to_boundary": [[0.5, 0.0], [0.5, 1.0]], "crossing": [[-0.2, 0.4], [1.2, 0.6]]}


def test_default_place_cells_in_a_one_wall_box_are_geodesic():
    E, env, Ag = _setup([[0.5, 0.2], [0.5, 0.8]])
    N = rb.PlaceCells(Ag)
    assert N.wall_geometry == "geodesic" and N._effective_geometry() == "geodesic"


@pytest.mark.parametrize("name", list(NO_END_INSIDE))
def test_wall_with_no_end_inside_raises(name):
    """The reference raises ValueError at PlaceCells.get_state (the constructor succeeds), at
    PhasePrecessingPlaceCells.update and in the RandomSpatialNeurons constructor; so do the oracle and the device path,
    before anything is launched."""
    wall = NO_END_INSIDE[name]
    E, env, Ag = _setup(wall)
    lib = _lib.load()
    rs = np.random.RandomState(1)
    centres, P = rs.uniform(0, 1, (12, 2)), rs.uniform(0, 1, (30, 2))
    with pytest.raises(ValueError):
        O.place_cells_get_state(env, centres, np.full(12, 0.2), P, O.TapeRNG(), "gaussian", "geodesic")
    N = rb.PlaceCells(Ag, {"place_cell_centres": centres})
    assert N.wall_geometry == "geodesic"
    c0 = lib.riab_launch_count()
    with pytest.raises(ValueError):
        N.get_state(evaluate_at=None, pos=P)
    with pytest.raises(ValueError):
        N.update()
    with pytest.raises(ValueError):
        Ag.run(3)
    assert lib.riab_launch_count() == c0
    Ag.Neurons.remove(N)
    M = PPPC(Ag, {"place_cell_centres": centres})
    with pytest.raises(ValueError):
        PP.get_state_rows(env, Ag.pos, Ag.velocity, Ag.t, centres, M.place_cell_widths, O.TapeRNG(), M.description,
                          "geodesic", 0.0, 1.0, M.theta_freq, M.sigma, M.precess_fraction)
    c0 = lib.riab_launch_count()
    with pytest.raises(ValueError):
        M.update()
    assert lib.riab_launch_count() == c0
    Ag.Neurons.remove(M)
    with pytest.raises(ValueError):
        rb.RandomSpatialNeurons(Ag, {"n": 4, "lengthscale": 0.1})

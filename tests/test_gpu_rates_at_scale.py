"""Rate kernels away from the unit box, against the float64 oracles (oracle/riab_oracle*.py).

Every rate kernel works in float32 on coordinates taken relative to the box centre, so its error grows with the box size
over the tuning width (L / w) and over the grid period (L / lambda), and host-set bands tuned at scale 1 may be too
narrow further out.  Here the kernels run at scales 0.25 .. 10, with narrow and wide tunings, in polygons a kilometre
from the origin, and on the decision edges of the classifiers (top_hat, one_hot, line of sight, goal radius):

* every profile: max |err| <= 1e-5 (max_fr - min_fr);
* Gaussian profiles: also |err| / |rate| <= 1e-5 where |rate| > 1e-3 (max_fr - min_fr);
* top_hat / one_hot / goal classifications and line-of-sight decisions: identical to the oracle's.

The oracles' float64 arithmetic does not depend on the scale; they are pinned to the reference at scale 1 elsewhere."""
import numpy as np
import pytest

import riab_oracle as O
import riab_oracle_avc as V
import riab_oracle_pppc as PP
import riab_oracle_rsn as R

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                                  # noqa: E402
from ratinabox_b200.contribs import PhasePrecessingPlaceCells as PPPC   # noqa: E402
from ratinabox_b200.contribs import SpatialGoalEnvironment   # noqa: E402

TOL = 1e-5
C2 = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]   # two walls of the unit box, scaled with the box below
GEO = [[[0.5, 0.2], [0.5, 0.8]]]                            # geodesic: one wall, both ends inside the box
GEO_END = [[[0.5, 0.0], [0.5, 0.6]]]                        # geodesic: one wall, one end on the boundary
SHIFT = np.array([1000.0, -500.0])
LROOM = {"boundary": [[0, 0], [1, 0], [1, 0.5], [0.5, 0.5], [0.5, 1], [0, 1]], "walls": [[[0.25, 0.0], [0.25, 0.3]]]}
HOLED = {"boundary": [[0, 0], [1, 0], [1, 1], [0, 1]], "holes": [[[0.4, 0.4], [0.6, 0.4], [0.6, 0.6], [0.4, 0.6]]],
         "walls": [[[0.8, 0.0], [0.8, 0.35]]]}


def _close(got, want, lo, hi, gaussian, what=""):
    got, want = np.asarray(got, dtype=float), np.asarray(want, dtype=float)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    span = abs(hi - lo)
    err = np.abs(got - want)
    assert err.max() <= TOL * span, f"{what}: max |err| {err.max():.3e} = {err.max() / span:.2e} of the span"
    if gaussian:
        big = np.abs(want) > 1e-3 * span
        rel = (err[big] / np.abs(want[big])).max()
        assert rel <= TOL, f"{what}: max relative err {rel:.3e}"


def _box(scale, walls=(), periodic=False):
    """The box of side `scale` with the unit box's `walls` scaled into it: (engine, oracle) environments."""
    walls = (np.asarray(walls, dtype=float).reshape(-1, 2, 2) * scale).tolist()
    bc = "periodic" if periodic else "solid"
    E = rb.Environment({"scale": scale, "boundary_conditions": bc})
    for w in walls:
        E.add_wall(w)
    return E, O.OracleEnvironment(scale=scale, walls=walls, boundary_conditions=bc)


def _polygon(spec):
    """A unit-size polygon environment of test_polygon_boundary_and_holes_golden, translated by SHIFT."""
    mv = lambda pts: (np.asarray(pts, dtype=float) + SHIFT).tolist()
    prm = {"boundary": mv(spec["boundary"]), "walls": [mv(w) for w in spec["walls"]]}
    if "holes" in spec:
        prm["holes"] = [mv(h) for h in spec["holes"]]
    return rb.Environment(dict(prm)), O.OracleEnvironment(**prm)


def _inside(env, P):
    return np.array([env.contains(p) for p in P], dtype=bool)


def _positions(rs, env, centres=(), widths=(), n_random=2000, n_ring_centres=24):
    """Random positions in the environment, its extent's corners (where |p - box centre| is largest) and 1e-9 inside
    them, and rings at d in [0, 3.7 w] around centres (so the relative check has samples at every rate level)."""
    e = env.extent
    lo, hi = np.array([e[0], e[2]]), np.array([e[1], e[3]])
    P = [lo + rs.uniform(size=(n_random, 2)) * (hi - lo)]
    for cx in (0, 1):
        for cy in (0, 1):
            c = np.array([e[cx], e[2 + cy]])
            P.append(np.array([c, c + 1e-9 * np.sign((lo + hi) / 2 - c)]))
    centres, widths = np.asarray(centres, dtype=float).reshape(-1, 2), np.asarray(widths, dtype=float).reshape(-1)
    if len(centres):
        idx = rs.choice(len(centres), min(n_ring_centres, len(centres)), replace=False)
        ang = np.linspace(0, 2 * np.pi, 6, endpoint=False)
        d = np.linspace(0, 3.7, 16)
        for i in idx:
            r = d[:, None] * widths[i]
            P.append((centres[i] + np.stack([r * np.cos(ang), r * np.sin(ang)], -1)).reshape(-1, 2))
    P = np.concatenate(P)
    if env.boundary_conditions == "periodic":
        return np.mod(P, env.scale)
    keep = (P[:, 0] >= e[0]) & (P[:, 0] <= e[1]) & (P[:, 1] >= e[2]) & (P[:, 1] <= e[3])
    if not env.is_rectangular or env.holes:
        keep &= _inside(env, P)
    return P[keep]


def _centres(rs, extent, n):
    """n cell centres in the extent, four of them at its corners (the largest |c - box centre|)."""
    lo, hi = np.array([extent[0], extent[2]]), np.array([extent[1], extent[3]])
    c = lo + rs.uniform(size=(n, 2)) * (hi - lo)
    c[:4] = [[extent[0], extent[2]], [extent[1], extent[2]], [extent[0], extent[3]], [extent[1], extent[3]]]
    return c


def _agent(E, n=1, seed=3):
    return rb.Agent(E, {"dt": 0.01, "n_agents": n, "seed": seed})


def _walls_of(geom):
    return {"line_of_sight": C2, "geodesic": GEO}.get(geom, ())


def _wall_ends(env):
    """The ends of the one inner wall that lie inside the box (the geodesic detours' corners)."""
    return [e for e in np.asarray(env.walls[4], dtype=float) if env.contains(e)]


def _around_ends(rs, env, r_max, n_r=12, n_a=16, jitter=True):
    """Rings of radius (0, r_max] around the inner wall's ends inside the box, clipped to the box: both sides of the wall
    near an end, where blocked pairs have short detours."""
    P = []
    for e in _wall_ends(env):
        r = np.linspace(0, r_max, n_r + 1)[1:, None]
        a = np.linspace(0, 2 * np.pi, n_a, endpoint=False) + (rs.uniform(0, 0.2) if jitter else 0.0)
        P.append((e + np.stack([r * np.cos(a), r * np.sin(a)], -1)).reshape(-1, 2))
    P = np.concatenate(P)
    return P[(P > 0).all(axis=1) & (P < env.scale).all(axis=1)]


def _blocked_big(env, centres, P, want, lo, hi):
    """Pairs whose straight segment crosses the wall and whose reference rate exceeds 1e-3 of the span."""
    blocked = O.distances_accounting_for_environment(env, centres, P, "line_of_sight", O.TapeRNG()) == 1000
    return int((blocked & (np.abs(want - lo) > 1e-3 * abs(hi - lo))).sum())


# ---------------------------------------------------------------------------------------------------- PlaceCells
PC_DESCS = ("gaussian", "gaussian_threshold", "diff_of_gaussians")


def _place_case(E, env, Ag, centres, w, geom, P, expect_expanded, tag):
    """Every profile x {uniform, mixed widths} x {min_fr 0 (folded scale), min_fr > 0}: rates against the oracle, and the
    exponent form the packed meta selects (expanded: one common width, k r2_max <= 10, never geodesic).  Geodesic: the
    sample must hold >= 200 blocked pairs with Gaussian rates above 1e-3 of the span (detours the relative check covers)."""
    rs = np.random.RandomState(11)
    mixed = w * rs.uniform(0.8, 1.25, len(centres))
    for desc in PC_DESCS:
        for widths in ("uniform", "mixed"):
            for lo, hi in ((0.0, 1.0), (0.5, 3.0)):
                N = rb.PlaceCells(Ag, {"place_cell_centres": centres, "widths": w, "description": desc,
                                       "wall_geometry": geom, "min_fr": lo, "max_fr": hi})
                if widths == "mixed":
                    N.place_cell_widths = mixed
                c = N._cells()
                assert (c.k_uniform > 0) == (widths == "uniform")
                expanded = desc == "gaussian" and c.k_uniform > 0 and c.k_uniform * c.r2_max <= 10 and \
                    E.boundary_conditions != "periodic" and geom != "geodesic"
                assert expanded == (expect_expanded and desc == "gaussian" and widths == "uniform"), (tag, desc, widths)
                got = N.get_state(evaluate_at=None, pos=P)
                want = O.place_cells_get_state(env, centres, N.place_cell_widths, P, O.TapeRNG(), desc,
                                               N._effective_geometry(), lo, hi)
                form = "expanded" if expanded else "direct"
                _close(got, want, lo, hi, desc == "gaussian", f"{tag} {desc} {widths} widths ({form}) min_fr {lo}")
                if geom == "geodesic" and desc == "gaussian":
                    assert N._effective_geometry() == "geodesic"
                    assert _blocked_big(env, centres, P, want, lo, hi) >= 200, (tag, desc, widths)
                Ag.Neurons.remove(N)


@pytest.mark.parametrize("geom", ["euclidean", "line_of_sight", "geodesic"])
@pytest.mark.parametrize("wkind", ["0.2", "0.2*scale", "0.05"])
@pytest.mark.parametrize("scale", [0.25, 1.0, 2.5, 10.0])
def test_place_cells_at_scale(scale, wkind, geom):
    w = {"0.2": 0.2, "0.2*scale": 0.2 * scale, "0.05": 0.05}[wkind]
    E, env = _box(scale, _walls_of(geom))
    rs = np.random.RandomState(int(scale * 100) + len(wkind))
    centres = _centres(rs, E.extent, 64)
    P = _positions(rs, env, centres, np.full(64, w))
    expanded = w / scale >= 0.2 - 1e-12
    if geom == "geodesic":                       # never the expanded form; centres and positions around the wall ends
        r = min(2.0 * w, 0.25 * scale)
        near = _around_ends(rs, env, r, n_r=4, n_a=12, jitter=False)
        centres[4:4 + min(40, len(near))] = near[rs.choice(len(near), min(40, len(near)), replace=False)]
        P = np.concatenate([P, _around_ends(rs, env, min(3.0 * w, 0.3 * scale))])
        expanded = False
    Ag = _agent(E)
    # centres inside the box: r2_max = half-diagonal^2, k r2_max = log2(e) (scale / w)^2 / 4, at most 10 for w >= 0.2 scale
    _place_case(E, env, Ag, centres, w, geom, P, expanded, f"scale {scale} w {w} {geom}")


@pytest.mark.parametrize("w", [0.05, 0.2, 2.0])
def test_place_cells_periodic_box_at_scale_10(w):
    E, env = _box(10.0, periodic=True)
    rs = np.random.RandomState(int(w * 10))
    centres = _centres(rs, E.extent, 64)
    P = _positions(rs, env, centres, np.full(64, w))
    P = np.concatenate([P, np.mod(centres[:4] + rs.uniform(-0.5, 0.5, (4, 2)) * w, 10.0)])    # across the wrap
    _place_case(E, env, _agent(E), centres, w, "euclidean", P, False, f"periodic w {w}")


# ------------------------------------------------------------------------------------------------------ top_hat
EPS = (1e-9, 1e-7, 1e-6, 3e-6)


def _edge_positions(rs, centres, r, n_dirs=8):
    """Positions at r (1 +- eps) from every centre, eps in EPS, in n_dirs random directions each."""
    P = []
    for c in centres:
        for eps in EPS:
            for s in (-1.0, 1.0):
                a = rs.uniform(0, 2 * np.pi, n_dirs)
                P.append(c + r * (1 + s * eps) * np.stack([np.cos(a), np.sin(a)], -1))
    return np.concatenate(P)


def _detour_edge(rs, env, w, n_c=6, n_dirs=6):
    """Centres within w of each inner-wall end inside the box, on one side of the wall, and positions on the other side at
    detour distance |c - e| + |e - p| = w (1 +- eps) for eps in EPS: p = e + (w (1 +- eps) - |c - e|) u, with the centre
    and u both pointing away from the wall's other end (so the straight segment c -> p crosses the wall)."""
    C, P = [], []
    wall = np.asarray(env.walls[4], dtype=float)
    for k, e in enumerate(wall):
        if not env.contains(e):
            continue
        along = (e - wall[1 - k]) / np.linalg.norm(e - wall[1 - k])      # from the other end out through e
        side = np.array([-along[1], along[0]])
        for _ in range(n_c):
            a = rs.uniform(0.2, 0.8) * w
            t = rs.uniform(0.15, 0.85) * np.pi / 2                         # back along the wall, on side +1
            c = e + a * (-np.cos(t) * along + np.sin(t) * side)
            C.append(c)
            for eps in EPS:
                for s in (-1.0, 1.0):
                    t2 = rs.uniform(0.15, 0.85, n_dirs)[:, None] * np.pi / 2   # back along the wall, on side -1
                    u = -np.cos(t2) * along - np.sin(t2) * side
                    P.append(e + (w * (1 + s * eps) - a) * u)
    return np.array(C), np.concatenate(P)


@pytest.mark.parametrize("geom", ["euclidean", "line_of_sight", "periodic", "geodesic"])
@pytest.mark.parametrize("scale", [1.0, 10.0])
def test_top_hat_on_the_edge(scale, geom):
    w = 0.1
    E, env = _box(scale, _walls_of(geom), periodic=geom == "periodic")
    rs = np.random.RandomState(int(scale) + len(geom))
    centres = _centres(rs, E.extent, 40)
    centres[:4] += np.sign(scale / 2 - centres[:4]) * 1.5 * w          # corner cells with their whole edge in the box
    P = _edge_positions(rs, centres, w)
    if geom == "geodesic":
        dc, dp = _detour_edge(rs, env, w)
        centres = np.concatenate([centres, dc])
        P = np.concatenate([P, dp])
    if geom == "periodic":
        P = np.mod(P, scale)
    else:
        P = P[(P >= 0).all(axis=1) & (P <= scale).all(axis=1)]
    Ag = _agent(E)
    N = rb.PlaceCells(Ag, {"place_cell_centres": centres, "widths": w, "description": "top_hat",
                           "wall_geometry": "euclidean" if geom == "periodic" else geom})
    got = N.get_state(evaluate_at=None, pos=P)
    want = O.place_cells_get_state(env, centres, N.place_cell_widths, P, O.TapeRNG(), "top_hat", N._effective_geometry(),
                                   scalar_width=w)
    near = np.abs(O.distances_accounting_for_environment(env, centres, P, "euclidean", O.TapeRNG()) / w - 1) < 1e-5
    assert near.sum() > 1000 and 0 < want[near].mean() < 1                  # both sides of the edge are represented
    if geom == "geodesic":                                                  # and both sides of the detour edge
        blocked = O.distances_accounting_for_environment(env, centres, P, "line_of_sight", O.TapeRNG()) == 1000
        dg = O.distances_accounting_for_environment(env, centres, P, "geodesic", O.TapeRNG())
        edge = blocked & (np.abs(dg / w - 1) < 1e-5)
        assert edge.sum() > 200 and 0 < want[edge].mean() < 1, edge.sum()
    bad = got != want
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} pairs classified differently (near the edge: {near.sum()})"


def test_goal_radius_at_scale_10():
    """SpatialGoalEnvironment's goal test (the top_hat kernel, line of sight) at scale 10 with a 0.1 m goal radius, with
    agents on both sides of the radius; the expected decisions are the oracle's float64 line-of-sight distances."""
    scale, r = 10.0, 0.1
    walls = (np.asarray(C2) * scale).tolist()
    rs = np.random.RandomState(5)
    goals = _centres(rs, [0, scale, 0, scale], 24)
    goals[:4] += np.sign(scale / 2 - goals[:4]) * 1.5 * r
    P = _edge_positions(rs, goals, r, n_dirs=4)
    P = P[(P > 0).all(axis=1) & (P < scale).all(axis=1)]
    np.random.seed(1)
    genv = SpatialGoalEnvironment({"scale": scale, "walls": walls}, n_agents=len(P), possible_goal_positions=goals,
                                  reset_n_goals=len(goals), goal_radius=r)
    reached = genv._apply_rules(0.01, positions=P).cpu().numpy()              # (A, G), every goal active
    env = O.OracleEnvironment(scale=scale, walls=walls)
    want = (O.distances_accounting_for_environment(env, goals, P, "line_of_sight", O.TapeRNG()) < r).T
    assert 0.2 < want.sum() / len(P) < 0.8
    bad = reached != want
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} goal decisions differ"


# ------------------------------------------------------------------------------------------------------ one_hot
def _one_hot_layout(scale, periodic):
    """Centres on a uniform grid (spacing 1 cm at scale 1, 10 cm at scale 10) at the far corner -- across the wrap in the
    periodic box -- with agents on the midpoints of the grid's edges and on its 4-way corners; exact duplicates of some
    centres at later indices (the first index wins); pairs of centres whose distances to an agent differ by 1e-9 m, the
    farther one first."""
    h = 0.01 * scale
    k = 12
    x0 = scale - 6.3 * h if periodic else scale - (k + 0.7) * h
    g = x0 + h * np.arange(k)
    if periodic:
        g = np.mod(g, scale)
    gx, gy = np.meshgrid(g, g)
    C = [np.stack([gx.ravel(), gy.ravel()], -1)]
    mid = x0 + h * (np.arange(k - 1) + 0.5)
    P = [np.stack(np.meshgrid(mid, g), -1).reshape(-1, 2), np.stack(np.meshgrid(g, mid), -1).reshape(-1, 2),
         np.stack(np.meshgrid(mid, mid), -1).reshape(-1, 2)]
    C.append(C[0][::7].copy())                                                 # duplicates, later indices
    rs = np.random.RandomState(int(scale))
    pairs, pts = [], []
    for i in range(60):
        p = np.array([0.05, 0.05]) * scale + rs.uniform(size=2) * 0.3 * scale
        d = rs.uniform(0.1, 1.0) * h
        a, b = rs.uniform(0, 2 * np.pi, 2)
        pairs += [p + (d + 1e-9) * np.array([np.cos(a), np.sin(a)]), p + d * np.array([np.cos(b), np.sin(b)])]
        pts.append(p)
    C.append(np.array(pairs))
    P.append(np.array(pts))
    P.append(rs.uniform(size=(300, 2)) * scale)
    P = np.concatenate(P)
    return np.concatenate(C), (np.mod(P, scale) if periodic else P)


@pytest.mark.parametrize("geom", ["euclidean", "line_of_sight", "periodic", "geodesic"])
@pytest.mark.parametrize("scale", [1.0, 10.0])
def test_one_hot_arg_min_at_scale(scale, geom):
    periodic = geom == "periodic"
    cut = [[[0.9, 0.85], [0.9, 0.95]]]                                       # a wall through the grid
    walls = {"line_of_sight": C2 + cut, "geodesic": cut}.get(geom, ())
    E, env = _box(scale, walls, periodic=periodic)
    centres, P = _one_hot_layout(scale, periodic)
    Ag = _agent(E)
    N = rb.PlaceCells(Ag, {"place_cell_centres": centres, "description": "one_hot",
                           "wall_geometry": "euclidean" if periodic else geom})
    got = N.get_state(evaluate_at=None, pos=P)
    dist = O.distances_accounting_for_environment(env, centres, P, N._effective_geometry(), O.TapeRNG())
    want_idx = np.argmin(dist, axis=0)
    assert np.array_equal(got.sum(axis=0), np.ones(len(P)))
    got_idx = np.argmax(got, axis=0)
    bad = got_idx != want_idx
    assert not bad.any(), f"{int(bad.sum())} of {len(P)} arg-min indices differ, e.g. {got_idx[bad][:5]} vs {want_idx[bad][:5]}"
    # the layout does produce ties and near-ties
    s = np.sort(dist, axis=0)
    assert ((s[1] - s[0]) <= 1e-9 * scale).sum() > 100


# ---------------------------------------------------------------------------------------------------- GridCells
@pytest.mark.parametrize("desc", ["rectified_cosines", "shifted_cosines"])
@pytest.mark.parametrize("scale,gridscale", [(1.0, None), (1.0, 0.1), (2.5, None), (10.0, None)])
def test_grid_cells_at_scale(scale, gridscale, desc):
    E, env = _box(scale)
    rs = np.random.RandomState(int(scale * 10) + len(desc))
    Ag = _agent(E)
    lo, hi = (0.0, 1.0) if desc == "rectified_cosines" else (0.5, 3.0)
    prm = {"n": 60, "description": desc, "min_fr": lo, "max_fr": hi}
    if gridscale is not None:
        prm.update({"gridscale_distribution": "delta", "gridscale": gridscale})
    N = rb.GridCells(Ag, prm)
    ph = rs.uniform(-300, 300, (N.n, 2))                                       # phase offsets far from [0, 2 pi)
    ph[: N.n // 4] = rs.uniform(0, 2 * np.pi, (N.n // 4, 2))
    N.phase_offsets = ph
    P = _positions(rs, env, n_random=5000)
    got = N.get_state(evaluate_at=None, pos=P)
    want = O.grid_cells_get_state(N.gridscales, N.phase_offsets, N.w, P, desc, N.width_ratio, lo, hi)
    _close(got, want, lo, hi, False, f"grid scale {scale} gridscale {gridscale} {desc}")


# -------------------------------------------------------------------------------------------- far-off coordinates
@pytest.mark.parametrize("name", ["lroom", "holed"])
def test_polygons_far_from_the_origin(name):
    """Every positional kernel must centre its float32 coordinates: one that does not is off by ~1e-4 m here."""
    E, env = _polygon(LROOM if name == "lroom" else HOLED)
    rs = np.random.RandomState(9)
    e = env.extent
    centres = e[[0, 2]] + rs.uniform(size=(300, 2)) * (e[[1, 3]] - e[[0, 2]])
    centres = centres[_inside(env, centres)][:48]
    P = _positions(rs, env, centres, np.full(len(centres), 0.1), n_random=1500)
    assert len(P) > 1000
    Ag = _agent(E)
    for geom in ("euclidean", "line_of_sight"):
        N = rb.PlaceCells(Ag, {"place_cell_centres": centres, "widths": 0.1, "wall_geometry": geom})
        want = O.place_cells_get_state(env, centres, N.place_cell_widths, P, O.TapeRNG(), "gaussian", geom)
        _close(N.get_state(evaluate_at=None, pos=P), want, 0, 1, True, f"{name} place {geom}")
    G = rb.GridCells(Ag, {"n": 30})
    want = O.grid_cells_get_state(G.gridscales, G.phase_offsets, G.w, P)
    _close(G.get_state(evaluate_at=None, pos=P), want, 0, 1, False, f"{name} grid")
    B = rb.BoundaryVectorCells(Ag, {"n": 20})
    want = O.bvc_get_state(env, B.tuning_distances, B.tuning_angles, B.sigma_distances, B.sigma_angles, P, O.TapeRNG())
    _close(B.get_state(evaluate_at=None, pos=P), want, 0, 1, False, f"{name} bvc")
    objs = centres[:3]
    for o in objs:
        E.add_object(o, type=0)
    ovc = rb.ObjectVectorCells(Ag, {"n": 20, "object_tuning_type": 0})
    want = O.ovc_get_state(env, E.objects["objects"], E.objects["object_types"], ovc.tuning_distances, ovc.tuning_angles,
                           ovc.sigma_distances, ovc.sigma_angles, ovc.tuning_types, P, O.TapeRNG(), "line_of_sight")
    _close(ovc.get_state(evaluate_at=None, pos=P), want, 0, 1, False, f"{name} ovc")
    _pppc_at(E, env, centres, 0.1, P, f"{name} pppc")
    N = rb.RandomSpatialNeurons(Ag, {"n": 10, "lengthscale": 0.1, "wall_geometry": "euclidean"})
    want = R.get_state(env, N.X, N.targets, N.lengthscale, "euclidean", P, O.TapeRNG())
    _close(N.get_state(evaluate_at=None, pos=P), want, 0, 1, False, f"{name} rsn")


def _pppc_at(E, env, centres, w, P, tag, geom="euclidean"):
    """PhasePrecessingPlaceCells evaluated at agents placed on P with random velocities (the factor needs the velocity)."""
    rs = np.random.RandomState(len(P))
    Ag = _agent(E, n=len(P))
    Ag.pos = P
    vel = rs.normal(0, 0.1, P.shape)
    Ag.velocity = vel
    for desc in ("gaussian", "gaussian_threshold"):
        N = PPPC(Ag, {"place_cell_centres": centres, "widths": w, "description": desc, "wall_geometry": geom,
                      "kappa": 1.0, "theta_freq": 8.0, "precess_fraction": 0.7})
        want = PP.get_state_rows(env, P, vel, Ag.t, centres, N.place_cell_widths, O.TapeRNG(), desc, N._effective_geometry(),
                                 0.0, 1.0, N.theta_freq, N.sigma, N.precess_fraction)
        _close(N.get_state(), want, 0, PP.peak_factor(N.sigma), False, f"{tag} {desc}")


# ------------------------------------------------------------------------------------ other producers at scale 10
def test_vector_cells_at_scale_10():
    scale = 10.0
    E, env = _box(scale, C2)
    rs = np.random.RandomState(4)
    P = _positions(rs, env, n_random=3000)
    P = P[((P > 0) & (P < scale)).all(axis=1)]     # not on the boundary walls, where the reference's rays are 0 / 0
    Ag = _agent(E)
    for scaled in (False, True):
        B = rb.BoundaryVectorCells(Ag, {"n": 30})
        if scaled:                                                             # tunings scaled with the box
            B.tuning_distances, B.sigma_distances = B.tuning_distances * scale, B.sigma_distances * scale
        want = O.bvc_get_state(env, B.tuning_distances, B.tuning_angles, B.sigma_distances, B.sigma_angles, P, O.TapeRNG())
        _close(B.get_state(evaluate_at=None, pos=P), want, 0, 1, False, f"bvc scaled tuning {scaled}")
    objs = [[1.5, 2.0], [5.0, 8.0], [8.5, 3.0], [9.9, 9.9]]
    for i, o in enumerate(objs):
        E.add_object(o, type=i % 2)
    for occlude in (True, False):
        ovc = rb.ObjectVectorCells(Ag, {"n": 24, "walls_occlude": occlude, "tuning_distance": (0.5, 3.0),
                                        "sigma_distance": (0.8, 12)})
        want = O.ovc_get_state(env, E.objects["objects"], E.objects["object_types"], ovc.tuning_distances,
                               ovc.tuning_angles, ovc.sigma_distances, ovc.sigma_angles, ovc.tuning_types, P, O.TapeRNG(),
                               ovc.wall_geometry)
        _close(ovc.get_state(evaluate_at=None, pos=P), want, 0, 1, False, f"ovc occlude {occlude}")
    Ag2 = _agent(E, n=1, seed=4)
    for occlude in (True, False):
        A = rb.AgentVectorCells(Ag, Ag2, {"n": 16, "walls_occlude": occlude, "tuning_distance": (0.5, 3.0)})
        X, Y = P[:1000], P[::-1][:1000]
        want = V.avc_get_state(env, Y, (A.tuning_distances, A.tuning_angles, A.sigma_distances, A.sigma_angles), X,
                               O.TapeRNG(), A.wall_geometry)
        _close(A.get_state(evaluate_at=None, pos=X, other_pos=Y), want, 0, 1, False, f"avc occlude {occlude}")


@pytest.mark.parametrize("geom,w", [("euclidean", 0.2), ("line_of_sight", 0.2), ("geodesic", 0.2), ("geodesic", 0.05)])
def test_phase_precessing_place_cells_at_scale_10(geom, w):
    E, env = _box(10.0, _walls_of(geom))
    rs = np.random.RandomState(6)
    centres = _centres(rs, E.extent, 40)
    P = _positions(rs, env, centres, np.full(40, w), n_random=600, n_ring_centres=8)
    if geom == "geodesic":
        near = _around_ends(rs, env, 2.0 * w, n_r=4, n_a=6, jitter=False)
        n = min(36, len(near))
        centres[4:4 + n] = near[:n]
        P = np.concatenate([P, _around_ends(rs, env, 3.0 * w, n_r=8, n_a=12)])
    _pppc_at(E, env, centres, w, P, f"pppc scale 10 {geom} w {w}", geom)


def test_random_spatial_neurons_large_box():
    """The sample grid has 0.05 m spacing whatever the lengthscale, so a scale-10 box would need a 40 000^2 covariance at
    set-up: the box is 2.5 m with a 5 cm lengthscale instead (L / w = 50, as scale 10 with w = 0.2)."""
    rs = np.random.RandomState(8)
    np.random.seed(8)
    for geom in ("euclidean", "line_of_sight", "geodesic"):
        E, env = _box(2.5, GEO if geom == "geodesic" else C2)
        Ag = _agent(E)
        N = rb.RandomSpatialNeurons(Ag, {"n": 12, "lengthscale": 0.05, "wall_geometry": geom})
        assert N._effective_geometry() == geom
        P = _positions(rs, env, N.X, np.full(len(N.X), 0.05), n_random=1000, n_ring_centres=8)
        want = R.get_state(env, N.X, N.targets, N.lengthscale, geom, P, O.TapeRNG())
        _close(N.get_state(evaluate_at=None, pos=P), want, 0, 1, False, f"rsn {geom}")


# ----------------------------------------------------------------------------------------- launch paths at scale 10
@pytest.mark.parametrize("kind,w", [("place_los", 0.2), ("place_los", 0.05), ("place", 0.2), ("place", 0.05),
                                    ("place_geo", 0.2), ("place_geo", 0.05), ("grid", None)])
def test_run_and_stepped_updates_at_scale_10(kind, w):
    """The agent records are built by the step kernel's producer warps on these paths (not by get_state): the whole-run
    launch of one population, then the stepped API, against the oracle at Ag.pos."""
    E, env = _box(10.0, {"place_los": C2, "place_geo": GEO_END}.get(kind, ()))
    np.random.seed(2)
    A = 700
    Ag = rb.Agent(E, {"dt": 0.05, "n_agents": A, "seed": 5, "speed_mean": 0.5})
    if kind == "grid":
        N = rb.GridCells(Ag, {"n": 48})
        oracle = lambda pos: O.grid_cells_get_state(N.gridscales, N.phase_offsets, N.w, pos).T
    else:
        geom = {"place_los": "line_of_sight", "place_geo": "geodesic"}.get(kind, "euclidean")
        N = rb.PlaceCells(Ag, {"n": 200, "widths": w, "wall_geometry": geom})
        assert N._effective_geometry() == geom
        assert not (N._cells().k_uniform * N._cells().r2_max <= 10)             # the direct exponent form
        oracle = lambda pos: O.place_cells_get_state(env, N.place_cell_centres, N.place_cell_widths, pos, O.TapeRNG(),
                                                     "gaussian", geom).T
    Ag.run(12)
    _close(N.firingrate, oracle(Ag.pos), 0, 1, kind != "grid", f"{kind} run")
    for _ in range(3):
        Ag.update()
        N.update()
    _close(N.firingrate, oracle(Ag.pos), 0, 1, kind != "grid", f"{kind} stepped")

"""History rate maps on the GPU (riab_history_rate_maps / k_history_maps): ``Agent.get_position_heatmap`` and
``Neurons.get_history_rate_maps`` against a float64 NumPy reference of ``utils.bin_data_for_histogramming``
(utils.py:544-589) over the same float32 history rows.

* Bin edges: agents forced onto every edge of dx = 0.25 (exact in float32), onto the float32 neighbours of every edge of
  dx = 0.1 and 0.07 (not representable), onto the edges of dx = 0.4 (whose last edge lies beyond the extent), a float32
  ulp outside the extent, and onto NaN positions; PlaceCells (n = 70: more than one lane pass, a padded row), a linear
  FeedForwardLayer (signed rates) and AgentVectorCells with a NaN partner row (NaN rates at finite positions);
  one agent.
* Rings: the Agent ring wrapped, a population ring shorter than the Agent's, a population created after Agent steps:
  the maps pair the last min(rows) steps of both rings by step.
* Full size: 65 536 agents x the default 1 024-row Agent ring (2^26 samples, 2^24 a bin at dx = 0.5) and a 256-row
  ring of 64 PlaceCells (2^24 samples).

Counts must equal np.histogram2d's; maps must be within 1e-9 * sum|r| / count of the float64 reference in every bin,
with NaN in the same bins and the same empty-bin mask."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ratinabox_b200 as rb                      # noqa: E402

REL = 1e-9                                       # float64 sums of <= 2^23 samples a bin, in any order
F32 = np.float32


def _edges(extent, dx):
    """bin_data_for_histogramming's edges."""
    return np.arange(extent[0], extent[1] + dx, dx), np.arange(extent[2], extent[3] + dx, dx)


def _bin_index(x, e):
    """np.histogramdd's bin of every x over edges e (searchsorted right, the last edge inclusive), -1 outside / NaN."""
    i = np.searchsorted(e, x, side="right") - 1
    i[x == e[-1]] = len(e) - 2
    i[(i < 0) | (i > len(e) - 2)] = -1
    return i


def _check_heatmap(Ag, dx, pos):
    """get_position_heatmap(dx) equals np.histogram2d of ``pos`` (float64 of the float32 history rows)."""
    ex, ey = _edges(Ag.Environment.extent, dx)
    want = np.histogram2d(pos[:, 0], pos[:, 1], bins=[ex, ey])[0].T[::-1, :]
    got = Ag.get_position_heatmap(dx=dx)
    assert got.shape == want.shape and np.array_equal(got, want), f"dx={dx}: counts differ by {np.abs(got - want).max()}"
    return want


def _check_maps(Ns, dx, pos, fr):
    """get_history_rate_maps(dx) against per-cell weighted np.histogram2d of the paired rows ``pos`` / ``fr``."""
    ex, ey = _edges(Ns.Agent.Environment.extent, dx)
    count = np.histogram2d(pos[:, 0], pos[:, 1], bins=[ex, ey])[0]
    c1 = np.maximum(count, 1)
    maps, zero = Ns.get_history_rate_maps(dx=dx, return_zero_bins=True)
    assert maps.shape == (Ns.n,) + count.T.shape
    assert np.array_equal(zero, (count == 0).T[::-1, :])
    for c in range(Ns.n):
        s = np.histogram2d(pos[:, 0], pos[:, 1], bins=[ex, ey], weights=fr[:, c])[0]
        a = np.histogram2d(pos[:, 0], pos[:, 1], bins=[ex, ey], weights=np.abs(fr[:, c]))[0]
        want, bound = (s / c1).T[::-1, :], (REL * a / c1).T[::-1, :]
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(maps[c]), nan), f"dx={dx} cell {c}: NaN bins differ"
        err = np.abs(maps[c] - want)[~nan]
        assert np.all(err <= bound[~nan]), f"dx={dx} cell {c}: {np.max(err - bound[~nan])} over the bound"


def _paired(Ag, Ns):
    """The last min(rows) steps of both rings, paired by step: (positions (n*A, 2), rates (n*A, n_cells))."""
    ha, hn = Ag.get_history_arrays(), Ns.get_history_arrays()
    n = min(len(ha["t"]), len(hn["t"]))
    assert n > 0 and np.array_equal(ha["t"][len(ha["t"]) - n:], hn["t"][len(hn["t"]) - n:])
    A = Ag.n_agents
    pos = ha["pos"].reshape(-1, A, 2)[-n:].reshape(-1, 2)
    fr = hn["firingrate"].reshape(-1, A, Ns.n)[-n:].reshape(-1, Ns.n)
    return pos, fr


# ----------------------------------------------------------------------------------------------------------- bin edges
EXTENT = (0.0, 3.0, 0.0, 1.5)                     # Environment aspect 2, scale 1.5
DXS = (0.25, 0.1, 0.07, 0.4)


def _neighbours(v):
    """The float32 values on either side of v (v itself when it is a float32), as float64."""
    f = F32(v)
    return np.unique(np.array([np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))], dtype=np.float64))


def _probe_positions():
    """Float32-exact positions: every edge of every DXS grid and its float32 neighbours on x (at a fixed interior y) and
    on y (at a fixed interior x), every dx = 0.25 grid point (interior edges, the right-most x and top y edges, the
    corners), the extent's corners with their float32 neighbours (an ulp outside the extent included), and NaN rows."""
    x0, y0 = float(F32(1.2345678)), float(F32(0.6180339))
    pts = []
    for dx in DXS:
        ex, ey = _edges(EXTENT, dx)
        for e in ex:
            pts += [(x, y0) for x in _neighbours(e)]
        for e in ey:
            pts += [(x0, y) for y in _neighbours(e)]
    ex, ey = _edges(EXTENT, 0.25)
    pts += [(x, y) for x in ex for y in ey]
    for cx in (EXTENT[0], EXTENT[1]):
        for cy in (EXTENT[2], EXTENT[3]):
            pts += [(x, y) for x in _neighbours(cx) for y in _neighbours(cy)]
    pts += [(np.nan, y0), (x0, np.nan), (np.nan, np.nan)] * 3
    return np.array(pts, dtype=np.float64)


def _forced_run(Ag, pops, probes, rs):
    """Step the Agent through ``probes`` (shuffled over agents and steps, the last step padded with interior points),
    updating every population after each step."""
    A = Ag.n_agents
    steps = -(-len(probes) // A)
    pad = np.stack([rs.uniform(0.05, 2.95, steps * A - len(probes)), rs.uniform(0.05, 1.45, steps * A - len(probes))], 1)
    pad = pad.astype(F32).astype(np.float64)
    allpos = np.concatenate([probes, pad])[rs.permutation(steps * A)].reshape(steps, A, 2)
    for s in range(steps):
        Ag.update(forced_next_position=allpos[s] if A > 1 else allpos[s, 0])
        for N in pops:
            N.update()
    return allpos


@pytest.fixture(scope="module")
def edge_run():
    np.random.seed(5)
    E = rb.Environment({"aspect": 2, "scale": 1.5})
    assert list(E.extent) == list(EXTENT)
    A = 97
    Ag = rb.Agent(E, {"dt": 0.01, "n_agents": A, "seed": 3})
    Ag2 = rb.Agent(E, {"dt": 0.01, "n_agents": A, "seed": 4})
    partner = Ag2.pos.copy()
    partner[13] = np.nan
    Ag2.pos = partner
    PCs = rb.PlaceCells(Ag, {"n": 70, "widths": 0.4, "wall_geometry": "euclidean"})
    FFL = rb.FeedForwardLayer(Ag, {"n": 9, "input_layers": [PCs], "activation_function": {"activation": "linear"}})
    AVCs = rb.AgentVectorCells(Ag, Ag2)
    rs = np.random.RandomState(7)
    probes = _probe_positions()
    allpos = _forced_run(Ag, [PCs, FFL, AVCs], probes, rs)
    return Ag, {"place": PCs, "ffl": FFL, "avc": AVCs}, allpos


@pytest.mark.parametrize("dx", DXS)
def test_heatmap_on_bin_edges(edge_run, dx):
    Ag, _, allpos = edge_run
    pos = Ag.get_history_arrays()["pos"].reshape(-1, 2)
    # forced positions get no boundary condition: the history holds the probes exactly (NaN rows included)
    assert np.array_equal(pos, allpos.reshape(-1, 2), equal_nan=True)
    heat = _check_heatmap(Ag, dx, pos)
    ex, ey = _edges(EXTENT, dx)
    inside = (pos[:, 0] >= ex[0]) & (pos[:, 0] <= ex[-1]) & (pos[:, 1] >= ey[0]) & (pos[:, 1] <= ey[-1])
    assert heat.sum() == inside.sum() < len(pos)                     # NaN rows and outside rows are dropped
    if dx == 0.25:
        # every dx = 0.25 grid point is a sample: a point on the right-most / top edge lands in the last bin
        top_right = (pos[:, 0] == 3.0) & (pos[:, 1] == 1.5)
        assert top_right.sum() > 0 and heat[0, -1] >= top_right.sum()
        assert np.any(pos[:, 0] == np.float64(np.nextafter(F32(3.0), F32(4.0))))


@pytest.mark.parametrize("dx", DXS)
@pytest.mark.parametrize("kind", ["place", "ffl", "avc"])
def test_rate_maps_on_bin_edges(edge_run, kind, dx):
    Ag, pops, _ = edge_run
    Ns = pops[kind]
    pos, fr = _paired(Ag, Ns)
    if kind == "place":
        assert Ns.n == 70 and Ns._ld() == 72
        # Neurons.update zeroes the rates when x is NaN (the reference tests pos[0] only); a NaN y gives NaN rates.
        # Both samples are dropped, so neither their zeros nor their NaNs reach a bin.
        xnan, ynan = np.isnan(pos[:, 0]), np.isnan(pos[:, 1]) & ~np.isnan(pos[:, 0])
        assert xnan.any() and np.all(fr[xnan] == 0) and ynan.any() and np.all(np.isnan(fr[ynan]))
    if kind == "ffl":
        assert (fr < 0).any() and (fr > 0).any()
    if kind == "avc":
        assert np.isnan(fr).any() and not np.isnan(fr[:, 0].reshape(-1, Ag.n_agents)[:, 12]).any()
    _check_maps(Ns, dx, pos, fr)
    if kind == "avc":
        maps = Ns.get_history_rate_maps(dx=dx)
        assert np.isnan(maps).any() and not np.isnan(maps).all()


def test_one_agent_on_bin_edges():
    np.random.seed(6)
    E = rb.Environment({"aspect": 2, "scale": 1.5})
    Ag = rb.Agent(E, {"dt": 0.01, "n_agents": 1, "seed": 3})
    PCs = rb.PlaceCells(Ag, {"n": 70, "widths": 0.4, "wall_geometry": "euclidean"})
    rs = np.random.RandomState(8)
    ex, ey = _edges(EXTENT, 0.25)
    probes = np.array([(x, y) for x in ex[::3] for y in ey[::2]] + [(3.0, 1.5), (np.nan, 0.5)])
    _forced_run(Ag, [PCs], probes, rs)
    pos, fr = _paired(Ag, PCs)
    assert pos.shape == (len(probes), 2)
    for dx in (0.25, 0.07):
        _check_heatmap(Ag, dx, pos)
        _check_maps(PCs, dx, pos, fr)


# --------------------------------------------------------------------------------------------------------------- rings
def _ring_maps(Ag, pops, dx=0.1):
    pos_all = Ag.get_history_arrays()["pos"].reshape(-1, 2)
    _check_heatmap(Ag, dx, pos_all)
    for Ns in pops:
        pos, fr = _paired(Ag, Ns)
        _check_maps(Ns, dx, pos, fr)


def test_rings_wrapped_and_population_ring_shorter():
    np.random.seed(9)
    A = 130
    E = rb.Environment()
    Ag = rb.Agent(E, {"dt": 0.05, "n_agents": A, "seed": 1, "history_bytes_limit": 30 * A * 32})
    PCs = rb.PlaceCells(Ag, {"n": 70, "widths": 0.3, "history_bytes_limit": 11 * A * 72 * 4})
    for _ in range(4):
        Ag.update(); PCs.update()
    Ag.run(41)
    assert Ag._hist_cap == 30 and PCs._hist_cap == 11 and Ag._hist_rows == PCs._hist_rows == 45
    assert (Ag._hist_rows - 11) % Ag._hist_cap != 0                  # the maps start mid-ring in the Agent ring
    assert len(Ag.get_history_arrays()["t"]) == 30 and len(PCs.get_history_arrays()["t"]) == 11
    _ring_maps(Ag, [PCs])


def test_population_created_after_agent_steps():
    np.random.seed(10)
    A = 130
    E = rb.Environment()
    Ag = rb.Agent(E, {"dt": 0.05, "n_agents": A, "seed": 2, "history_bytes_limit": 40 * A * 32})
    for _ in range(7):
        Ag.update()
    PCs = rb.PlaceCells(Ag, {"n": 33, "widths": 0.3})
    Ag.run(20)
    GCs = rb.GridCells(Ag, {"n": 6})
    Ag.run(25)                                                          # the Agent ring (40 rows) wraps
    assert Ag._hist_rows == 52 and Ag._hist_cap == 40
    assert len(PCs.get_history_arrays()["t"]) == 45 and len(GCs.get_history_arrays()["t"]) == 25
    _ring_maps(Ag, [PCs, GCs])


# ----------------------------------------------------------------------------------------------------------- full size
FULL_A, FULL_N, FULL_ROWS, FULL_STEPS = 65536, 64, 256, 1100
CHUNK = 8                                                               # ring rows per host chunk


@pytest.fixture(scope="module")
def full_run():
    np.random.seed(11)
    E = rb.Environment()
    Ag = rb.Agent(E, {"dt": 0.01, "n_agents": FULL_A, "seed": 5})
    PCs = rb.PlaceCells(Ag, {"n": FULL_N, "wall_geometry": "euclidean",
                             "history_bytes_limit": FULL_ROWS * FULL_A * FULL_N * 4})
    Ag.run(FULL_STEPS)
    torch.cuda.synchronize()
    yield Ag, PCs
    del Ag, PCs
    import gc
    gc.collect()
    torch.cuda.empty_cache()


def _ring_rows(obj, n):
    """Ring indices of the last n rows, oldest first."""
    return (np.arange(obj._hist_rows - n, obj._hist_rows)) % obj._hist_cap


def test_full_size_rings(full_run):
    Ag, PCs = full_run
    assert Ag._hist_cap == 1024 and Ag._hist_rows == FULL_STEPS                  # the default ring, wrapped
    assert PCs._hist_cap == FULL_ROWS and PCs._hist_rows == FULL_STEPS
    # the step times of the rows the maps pair (get_history_arrays would copy 2 GiB + 4 GiB of rows to the host)
    assert np.array_equal(Ag._t_hist[-FULL_ROWS:], PCs._t_hist[-FULL_ROWS:])


@pytest.mark.parametrize("dx", [0.5, None])
def test_full_size_heatmap(full_run, dx):
    """2^26 samples: dx = 0.5 puts 2^24 samples in the mean bin, beyond a float32 count."""
    Ag, _ = full_run
    ex, ey = _edges(Ag.Environment.extent, Ag.Environment.dx * 5 if dx is None else dx)
    want = np.zeros((len(ex) - 1, len(ey) - 1))
    rows = _ring_rows(Ag, 1024)
    for k in range(0, len(rows), 64):
        p = Ag._hist[torch.as_tensor(rows[k:k + 64], device=Ag.device), :, :2].cpu().numpy().astype(np.float64)
        want += np.histogram2d(p[..., 0].ravel(), p[..., 1].ravel(), bins=[ex, ey])[0]
    want = want.T[::-1, :]
    heat = Ag.get_position_heatmap() if dx is None else Ag.get_position_heatmap(dx=dx)
    assert want.sum() == 2 ** 26
    assert heat.shape == want.shape
    assert heat.sum() == 2 ** 26 and np.array_equal(heat, want), \
        f"heat sums to {heat.sum():.0f}, max |count error| {np.abs(heat - want).max():.0f}"
    assert np.array_equal(heat, Ag.get_position_heatmap() if dx is None else Ag.get_position_heatmap(dx=dx))


@pytest.mark.parametrize("dx", [0.5, 0.05])
def test_full_size_rate_maps(full_run, dx):
    """2^24 paired samples of 64 cells, float64 sums built on the host in chunks of ring rows."""
    Ag, PCs = full_run
    ex, ey = _edges(Ag.Environment.extent, dx)
    nx, ny, n = len(ex) - 1, len(ey) - 1, FULL_N
    count, s, a = np.zeros(nx * ny), np.zeros(nx * ny * n), np.zeros(nx * ny * n)
    arows, prows = _ring_rows(Ag, FULL_ROWS), _ring_rows(PCs, FULL_ROWS)
    cols = np.arange(n)
    for k in range(0, FULL_ROWS, CHUNK):
        p = Ag._hist[torch.as_tensor(arows[k:k + CHUNK], device=Ag.device), :, :2]
        p = p.cpu().numpy().astype(np.float64).reshape(-1, 2)
        r = PCs._hist[torch.as_tensor(prows[k:k + CHUNK], device=Ag.device), :, :n]
        r = r.cpu().numpy().astype(np.float64).reshape(-1, n)
        ix, iy = _bin_index(p[:, 0], ex), _bin_index(p[:, 1], ey)
        ok = (ix >= 0) & (iy >= 0)
        b = (ix * ny + iy)[ok]
        count += np.bincount(b, minlength=nx * ny)
        idx = (b[:, None] * n + cols).ravel()
        r = r[ok]
        s += np.bincount(idx, weights=r.ravel(), minlength=nx * ny * n)
        a += np.bincount(idx, weights=np.abs(r).ravel(), minlength=nx * ny * n)
    assert count.sum() == 2 ** 24
    count = count.reshape(nx, ny)
    c1 = np.maximum(count, 1)[:, :, None]
    want = (s.reshape(nx, ny, n) / c1).transpose(2, 1, 0)[:, ::-1, :]
    bound = (REL * a.reshape(nx, ny, n) / c1).transpose(2, 1, 0)[:, ::-1, :]
    maps, zero = PCs.get_history_rate_maps(dx=dx, return_zero_bins=True)
    assert np.array_equal(zero, (count == 0).T[::-1, :])
    assert maps.shape == want.shape
    rel = np.abs(maps - want) / np.where(bound > 0, bound / REL, 1)
    assert np.all(np.abs(maps - want) <= bound), f"worst error {rel.max():.3e} of sum|r| / count (bound {REL:.0e})"

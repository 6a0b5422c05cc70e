"""CPU checks of RandomSpatialNeurons (ratinabox/Neurons.py:2865-2954): the float64 oracle (oracle/riab_oracle_rsn.py)
and the host mirror's set-up against the live reference's fixture (tests/golden/rsn.npz, oracle/gen_rsn_golden.py),
the operand packing of riab_rsn_pack, the struct layouts and the kernel's resources.  No CUDA calls.

The targets come from multivariate_normal, i.e. LAPACK's SVD of a covariance with degenerate eigenspaces: they are
compared with a recomputation in this process, never with the fixture's numbers, which another BLAS may not give."""
import contextlib
import ctypes as C
import hashlib
import io
import json
import os
import re
import types

import numpy as np
import pytest

import riab_oracle as O
import riab_oracle_rsn as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C2_WALLS = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
HOLE = [[0.4, 0.4], [0.6, 0.4], [0.6, 0.6], [0.4, 0.6]]
BOX = [[0, 0], [1, 0], [1, 1], [0, 1]]
# name: (environment, RandomSpatialNeurons params, seed) -- oracle/gen_rsn_golden.py's ENVS
ENVS = {
    "box": (dict(), {"n": 10, "lengthscale": 0.1, "wall_geometry": "euclidean"}, 1),
    "wall21": (dict(aspect=2, walls=[[[1.0, 0.0], [1.0, 0.6]]]), {"n": 12, "lengthscale": 0.1}, 2),
    "c2": (dict(walls=C2_WALLS), {"n": 10, "lengthscale": 0.1}, 3),
    "periodic": (dict(boundary_conditions="periodic"), {"n": 9, "lengthscale": 0.15, "wall_geometry": "euclidean"}, 4),
    "holed": (dict(boundary=BOX, walls=[[[0.8, 0.0], [0.8, 0.35]]], holes=[HOLE]),
              {"n": 8, "lengthscale": 0.08, "wall_geometry": "line_of_sight", "min_fr": 0.5, "max_fr": 3.0}, 5),
    "long": (dict(), {"n": 10, "lengthscale": 0.02, "wall_geometry": "euclidean"}, 6),
}
DEFAULTS = {"lengthscale": 0.1, "max_fr": 1, "min_fr": 0, "n": 10, "wall_geometry": "geodesic"}


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _rng_state(g, name):
    return (g[f"{name}_rng_keys"], int(g[f"{name}_rng_pos"]), int(g[f"{name}_rng_has_gauss"]), float(g[f"{name}_rng_cached"]))


def _same_state(st, want):
    return (np.array_equal(st[1], want[0]) and st[2] == want[1] and st[3] == want[2] and st[4] == want[3])


def _oracle_env(spec):
    return O.OracleEnvironment(**spec)


def _mirror_env(spec):
    import ratinabox_b200 as rb
    spec = dict(spec)
    walls = spec.pop("walls", [])
    if "boundary" in spec:
        return rb.Environment(dict(spec, walls=walls))
    prm = {"aspect": spec["aspect"]} if "aspect" in spec else {}
    if "boundary_conditions" in spec:
        prm["boundary_conditions"] = spec["boundary_conditions"]
    env = rb.Environment(prm)
    for w in walls:
        env.add_wall(w)
    return env


def _mirror(env, params):
    """The host set-up of the mirror on a stand-in Agent (constructing a real Agent needs a GPU)."""
    import ratinabox_b200 as rb
    N = object.__new__(rb.RandomSpatialNeurons)
    N.Agent = types.SimpleNamespace(Environment=env)
    for k, v in dict(DEFAULTS, **params).items():
        setattr(N, k, v)
    N._set_up()
    return N


@pytest.mark.parametrize("name", list(ENVS))
def test_oracle_reproduces_the_fixture_bit_for_bit(golden, name):
    """Grid, covariance (hash and rows, the reference's jitter draws), the RNG tape through the target draw, and
    get_state at the fixture's positions (jitter off) from the fixture's targets."""
    g = golden("rsn.npz")
    spec, prm, seed = ENVS[name]
    env = _oracle_env(spec)
    geom = str(g[f"{name}_geometry"])
    X = R.sample_grid(env.extent, prm["lengthscale"])
    assert np.array_equal(X, g[f"{name}_X"])
    np.random.seed(seed)
    Q = R.kernel(env, X, X, prm["lengthscale"], geom, O.GlobalRNG())
    assert _sha(Q) == str(g[f"{name}_Q_sha256"])
    assert np.array_equal(Q[g[f"{name}_Q_rows_idx"]], g[f"{name}_Q_rows"])
    R.targets_from(Q, prm["n"], prm.get("min_fr", 0), prm.get("max_fr", 1))
    assert _same_state(np.random.get_state(), _rng_state(g, name))
    gs = R.get_state(env, X, g[f"{name}_targets"], prm["lengthscale"], geom, g[f"{name}_P"], O.TapeRNG())
    assert np.array_equal(gs, g[f"{name}_gs"])


@pytest.mark.parametrize("name", list(ENVS))
def test_host_mirror_set_up_matches_the_reference(golden, name):
    """X and Q equal the reference's, construction consumes the same draws in the same order, the targets equal
    activate(multivariate_normal(Q)) recomputed here under the same seed, and the printed messages match."""
    g = golden("rsn.npz")
    spec, prm, seed = ENVS[name]
    np.random.seed(seed)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        N = _mirror(_mirror_env(spec), prm)
    st = np.random.get_state()
    assert buf.getvalue() == str(g[f"{name}_printed"])
    assert N.wall_geometry == str(g[f"{name}_geometry"])
    assert np.array_equal(N.X, g[f"{name}_X"])
    assert _sha(N.Q) == str(g[f"{name}_Q_sha256"])
    assert _same_state(st, _rng_state(g, name))
    np.random.seed(seed)
    env = _oracle_env(spec)
    Q = R.kernel(env, N.X, N.X, prm["lengthscale"], N.wall_geometry, O.GlobalRNG())
    want = R.targets_from(Q, prm["n"], prm.get("min_fr", 0), prm.get("max_fr", 1))
    assert N.targets.shape == (N.X.shape[0], prm["n"]) and np.array_equal(N.targets, want)


def test_parameters_and_messages(golden):
    import ratinabox_b200 as rb
    g = golden("rsn.npz")
    ref = json.loads(str(g["default_params_json"]))
    assert ref == rb.RandomSpatialNeurons.default_params
    with pytest.raises(AssertionError) as e:
        _mirror(_mirror_env({}), {"lengthscale": 0.01})
    assert str(e.value) == str(g["msg_lengthscale"])
    np.random.seed(0)
    with pytest.raises(AssertionError) as e:                      # no euclidean fall-back for periodic boundaries
        _mirror(_mirror_env({"boundary_conditions": "periodic"}), {"n": 2})
    assert str(e.value) == str(g["msg_periodic_geodesic"])
    with pytest.raises(NotImplementedError):                       # geodesic in a polygon environment
        _mirror(_mirror_env(dict(boundary=BOX)), {"lengthscale": 0.2})
    many = [[[0.05 + 0.1 * i, 0.1], [0.05 + 0.1 * i, 0.3]] for i in range(9)]
    with pytest.raises(NotImplementedError):                       # more inner walls than the kernels hold
        _mirror(_mirror_env(dict(walls=many)), {"lengthscale": 0.2, "wall_geometry": "line_of_sight"})


@pytest.mark.parametrize("n,n_points,geom", [(1, 37, 0), (10, 400, 1), (70, 64, 2)])
def test_rsn_pack_permutation_and_pads(n, n_points, geom):
    from ratinabox_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(n)
    X = rs.uniform(0.05, 0.95, (n_points, 2))
    T = rs.uniform(0.0, 1.0, (n_points, n))
    walls = np.array([[[1, 0], [0, 0]], [[1, 1], [1, 0]], [[0, 1], [1, 1]], [[0, 0], [0, 1]], [[0.5, 0.0], [0.5, 0.6]]],
                     dtype=np.float64)
    ext = np.array([0.0, 1.0, 0.0, 1.0])
    n_inner = 0 if geom == 0 else 1
    kp = (n_points + 31) // 32 * 32
    meta = _lib.RsnCells()
    out = np.full(lib.riab_rsn_pack_floats(n, n_points, n_inner), np.nan, dtype=np.float32)
    cen = np.zeros((kp, 2))
    f64 = lambda a: np.ascontiguousarray(a).ctypes.data_as(_lib.c_double_p)   # noqa: E731
    assert lib.riab_rsn_pack(f64(X), n_points, f64(T), n, 0.1, f64(walls), 5, 4, f64(ext), geom, C.byref(meta),
                             out.ctypes.data_as(_lib.c_float_p), cen.ctypes.data_as(_lib.c_double_p)) == 0
    assert (meta.n_cells, meta.n_points, meta.k_pad, meta.points.n_cells, meta.points.n_inner_walls) == (n, n_points, kp, kp, n_inner)
    # packed position p of stage s holds point s*32 + (8 k8 + q + 4 h) for p % 32 = 8 q + 2 k8 + h; pads repeat point 0
    perm = np.array([(p // 32) * 32 + 8 * ((p % 8) // 2) + (p % 32) // 8 + 4 * (p % 2) for p in range(kp)])
    assert sorted(perm) == list(range(kp))
    want = np.where((perm < n_points)[:, None], X[np.minimum(perm, n_points - 1)], X[0])
    assert np.array_equal(cen, want)
    npad = meta.points.n_pad
    assert np.array_equal(out[:kp], (cen[:, 0] - 0.5).astype(np.float32))          # the place block's centre x
    assert np.allclose(out[2 * npad:2 * npad + kp], np.log2(np.e) / (2 * 0.01), rtol=1e-7)
    tb = out[lib.riab_place_pack_floats(kp, n_inner):]
    n8 = (n + 7) // 8 * 8
    hi, lo = tb[: n8 * kp].reshape(n8, kp), tb[n8 * kp:].reshape(n8, kp)
    assert tb.size == 2 * n8 * kp and np.all(np.isfinite(tb))
    assert np.all(hi[n:] == 0) and np.all(hi[:, n_points:] == 0) and np.all(lo[n:] == 0) and np.all(lo[:, n_points:] == 0)
    s = hi[:n, :n_points].astype(np.float64) + lo[:n, :n_points].astype(np.float64)
    t32 = T.T.astype(np.float32).astype(np.float64)
    assert np.all(np.abs(s - t32) <= 2.0 ** -22 * np.abs(t32))
    assert lib.riab_rsn_pack(None, n_points, f64(T), n, 0.1, f64(walls), 5, 4, f64(ext), geom, C.byref(meta),
                             out.ctypes.data_as(_lib.c_float_p), cen.ctypes.data_as(_lib.c_double_p)) < 0


def test_rsn_kernel_resources():
    """Every k_rsn instantiation (inner-wall slots x profile x N tile x consumer warpgroups) has no local-memory spills
    and fits the register budget of its occupancy: two consumer warpgroups + the producer (288 threads) put 3 warps on
    one SM sub-partition (168 registers), one warpgroup (160 threads) 2 (255)."""
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([tool, "--dump-resource-usage", _lib.lib_path()], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*5k_rsnILi(\d+)ELi(n?\d+)ELi(\d+)ELi(\d+)E\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) "
                       r"LOCAL:(\d+)", txt)
    got = sorted((int(f[1]), f[2], int(f[3]), int(f[4])) for f in found)
    want = sorted([(wi, "0", bn, 2) for wi in (0, 1, 2) for bn in (8, 32, 64)] + [(1, "n1", bn, 2) for bn in (8, 32, 64)]
                  + [(4, "0", bn, 1) for bn in (8, 32, 64)] + [(8, "0", bn, 1) for bn in (8, 32)])
    assert got == want, got
    for name, wi, desc, bn, cwg, reg, stack, shared, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        assert int(reg) <= (168 if cwg == "2" else 255), (name, reg)


def test_rsn_struct_has_the_headers_layout(tmp_path):
    import shutil
    import subprocess
    from ratinabox_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "riab_b200.h"', "int main(void) {",
           '  printf("%zu %zu %zu %zu %zu %d\\n", sizeof(riab_rsn_cells), offsetof(riab_rsn_cells, targets_dev),'
           ' offsetof(riab_rsn_cells, k_pad), offsetof(riab_rsn_cells, max_fr), offsetof(riab_rsn_cells, reserved),'
           ' RIAB_CELLS_RSN);', "  return 0;", "}"]
    c = tmp_path / "rsn.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "rsn"
    subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    R_ = _lib.RsnCells
    assert got == [C.sizeof(R_), R_.targets_dev.offset, R_.k_pad.offset, R_.max_fr.offset, R_.reserved.offset, _lib.CELLS_RSN]

"""CPU checks of the oracle's geodesic branch (oracle/riab_oracle.py) against the live reference's fixture
(tests/golden/geodesic.npz, oracle/gen_geodesic_golden.py): PlaceCells.get_state bit for bit for every description and
each wall-end case (both ends inside the box, only end 0, only end 1, in an aspect-2 box too), and the same exception
type as the reference for a wall with no end inside the box.  No CUDA calls."""
import numpy as np
import pytest

import riab_oracle as O

DESCS = ("gaussian", "gaussian_threshold", "diff_of_gaussians", "top_hat", "one_hot")


def _env(g, case):
    return O.OracleEnvironment(aspect=float(g[f"{case}_aspect"]), walls=[g[f"{case}_wall"]])


@pytest.mark.parametrize("case", ["free", "end0_aspect2", "end1"])
def test_oracle_reproduces_geodesic_get_state(golden, case):
    g = golden("geodesic.npz")
    env = _env(g, case)
    assert sum(1 << e for e, end in enumerate(g[f"{case}_wall"]) if env.contains(end)) == int(g[f"{case}_ep_valid"])
    C, P = g[f"{case}_centres"], g[f"{case}_pos"]
    w = float(g["width"])
    blocked = O.distances_accounting_for_environment(env, C, P, "line_of_sight", O.TapeRNG()) == 1000
    for desc in DESCS:
        want = g[f"{case}_{desc}"]
        got = O.place_cells_get_state(env, C, np.full(len(C), w), P, O.TapeRNG(), desc, "geodesic",
                                      float(g["min_fr"]), float(g["max_fr"]), scalar_width=w)
        assert np.array_equal(got, want), (case, desc)
        if desc == "gaussian":                  # the fixture holds detours with rates above 1e-3 of the span
            span = float(g["max_fr"]) - float(g["min_fr"])
            assert (blocked & (want - float(g["min_fr"]) > 1e-3 * span)).sum() >= 100, case


def test_oracle_raises_as_the_reference_for_a_wall_with_no_end_inside(golden):
    g = golden("geodesic.npz")
    for k in ("no_end_place_get_state", "no_end_pppc_update", "no_end_rsn_init"):
        assert str(g[k]) == "ValueError", k
    env = O.OracleEnvironment(walls=[g["no_end_wall"]])
    with pytest.raises(ValueError):
        O.place_cells_get_state(env, [[0.2, 0.5], [0.8, 0.5]], [0.2, 0.2], [[0.2, 0.5]], O.TapeRNG(), "gaussian",
                                "geodesic")

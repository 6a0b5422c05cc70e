"""CPU: the NumPy restatement of ThetaSequenceAgent.update (oracle/riab_oracle_tsa.py) against tests/golden/tsa.npz, written
from the live reference by oracle/gen_tsa_golden.py; the lazy forward rollout against the eager one; and the positions
defined where the reference raises."""
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import riab_oracle as O  # noqa: E402
from riab_oracle_tsa import OracleTSA  # noqa: E402

G = np.load(os.path.join(ROOT, "tests", "golden", "tsa.npz"))
WALLS2 = [[[0.3, 0.0], [0.3, 0.5]], [[0.7, 1.0], [0.7, 0.5]]]
RUNS = ("open", "walls", "periodic")
REPLAYS = ("slow", "gap", "ahead_up", "ahead_down")


def oracle_env(kind):
    if kind == "periodic":
        return O.OracleEnvironment(boundary_conditions="periodic")
    return O.OracleEnvironment(walls=WALLS2 if kind == "walls" else ())


def replay(key, mode, xi=None):
    """(positions, raised, oracle) of the recorded lead through OracleTSA; xi: rollout normals (default: recorded)."""
    m = json.loads(str(G[f"{key}_meta"]))
    lp = m["lead_params"]
    sm = lp.get("speed_mean", 0.08)
    tsa = OracleTSA(oracle_env(m["env"]), m["tsa_params"], lp["dt"], sm, m["avg_speed"], m["lead_pos0"], mode=mode,
                    fwd_state0=(m["fwd_mv0"], m["fwd_hd0"]))
    xi = G[f"{key}_fwd_xi"] if xi is None else xi
    starts = list(G[f"{key}_fwd_start"])
    T = len(G[f"{key}_lead_t"])
    pos, raised, r = np.full((T, 2), np.nan), np.zeros(T, bool), -1
    for s in range(T):
        if s in starts:
            r = starts.index(s)
        normals = xi[r] if r >= 0 else np.zeros((0, 2))
        pos[s], raised[s] = tsa.step(G[f"{key}_lead_pos"][s], G[f"{key}_lead_vel"][s], G[f"{key}_lead_rot"][s],
                                     G[f"{key}_lead_dist"][s], G[f"{key}_lead_t"][s], normals[~np.isnan(normals[:, 0])],
                                     m["fwd_kwargs"])
    return pos, raised, tsa


@pytest.mark.parametrize("mode", ["eager", "lazy"])
@pytest.mark.parametrize("key", RUNS + REPLAYS)
def test_oracle_matches_the_reference_where_it_returns(key, mode):
    pos, raised, _ = replay(key, mode)
    ref, ref_raised = G[f"{key}_tsa_pos"], G[f"{key}_raised"]
    assert np.array_equal(raised, ref_raised)
    ok = ~ref_raised
    assert ok.sum() >= len(ok) - 1
    assert np.array_equal(pos[ok], ref[ok], equal_nan=True)
    if key in RUNS:                      # both halves of the sweep and the NaN ends occur
        nan = np.isnan(ref[:, 0])
        assert 0.3 < nan.mean() < 0.7
        assert (~nan & (G[f"{key}_phase"] < 0.5)).sum() > 20 and (~nan & (G[f"{key}_phase"] >= 0.5)).sum() > 20


@pytest.mark.parametrize("key", RUNS)
def test_oracle_rollouts_match_the_reference(key):
    _, _, tsa = replay(key, "eager")
    fd, fp = G[f"{key}_fwd_dist"], G[f"{key}_fwd_pos"]
    assert len(tsa.rollouts) == len(fd) > 10
    for i, (d, p) in enumerate(tsa.rollouts):
        n = min(len(d), fd.shape[1])
        assert np.array_equal(np.array(d[:n]), fd[i, :n]) and np.array_equal(np.array(p[:n]), fp[i, :n])


def test_runs_cover_the_window_and_the_counter_rule():
    m = json.loads(str(G["open_meta"]))
    assert len(G["open_lead_t"]) > int(5 * 0.125 / (0.01 * m["avg_speed"])) == 781     # a full look-behind window
    _, _, tsa = replay("walls", "lazy")
    assert tsa.keep_count == 1000 and len(G["walls_lead_t"]) > tsa.keep_count          # the stash counter wrapped
    assert tsa.counter < len(G["walls_lead_t"])


@pytest.mark.parametrize("key", RUNS)
def test_lazy_rollout_equals_eager_rollout_plus_interp1d(key):
    """The lazy rollout (steps taken only up to each query) gives the eager rollout's interp1d positions bit for bit, on
    fresh normals too; it takes far fewer forward steps."""
    rs = np.random.RandomState(11)
    xi = rs.normal(size=G[f"{key}_fwd_xi"].shape)
    pe, re, te = replay(key, "eager", xi)
    pl, rl, tl = replay(key, "lazy", xi)
    assert np.array_equal(re, rl)
    assert np.array_equal(pe, pl, equal_nan=True)
    assert sum(len(d) for d, _ in tl.rollouts) < sum(len(d) for d, _ in te.rollouts)


def test_defined_positions_where_the_reference_raises():
    for key in REPLAYS:
        m = json.loads(str(G[f"{key}_meta"]))
        assert m["error"].startswith("ValueError:"), (key, m["error"])
        assert G[f"{key}_raised"][-1]
    # slow lead: the target precedes every row of the window -> NaN
    pos, raised, _ = replay("slow", "lazy")
    assert raised[-1] and np.isnan(pos[-1]).all()
    # a gap: interpolated between the two window rows that bracket the target
    pos, raised, tsa = replay("gap", "lazy")
    rows = np.array(tsa.rows)                       # 12 rows: the whole window of the last step
    d, p = rows[:, 0], rows[:, 1:]
    c = tsa.d_half / tsa.theta_frac
    t = d[-1] - (-2 * c * G["gap_phase"][-1] + c)
    j = int(np.searchsorted(d, t))
    assert d[j - 1] < t < d[j] and j < 3
    want = ((t - d[j - 1]) / (d[j] - d[j - 1])) * p[j] + ((d[j] - t) / (d[j] - d[j - 1])) * p[j - 1]
    assert raised[-1] and np.array_equal(pos[-1], want)
    # look ahead with the lead's distance edited past the rollout's end / before its start -> NaN
    for key in ("ahead_up", "ahead_down"):
        pos, raised, _ = replay(key, "lazy")
        assert raised[-1] and np.isnan(pos[-1]).all() and not np.isnan(pos[-2]).any()


def test_messages():
    assert json.loads(str(G["default_params_json"])) == {"theta_frac": 0.5, "theta_freq": 10.0, "v_sequence": 5.0}
    assert str(G["assert_dt"]).startswith("params['dt'] for the LeadAgent is too large")
    assert str(G["assert_v"]).startswith("params['v_sequence'] is too small")
    assert "overwritten to match dt of the LeadAgent" in str(G["dt_warning"])

// ThetaSequenceAgent.update (ratinabox/contribs/SubAgent.py:245-350) for ONE agent per thread, in float64: the position
// of the theta sweep at this lead step.  The host decides the phase (one clock for every agent) and passes the signed
// distance offset of the sweep; the forced step that moves the ThetaSequenceAgent there is the ordinary
// riab_agent_update_src launch that follows.
//
// Look behind: interp1d over the lead's recent (distance, position) rows, kept in a private float64 ring.
// Look ahead: the reference rolls a forward agent out eagerly to a stop distance and interpolates in that rollout; here
// the rollout advances lazily, only as far as this step's query, keeping the last two rollout samples.  The query never
// decreases within a sweep and neither does the rollout's distance, so the pair interp1d would pick is the kept pair.
#pragma once
#include "riab_motion.cuh"

namespace riab {

RIAB_DEV double theta_nan() { return __longlong_as_double(0x7ff8000000000000ll); }

// scipy.interpolate.interp1d(kind="linear") between (x_lo, y_lo) and (x_hi, y_hi)  (_interpolate.py: _call_linear)
RIAB_DEV double interp_linear(double x, double x_lo, double x_hi, double y_lo, double y_hi) {
  const D w = D(x_hi) - D(x_lo);
  return ((D(x) - D(x_lo)) / w * D(y_hi) + (D(x_hi) - D(x)) / w * D(y_lo)).v;
}

// The look-behind window: logical rows j = 0 (oldest) .. w-1 (this step's lead row) of the (3, R, A) ring.
struct ThetaWindow {
  const double* ring;
  long long A, R, first, w, i;
  RIAB_DEV long long at(long long j) const {
    long long s = first + j;
    if (s >= R) s -= R;
    return s * A + i;
  }
  RIAB_DEV double d(long long j) const { return ring[2 * R * A + at(j)]; }
  RIAB_DEV double x(long long j) const { return ring[at(j)]; }
  RIAB_DEV double y(long long j) const { return ring[R * A + at(j)]; }
  // np.searchsorted(d, t) (side="left"): the first row whose distance is >= t (the distances never decrease)
  RIAB_DEV long long search_left(double t) const {
    long long lo = 0, hi = w;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (d(mid) < t) lo = mid + 1; else hi = mid;
    }
    return lo;
  }
  // interp1d over rows [s0, s1) at t, which lies in [d(s0), d(s1-1)]; `left` = search_left(t)
  RIAB_DEV void interp(double t, long long left, long long s0, long long s1, double& px, double& py) const {
    long long j = left < s0 + 1 ? s0 + 1 : left;
    if (j > s1 - 1) j = s1 - 1;
    const double dl = d(j - 1), dh = d(j);
    px = interp_linear(t, dl, dh, x(j - 1), x(j));
    py = interp_linear(t, dl, dh, y(j - 1), y(j));
  }
};

// SubAgent.py:274-300 for target distance t = lead distance - distance_back.
RIAB_DEV void theta_look_behind(const ThetaWindow& W, double t, double& px, double& py) {
  const long long w = W.w;
  const long long left = W.search_left(t);
  // idx = np.argmin(np.abs(d - t)): the first row of least |d - t|.  Rows below `left` have |d - t| = fl(t - d), which
  // does not increase with the row; rows from `left` on have fl(d - t), which does not decrease.
  long long idx;
  if (left == 0) {
    idx = 0;
  } else {
    const double va = fabs(__dsub_rn(W.d(left - 1), t));
    if (left < w && fabs(__dsub_rn(W.d(left), t)) < va) {
      idx = left;
    } else {
      // the first row before `left` whose |d - t| equals va (equal distances, or differences that round alike)
      long long lo = 0, hi = left - 1;
      if (hi > 0 && fabs(__dsub_rn(W.d(hi - 1), t)) > va) lo = hi;
      while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (fabs(__dsub_rn(W.d(mid), t)) > va) lo = mid + 1; else hi = mid;
      }
      idx = lo;
    }
  }
  // interp1d(d[idx-3:idx+3], pos[idx-3:idx+3]) -- where the reference raises (idx < 3: an empty slice; t outside the
  // slice: bounds_error), interpolate between the bracketing rows of the whole window; NaN before the window's start.
  if (idx >= 3) {
    const long long s0 = idx - 3, s1 = (idx + 3 < w) ? idx + 3 : w;
    if (t >= W.d(s0) && t <= W.d(s1 - 1)) { W.interp(t, left, s0, s1, px, py); return; }
  }
  if (w < 2 || !(t >= W.d(0))) { px = py = theta_nan(); return; }
  W.interp(t, left, 0, w, px, py);
}

// Two standard normals of forward-rollout step k of rollout r of one agent.
RIAB_DEV void theta_fwd_normals(uint64_t seed, uint64_t rollout, uint64_t k, uint64_t agent, double& n1, double& n2) {
  uint32_t c[4];
  philox_ctr(c, agent, (uint32_t)rollout, k, RIAB_STREAM_THETA_FWD, 0u);
  philox_normals(c, seed, n1, n2);
}

}  // namespace riab

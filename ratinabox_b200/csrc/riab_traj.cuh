// Imported trajectories: the not-a-knot cubic spline of scipy's interp1d(kind="cubic") (Agent.py:607-632) in second-
// derivative (M) form.  The times are shared by every trajectory, so the tridiagonal system is the same for every
// (trajectory, axis) column: the host eliminates it once (riab_trajectory_build), the device sweeps each column.
// D arithmetic throughout, so tests/spline_np.py reproduces M bit for bit.
#pragma once
#include "riab_motion.cuh"

namespace riab {

// Motion source of a step inside a kernel (riab_motion_source without the ABI padding)
struct SrcK {
  int kind, bcast;
  double t;                     // Agent.t of the first step of the launch
  const double* times;          // (T)
  const double* y;              // (T, n_traj, 2)
  const double* M;              // (T, n_traj, 2)
  long long T, n_traj;
  double t_max;
  const double* forced;         // (A,2) or (2)
};

// Host-side elimination factors of the not-a-knot system over M_1 .. M_{T-2} (m = T-2 rows), row j = node j+1:
//   h_j M_j + 2 (h_j + h_{j+1}) M_{j+1} + h_{j+1} M_{j+2} = 6 (d_{j+1} - d_j),  d_i = (y_{i+1} - y_i) / h_i,
// with M_0 = ((h_0 + h_1) M_1 - h_0 M_2) / h_1 eliminated from the first row (and M_{T-1} likewise from the last):
//   b_0 = (h_0 + h_1)(h_0 + 2 h_1) / h_1,  c_0 = (h_1^2 - h_0^2) / h_1.
// Diagonally dominant, so no pivoting.  Layout of `fac` (4m + T - 1 doubles): w[m] (forward multipliers, w[0] unused),
// bp[m] (eliminated diagonal), c[m] (super-diagonal), h[T-1].
inline void traj_factors(const double* x, long long T, double* fac) {
  const long long m = T - 2;
  double *w = fac, *bp = fac + m, *c = fac + 2 * m, *h = fac + 3 * m;
  for (long long i = 0; i + 1 < T; ++i) h[i] = x[i + 1] - x[i];
  std::vector<double> a(m);
  for (long long j = 0; j < m; ++j) { a[j] = h[j]; bp[j] = 2.0 * (h[j] + h[j + 1]); c[j] = h[j + 1]; }
  const double h0 = h[0], h1 = h[1], hm1 = h[T - 2], hm2 = h[T - 3];
  bp[0] = (h0 + h1) * (h0 + 2.0 * h1) / h1; c[0] = (h1 * h1 - h0 * h0) / h1; a[0] = 0.0;
  bp[m - 1] = (hm1 + hm2) * (hm1 + 2.0 * hm2) / hm2; a[m - 1] = (hm2 * hm2 - hm1 * hm1) / hm2; c[m - 1] = 0.0;
  w[0] = 0.0;
  for (long long j = 1; j < m; ++j) { w[j] = a[j] / bp[j - 1]; bp[j] = bp[j] - w[j] * c[j - 1]; }
}

// One thread per column (trajectory, axis) of the (T, ncol) layout: forward sweep of the right-hand side (stored in M),
// back substitution in place, then the two end values.
__global__ void __launch_bounds__(128) k_traj_build(const double* __restrict__ y, double* __restrict__ M,
                                                     const double* __restrict__ fac, long long T, long long ncol) {
  const long long col = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= ncol) return;
  const long long m = T - 2;
  const double *w = fac, *bp = fac + m, *c = fac + 2 * m, *h = fac + 3 * m;
  D y0(y[col]), y1(y[ncol + col]);
  D d0 = (y1 - y0) / D(h[0]);
  D r(0.0);
  for (long long j = 0; j < m; ++j) {
    const D y2(y[(j + 2) * ncol + col]);
    const D d1 = (y2 - y1) / D(h[j + 1]);
    const D rj = D(6.0) * (d1 - d0);
    r = (j == 0) ? rj : rj - D(w[j]) * r;
    M[(j + 1) * ncol + col] = r.v;
    y1 = y2; d0 = d1;
  }
  D mn = D(M[m * ncol + col]) / D(bp[m - 1]);
  M[m * ncol + col] = mn.v;
  D mnn(0.0);
  for (long long j = m - 2; j >= 0; --j) {
    mnn = mn;
    mn = (D(M[(j + 1) * ncol + col]) - D(c[j]) * mnn) / D(bp[j]);
    M[(j + 1) * ncol + col] = mn.v;
  }
  // mn = M_1, mnn = M_2
  const D h0(h[0]), h1(h[1]), hm1(h[T - 2]), hm2(h[T - 3]);
  M[col] = (((h0 + h1) * mn - h0 * mnn) / h1).v;
  const D ml(M[m * ncol + col]), ml2(M[(m - 1) * ncol + col]);
  M[(T - 1) * ncol + col] = (((hm1 + hm2) * ml - hm1 * ml2) / hm2).v;
}

// Segment k with times[k] <= q < times[k+1], clipped to [0, T-2] (the same q for a whole warp: broadcast loads).
RIAB_DEV long long traj_segment(const double* __restrict__ x, long long T, double q) {
  long long lo = 0, hi = T - 1;          // invariant: x[lo] <= q (or lo == 0), q < x[hi] (or hi == T-1)
  while (hi - lo > 1) {
    const long long mid = (lo + hi) >> 1;
    if (x[mid] <= q) lo = mid; else hi = mid;
  }
  return lo;
}

// S(q) of trajectory `tr_i` on segment k:
//   M_k A^3/6h + M_{k+1} B^3/6h + (y_k/h - M_k h/6) A + (y_{k+1}/h - M_{k+1} h/6) B,  A = x_{k+1} - q, B = q - x_k
RIAB_DEV double2 traj_eval(const SrcK& src, long long tr_i, long long k, double q) {
  const D x0(src.times[k]), x1(src.times[k + 1]);
  const D h = x1 - x0, A = x1 - D(q), B = D(q) - x0;
  const D A3 = A * A * A, B3 = B * B * B, h6 = D(6.0) * h;
  const double2 ya = reinterpret_cast<const double2*>(src.y)[k * src.n_traj + tr_i];
  const double2 yb = reinterpret_cast<const double2*>(src.y)[(k + 1) * src.n_traj + tr_i];
  const double2 ma = reinterpret_cast<const double2*>(src.M)[k * src.n_traj + tr_i];
  const double2 mb = reinterpret_cast<const double2*>(src.M)[(k + 1) * src.n_traj + tr_i];
  auto s = [&](double y0, double y1, double m0, double m1) {
    const D M0(m0), M1(m1);
    return (M0 * A3 / h6 + M1 * B3 / h6 + (D(y0) / h - M0 * h / D(6.0)) * A + (D(y1) / h - M1 * h / D(6.0)) * B).v;
  };
  return make_double2(s(ya.x, yb.x, ma.x, mb.x), s(ya.y, yb.y, ma.y, mb.y));
}

// The imported / forced branches of Agent.update for agent i at time t (Agent.py:202-242): new position from the
// source, then the shared A8-A10 tail with overwrite_velocity semantics.  f1, f2: keys of the zero-displacement draw.
RIAB_DEV void source_step(AgentState& s, const SrcK& src, long long i, double t, const riab_motion_params& p,
                          const MotionDerived& m, bool periodic, double scale, double f1, double f2) {
  double nx, ny;
  if (src.kind == RIAB_MOTION_IMPORTED) {
    const double q = fmod(t, src.t_max);                     // self.t % max(self.t_interp), Agent.py:257
    const long long k = traj_segment(src.times, src.T, q);
    const double2 v = traj_eval(src, src.n_traj == 1 ? 0 : i, k, q);
    nx = v.x; ny = v.y;
  } else {
    const long long j = src.bcast ? 0 : i;
    nx = src.forced[2 * j]; ny = src.forced[2 * j + 1];
  }
  const bool nan_step = (nx != nx) || (ny != ny) || (s.px != s.px) || (s.py != s.py);
  D stx, sty, mvx, mvy;
  step_displacement(D(nx), D(ny), D(s.px), D(s.py), periodic, scale, stx, sty);
  measure_tail<true>(s, stx, sty, s.mvx, s.mvy, D(p.dt), p, m, f1, f2, mvx, mvy, nan_step);
  s.px = nx; s.py = ny; s.mvx = mvx.v; s.mvy = mvy.v;
  // overwrite_velocity=True (Agent.py:462-463, :470-471); the NaN case returns before it (:451-454)
  if (!nan_step) { s.vx = mvx.v; s.vy = mvy.v; s.rot = s.mrot; }
}

}  // namespace riab

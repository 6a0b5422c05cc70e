// PhasePrecessingPlaceCells.get_state at the agents (ratinabox/contribs/PhasePrecessingPlaceCells.py:66-119): the
// PlaceCells rate (riab_place.cuh, already scaled to [min_fr, max_fr]) times the theta modulation factor
//   d       = velocity / (1e-8 + |velocity|)                                              (:99, Agent.velocity)
//   phi     = theta_freq (t % (1 / theta_freq)) 2 pi                                       (:100-102)
//   s_i     = ((pos - c_i) . d) / sigma_i,  sigma_i = widths_i (x 2 for "gaussian")        (:103-110)
//   factor  = von_mises(pi - s_i precess_fraction pi - phi, 0, sigma) 2 pi = exp(kappa' cos x) / I0(kappa'),
//             kappa' = 1 / sigma^2                                                         (:111-117, utils.py:441-457)
//
// In turns, x / 2 pi = tau = u - g_i (p.d) + (g_i c_ix) d_x + (g_i c_iy) d_y  with  u = (pi - phi) / 2 pi a launch
// constant and g_i = precess_fraction / (2 sigma_i).  The producer appends (d_x, d_y, p.d) to the place record, in the
// box-centred coordinates of the record (d in float64, rounded once); the consumers hold (g_i, g_i c_ix, g_i c_iy) next
// to the place-cell registers and spend per rate 3 FFMA for tau, an exact reduction tau - rint(tau) into [-1/2, 1/2], one
// cos.approx of 2 pi times that, and ex2(kappa' log2(e) cos + log2 C) with C the reference's normalisation, computed per
// launch on the host in float64 (make_pppc).  g_i comes from the packed k_i = log2(e) / (2 w_i^2): g_i = gs sqrt(k_i),
// gs = precess_fraction / (2 m) sqrt(2 / log2(e)), m = 2 for "gaussian" else 1.
#pragma once
#include "riab_common.cuh"
#include "riab_place.cuh"

namespace riab {

constexpr int pppc_dir(int wi, bool geo) { return place_rec(wi, geo); }   // float index of (d_x, d_y, p.d, 0) in the record
constexpr int pppc_rec(int wi, bool geo) { return place_rec(wi, geo) + 4; }

struct PppcConst : PlaceConst {      // uniform per launch; the PlaceCells constants in their direct form (expanded = fold = 0)
  float u;                          // (pi - phi) / 2 pi of the launch's clock
  float k2;                          // kappa' log2(e)
  float lnorm;                       // log2 of the von Mises normalisation C = 2 pi exp(kappa) / (2 pi I0(kappa)) / exp(kappa)
  double gs;                         // g_i = gs sqrt(k_i)
  const double* vel;                 // MODE 0: the rows' velocities (n_rows, 2)
};

template <int WI>
struct PppcCellRegs {
  PlaceCellRegs<WI> p;
  float g[4], gx[4], gy[4];          // g_i, g_i c_ix, g_i c_iy (box-centred centres)
};

// The cells' phase registers, after the place registers are loaded (r.p.k = k_i, r.p.cx / cy = centres: direct form).
template <int WI>
RIAB_DEV void pppc_load_phase(PppcCellRegs<WI>& r, const PppcConst& c) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double g = c.gs * sqrt((double)r.p.k[i]);          // padding cells: k = 0, g = 0
    r.g[i] = (float)g;
    r.gx[i] = (float)(g * (double)r.p.cx[i]);
    r.gy[i] = (float)(g * (double)r.p.cy[i]);
  }
}

// The record's direction block from the agent's float64 position and velocity.
RIAB_DEV void pppc_direction_record(float* __restrict__ rec, double px, double py, double vx, double vy, double cxm,
                                    double cym) {
  const D n = D(1e-8) + dsqrt(D(vx) * D(vx) + D(vy) * D(vy));   // 1e-8 + np.linalg.norm(velocity)
  const double dx = (D(vx) / n).v, dy = (D(vy) / n).v;
  const double pd = (px - cxm) * dx + (py - cym) * dy;
  *reinterpret_cast<float4*>(rec) = make_float4((float)dx, (float)dy, (float)pd, 0.f);
}

// rates o[i] *= factor_i
template <int WI>
RIAB_DEV void pppc_modulate4(float (&o)[4], const PppcCellRegs<WI>& r, const PppcConst& c, const float* __restrict__ dir) {
  const float4 q = *reinterpret_cast<const float4*>(dir);      // d_x, d_y, p.d
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float tau = fmaf(r.gy[i], q.y, fmaf(r.gx[i], q.x, fmaf(-r.g[i], q.z, c.u)));
    const float f = tau - rintf(tau);                          // exact: the phase in turns, in [-1/2, 1/2]
    const float cs = __cosf(6.2831853071795865f * f);          // cos.approx on an argument within +-pi
    o[i] *= ex2f(fmaf(c.k2, cs, c.lnorm));
  }
}

}  // namespace riab

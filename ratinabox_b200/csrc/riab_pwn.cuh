// PlaneWaveNeurons.get_state (ratinabox/contribs/PlaneWaveNeurons.py:63-91): one cosine per cell,
//   phi  = (2 pi / lambda_i) ((phase_offset_i - pos) . w_i)
//   rate = 0.5 (cos phi + 1) (max_fr - min_fr) + min_fr
// With k_i = w_i / lambda_i (turns per metre) and p' = pos - box centre c, phi / 2 pi = k_i . (phase_offset_i - c) - k_i . p'.
//
// Packed block (float32, riab_pwn_pack), Np = n_cells rounded up to 128:  kx[Np] | ky[Np] | kxl[Np] | kyl[Np] | ph[Np]
//   phase_turns = 0 (radians):  kx, ky = 2 pi k_i,  kxl = kyl = 0,  ph = 2 pi (k_i . (phase_offset_i - c)) reduced to
//                               [-pi, pi] in float64.  Rate error ~ 1.2e-7 |2 pi k| r_max of the rate span (DESIGN.md).
//   phase_turns = 1 (turns):    (kx, kxl), (ky, kyl) = k_i as float32 hi / lo pairs, ph = k_i . (phase_offset_i - c)
//                               reduced to [-1/2, 1/2] in float64.  The record carries p' as float32 hi / lo pairs too, so
//                               k . p' is formed from exact two-products (pwn_phase_turns) to ~1e-7 turns at any |k| |p'|.
#pragma once
#include "riab_common.cuh"

namespace riab {

struct PwnConst {
  int n_cells, n_pad;
  float As, Bs;        // rate = As cos(phi) + Bs:  As = span / 2, Bs = span / 2 + min_fr
  const float* packed;
  int turns;           // riab_pwn_cells::phase_turns
};

struct PwnCellRegs {
  float kx[4], ky[4], kxl[4], kyl[4], ph[4];
};

RIAB_DEV void pwn_load_cells(PwnCellRegs& r, const PwnConst& c, int cell0) {
  const int np = c.n_pad;
  ldv(r.kx, c.packed + 0 * np + cell0);
  ldv(r.ky, c.packed + 1 * np + cell0);
  ldv(r.kxl, c.packed + 2 * np + cell0);
  ldv(r.kyl, c.packed + 3 * np + cell0);
  ldv(r.ph, c.packed + 4 * np + cell0);
}

// The record: p' = pos - c as float32 hi / lo pairs (the lo part is what float32 drops of the float64 difference).
RIAB_DEV void pwn_agent_record(float* __restrict__ rec, double px, double py, double cxm, double cym) {
  const double dx = px - cxm, dy = py - cym;
  const float hx = (float)dx, hy = (float)dy;
  *reinterpret_cast<float4*>(rec) = make_float4(hx, hy, (float)(dx - (double)hx), (float)(dy - (double)hy));
}

// Compensated phase in radians, from turns: -k . p' = -(kh + kl) . (ph + pl).  kh px and kh py are exact two-products
// (product + FMA residual), each product reduced by t - rint(t) (exact in float32) as in grid_phase_turns; the cross terms
// kh pl + kl ph are ~2^-24 |k| |p'| and take plain FMAs (their own rounding is ~2^-48 |k| |p'|), kl pl is dropped.
RIAB_DEV float pwn_phase_turns(float kx, float ky, float kxl, float kyl, float ph, float npx, float npy, float nlx,
                               float nly) {
  float t = __fmul_rn(kx, npx);
  float f = ph + (t - rintf(t));
  f += fmaf(kx, npx, -t);
  t = __fmul_rn(ky, npy);
  f += t - rintf(t);
  f += fmaf(ky, npy, -t);
  f += fmaf(kx, nlx, fmaf(ky, nly, fmaf(kxl, npx, kyl * npy)));
  return 6.28318530717958648f * (f - rintf(f));
}

// The block's form is uniform per launch (PwnConst::turns): one branch per 4 rates, no divergence.
RIAB_DEV void pwn_rates4(float (&out)[4], const PwnCellRegs& r, const PwnConst& c, const float* __restrict__ rec) {
  const float4 p = *reinterpret_cast<const float4*>(rec);
  const float npx = -p.x, npy = -p.y;
  if (c.turns) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      out[i] = fmaf(__cosf(pwn_phase_turns(r.kx[i], r.ky[i], r.kxl[i], r.kyl[i], r.ph[i], npx, npy, -p.z, -p.w)), c.As, c.Bs);
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) out[i] = fmaf(__cosf(fmaf(r.ky[i], npy, fmaf(r.kx[i], npx, r.ph[i]))), c.As, c.Bs);
  }
}

}  // namespace riab

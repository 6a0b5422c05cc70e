// GridCells.get_state, 2D (ratinabox/Neurons.py:1172-1236): rectified / shifted sum
// of three cosines, float32.
//
// Packed block (float32, riab_grid_pack), Np = n_cells rounded up to 4:
//   for k = 0..2:  kx_k[Np] | ky_k[Np] | ph_k[Np]
// with (kx,ky) = (2 pi / gridscale) * w_k  and  ph_k = (2 pi / gridscale) * ((origin - box centre) . w_k)
// reduced to [-pi, pi] in float64, so that   phi_k = ph_k - (p' . k_k),  p' = pos - box centre;
// all three divided by 2 pi (turns) when riab_grid_pack sets phase_turns (large |k| r_max, see grid_phase_turns)
// (Neurons.py:1191-1201: vecs = origin - pos, phi = (2 pi / gridscale) (vecs . w)).
#pragma once
#include "riab_common.cuh"

namespace riab {

struct GridConst {
  int n_cells, n_pad, rectify;
  float A, B;          // f = A * (cos1+cos2+cos3) + B   (then max(0,.) when rectify)
  float min_fr, span;
  // scale folded into the affine map (make_grid): rate = clamp(As * sum + Bs) with As = A span, Bs = B span + min_fr;
  // max(f, 0) span + min_fr = max(As sum + Bs, min_fr) for span >= 0 (min(.) for span < 0)   (Neurons.py:1214,1232-1234)
  float As, Bs;
  int clamp;           // 0: none (shifted cosines), 1: max(., min_fr), 2: min(., min_fr)
  const float* packed;
  double cxm, cym;
  int turns;           // riab_grid_cells::phase_turns: the block holds turns, rates take grid_phase_turns
};

struct GridCellRegs {
  float kx[3][4], ky[3][4], ph[3][4];
};

RIAB_DEV void grid_load_cells(GridCellRegs& r, const GridConst& c, int cell0) {
  const int np = c.n_pad;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    ldv(r.kx[k], c.packed + (3 * k + 0) * np + cell0);
    ldv(r.ky[k], c.packed + (3 * k + 1) * np + cell0);
    ldv(r.ph[k], c.packed + (3 * k + 2) * np + cell0);
  }
}

// Compensated phase in turns (block packed with phase_turns = 1): kx p and ky p as exact two-products (product + FMA
// residual), each product reduced by t - rint(t) (exact in float32), so no rounding ever sees more than ~1.5 turns;
// the sum is reduced once more to [-1/2, 1/2] before __cosf.  What is left is the float32 rounding of p' and of the
// packed wave vector (~2^-24 |k| |p'| each), 3.8e-6 of the rate scale at scale 10 with the default grid scales.
RIAB_DEV float grid_phase_turns(float kx, float ky, float ph, float npx, float npy) {
  // one product at a time (two live values besides the operands); __fmul_rn is never contracted into the sums
  float t = __fmul_rn(kx, npx);
  float f = ph + (t - rintf(t));
  f += fmaf(kx, npx, -t);
  t = __fmul_rn(ky, npy);
  f += t - rintf(t);
  f += fmaf(ky, npy, -t);
  return 6.28318530717958648f * (f - rintf(f));
}

// TURNS = 1: the block holds turns (GridConst::turns, GridPolicy<1>), else radians
template <int TURNS = 0>
RIAB_DEV void grid_rates4(float (&out)[4], const GridCellRegs& r, const GridConst& c, const float* __restrict__ rec) {
  const float2 p = *reinterpret_cast<const float2*>(rec);
  const float npx = -p.x, npy = -p.y;
#pragma unroll
  for (int h = 0; h < 2; ++h) {                       // cell pairs: the three phases are 2 FFMA each per rate
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      float a, b;
      if (TURNS) {
        a = grid_phase_turns(r.kx[k][2 * h], r.ky[k][2 * h], r.ph[k][2 * h], npx, npy);
        b = grid_phase_turns(r.kx[k][2 * h + 1], r.ky[k][2 * h + 1], r.ph[k][2 * h + 1], npx, npy);
      } else {
        a = fmaf(r.ky[k][2 * h], npy, fmaf(r.kx[k][2 * h], npx, r.ph[k][2 * h]));
        b = fmaf(r.ky[k][2 * h + 1], npy, fmaf(r.kx[k][2 * h + 1], npx, r.ph[k][2 * h + 1]));
      }
      if (k == 0) { s0 = __cosf(a); s1 = __cosf(b); }
      else { s0 += __cosf(a); s1 += __cosf(b); }
    }
    float v0 = fmaf(s0, c.As, c.Bs), v1 = fmaf(s1, c.As, c.Bs);
    if (c.clamp == 1) { v0 = fmaxf(v0, c.min_fr); v1 = fmaxf(v1, c.min_fr); }
    else if (c.clamp == 2) { v0 = fminf(v0, c.min_fr); v1 = fminf(v1, c.min_fr); }
    out[2 * h] = v0; out[2 * h + 1] = v1;
  }
}

}  // namespace riab

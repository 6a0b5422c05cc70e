// BoundaryVectorCells.get_state, allocentric (ratinabox/Neurons.py:1617-1778).
//
// Phase A (float64, per agent x test angle): the reference casts T rays
// pos -> pos + test_direction, intersects each with every wall
// (utils.vector_intercepts, utils.py:30-118), scores the walls with
// boundary_vector_preference_function (Neurons.py:1746-1778) and keeps
// l_a of the arg-max wall = distance to the first wall along the ray.  We
// evaluate exactly those float64 expressions (D = non-contracting double) so
// the chosen wall and distance equal the oracle's; the only short-cut is that
// the `l_b < 0` / `l_b > 1` rejections are decided from the signs / magnitudes of
// numerator and denominator (exact for IEEE division) so l_a's division is only
// done for walls that survive.
//
// Phase B (float32, per agent x cell): fr = sum_theta gauss(d_theta; mu_d, sigma_d) *
// vonmises(theta; mu_theta, sigma_theta) / cell_fr_norm.  The von Mises factor does
// not depend on the agent, so it is a precomputed (cell tile x T) table staged into
// shared memory by TMA bulk copies; the Gaussian is one FFMA + FMUL + MUFU.EX2.
//
// Packed block (float32, riab_bvc_pack), Np = n_cells rounded up to BVC_CT (64):
//   s[Np] | m[Np] | scale[Np] | VM tiles: [Np/64][T][64] | kap[Np] | cmu[Np] | smu[Np] | cth[T] | sth[T]
//   s = sqrt(log2(e)/2)/sigma_d, m = mu_d*s, scale = 1/cell_fr_norm,
//   kap = log2(e)/sigma_theta^2, (cmu,smu) = (cos,sin)(mu_theta), (cth,sth) = (cos,sin)(test angle).
// Egocentric cells (FieldOfViewBVCs): the von Mises argument is theta - head_bearing - mu_theta, which
// depends on the agent, so no table: cos(theta - phi) = cth*cos(phi) + sth*sin(phi) with
// (cos,sin)(phi = bearing + mu_theta) formed algebraically per (agent, cell) from the head direction
// (cos(bearing), sin(bearing)) = (x+1e-6, y)/|(x+1e-6, y)|  -- utils.get_angle's eps quirk included --
// and both exponentials share ONE ex2:  2^(kap*(cos-1) - u^2).
// Scratch (phase A -> B): dist_to_first_wall as [agent tile of 32][T][32] float32.
#pragma once
#include "riab_common.cuh"

namespace riab {

constexpr int BVC_CT = 64;   // cells per tile
constexpr int BVC_AT = 32;   // agents per tile

// One ray against all walls -> (distance to first wall, wall id).  Neurons.py:1655-1684.
// wf: float32 copy of the walls as (ax, ay, sbx, sby) per wall (pre-filter only).
//
// Two phases per ray so that the lanes of a warp (different agents / angles) do not serialise on each
// other's walls: (1) a float32 pre-filter over all walls builds a bit mask of the walls that can still be
// the answer; (2) each lane walks ITS OWN set bits in increasing wall order -- same code path for every
// lane, different wall index as data -- and evaluates the reference's float64 expressions.
//
// The pre-filter drops a wall when (a) its l_b is outside [0,1] by more than a margin 1e-3 (>> float32
// rounding; the exact test rejects it too, pref = -1), (b) its l_a is certainly negative (pref = -1, never
// beats the initial maximum), or (c) its l_a is certainly larger than that of another wall that certainly
// scores: the answer is the FIRST wall of maximal 1/l_a, i.e. of minimal positive l_a (Neurons.py:1672-1679),
// so a wall with l_a - err > min over certainly-positive walls of (l_a + err) cannot be it.  err bounds the
// float32 evaluation of l_a = numA / denA generously (1e-5 relative on every product, 1e-6 of the coordinate
// magnitude on every difference; float32 rounding is 6e-8); anything uncertain (NaN, parallel ray, agent on
// a wall line) compares false and is kept for the exact walk.  Typically one wall survives (two at corners).
struct BvcScreen {
  float la_lo, la_hi;
  bool lb_rejected, lb_certain;   // l_b outside [0,1] beyond the margin / inside it beyond the margin
};
// flo = 1e-6 * (coordinate magnitude of the ray origin and all walls) * (longest wall): absolute floor of the numerator's error
RIAB_DEV BvcScreen bvc_screen(const float4 wl, float pxf, float pyf, float sapxf, float sapyf, float flo) {
  const float d0xf = wl.x - pxf, d0yf = wl.y - pyf;
  const float t1 = d0xf * sapxf, t2 = d0yf * sapyf, t3 = wl.z * sapxf, t4 = wl.w * sapyf;
  const float nb = -(t1 + t2), db = t3 + t4;
  const float S = fabsf(t1) + fabsf(t2) + fabsf(t3) + fabsf(t4);
  float inv;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"(db));         // db = 0 (parallel ray): inf -> everything below is kept
  const float ainv = fabsf(inv);
  const float lb = nb * inv;
  const float tolb = fmaf(1e-6f * S, ainv, 1e-3f);                 // margin on l_b (>> float32 rounding of nb / db)
  const float off = fabsf(lb - 0.5f);
  BvcScreen r;
  r.lb_rejected = off > 0.5f + tolb;
  r.lb_certain = off < 0.5f - tolb;
  // l_a = (d0 . sb_perp) / (sa . sb_perp),  sb_perp = (-sby, sbx),  sa . sb_perp = -db
  const float u1 = d0xf * wl.w, u2 = d0yf * wl.z;
  const float la = (u1 - u2) * inv;
  const float e_n = fmaf(1e-5f, fabsf(u1) + fabsf(u2), flo);
  const float err = fmaf(fmaf(fabsf(la), 1e-5f * S, e_n), ainv, 1e-4f * fabsf(la));
  r.la_lo = la - err;
  r.la_hi = la + err;
  return r;
}

// The reference's float64 evaluation (utils.vector_intercepts, utils.py:74-97; preference Neurons.py:1763-1777) of the
// walls in `mask`, in increasing wall order; np.argmax keeps the first maximum.
// bvc_walk_bits: the walls w0 + (set bits of mask), carrying the running maximum (best, besti, best_la) so that
// consecutive blocks of walls walk like one mask; bvc_walk_end: the result.
template <typename MaskT>
RIAB_DEV void bvc_walk_bits(MaskT mask, int w0, double px, double py, double ux, double uy, const double* __restrict__ walls,
                            double& best, int& besti, double& best_la) {
  const D a0x(px), a0y(py);
  const D a1x = a0x + D(ux), a1y = a0y + D(uy);      // pos_line_segments[:, :, 1, :] += test_directions
  const D sax = a1x - a0x, say = a1y - a0y;
  const D sapx = -say, sapy = sax;
  while (mask) {
    const int w = w0 + ((sizeof(MaskT) == 8) ? __ffsll((long long)mask) - 1 : __ffs((int)mask) - 1);
    mask &= mask - 1;
    const D bx0(walls[4 * w]), by0(walls[4 * w + 1]), bx1(walls[4 * w + 2]), by1(walls[4 * w + 3]);
    const D d0x = bx0 - a0x, d0y = by0 - a0y;
    const D sbx = bx1 - bx0, sby = by1 - by0;
    const D sbpx = -sby, sbpy = sbx;
    const D numB = (-d0x) * sapx + (-d0y) * sapy;
    const D denB = sbx * sapx + sby * sapy;
    // l_b = numB/denB : decide (l_b < 0) || (l_b > 1) without dividing (exact for IEEE division)
    bool rej;
    if (denB.v != 0.0 && numB.v == numB.v && fabs(denB.v) != INFINITY && fabs(numB.v) != INFINITY) {
      const bool same = (numB.v > 0.0) == (denB.v > 0.0);
      rej = (numB.v != 0.0) && (!same || fabs(numB.v) > fabs(denB.v));
    } else {
      const double lb = (numB / denB).v;
      rej = (lb < 0.0) || (lb > 1.0);
    }
    if (rej) continue;                                   // pref = -1: never beats the running maximum
    const D numA = d0x * sbpx + d0y * sbpy;
    const D denA = sax * sbpx + say * sbpy;
    const double la = (numA / denA).v;
    const double pref = (la > 0.0) ? __ddiv_rn(1.0, la) : ((la < 0.0) ? -1.0 : 0.0);
    if (pref > best) { best = pref; besti = w; best_la = la; }
  }
}
RIAB_DEV void bvc_walk_end(double px, double py, double ux, double uy, const double* __restrict__ walls, int besti,
                           double best_la, double& dist, int& wall_id) {
  const D a0x(px), a0y(py);
  const D a1x = a0x + D(ux), a1y = a0y + D(uy);
  const D sax = a1x - a0x, say = a1y - a0y;
  if (besti < 0) {
    // every wall scored -1: np.argmax returns wall 0, whose l_a is reported (Neurons.py:1677-1684)
    besti = 0;
    const D bx0(walls[0]), by0(walls[1]), bx1(walls[2]), by1(walls[3]);
    const D d0x = bx0 - a0x, d0y = by0 - a0y;
    const D sbx = bx1 - bx0, sby = by1 - by0;
    const D sbpx = -sby, sbpy = sbx;
    best_la = ((d0x * sbpx + d0y * sbpy) / (sax * sbpx + say * sbpy)).v;
  }
  dist = best_la;
  wall_id = besti;
}
template <typename MaskT>
RIAB_DEV void bvc_walk(MaskT mask, double px, double py, double ux, double uy, const double* __restrict__ walls,
                       double& dist, int& wall_id) {
  double best = -1.0;                                    // rejected walls all score -1
  int besti = -1;
  double best_la = 0.0;
  bvc_walk_bits<MaskT>(mask, 0, px, py, ux, uy, walls, best, besti, best_la);
  bvc_walk_end(px, py, ux, uy, walls, besti, best_la, dist, wall_id);
}

// Generic screen (any number of walls): everything from the float32 wall copies, per (ray, wall).
template <typename MaskT>
RIAB_DEV void bvc_first_wall_impl(double px, double py, double ux, double uy, const double* __restrict__ walls,
                                  const float4* __restrict__ wf, int W, float flo_env, double& dist, int& wall_id) {
  const float pxf = (float)px, pyf = (float)py, sapxf = -(float)uy, sapyf = (float)ux;
  const float flo = flo_env + flo_env * (fabsf(pxf) + fabsf(pyf));
  MaskT mask = 0, bit = 1;
  float thr = INFINITY;                                  // min over certainly-scoring walls of l_a + err
  for (int w = 0; w < W; ++w, bit <<= 1) {
    const BvcScreen sc = bvc_screen(wf[w], pxf, pyf, sapxf, sapyf, flo);
    const bool drop = sc.lb_rejected || (sc.la_hi < 0.f) || (sc.la_lo > thr);
    if (!drop) mask |= bit;
    if (sc.lb_certain && sc.la_lo > 0.f) thr = fminf(thr, sc.la_hi);   // this wall certainly scores 1/l_a > 0
  }
  // walls kept under an earlier, looser bound: test them against the final one before any float64 work
  for (MaskT m = mask; m;) {
    const int w = (sizeof(MaskT) == 8) ? __ffsll((long long)m) - 1 : __ffs((int)m) - 1;
    m &= m - 1;
    if (bvc_screen(wf[w], pxf, pyf, sapxf, sapyf, flo).la_lo > thr) mask &= ~((MaskT)1 << w);
  }
  bvc_walk<MaskT>(mask, px, py, ux, uy, walls, dist, wall_id);
}
// More than 64 walls: the same walls kept as bvc_first_wall_impl keeps -- those not rejected and not behind the final
// bound, which is the minimum over every wall -- from a first pass for the bound and a second that screens and walks
// blocks of 64 walls in increasing order.
RIAB_DEV void bvc_first_wall_many(double px, double py, double ux, double uy, const double* __restrict__ walls,
                                  const float4* __restrict__ wf, int W, float flo_env, double& dist, int& wall_id) {
  const float pxf = (float)px, pyf = (float)py, sapxf = -(float)uy, sapyf = (float)ux;
  const float flo = flo_env + flo_env * (fabsf(pxf) + fabsf(pyf));
  float thr = INFINITY;
  for (int w = 0; w < W; ++w) {
    const BvcScreen sc = bvc_screen(wf[w], pxf, pyf, sapxf, sapyf, flo);
    if (sc.lb_certain && sc.la_lo > 0.f) thr = fminf(thr, sc.la_hi);
  }
  double best = -1.0, best_la = 0.0;
  int besti = -1;
  for (int w0 = 0; w0 < W; w0 += 64) {
    unsigned long long mask = 0;
    const int n = (W - w0) < 64 ? (W - w0) : 64;
    for (int j = 0; j < n; ++j) {
      const BvcScreen sc = bvc_screen(wf[w0 + j], pxf, pyf, sapxf, sapyf, flo);
      if (!(sc.lb_rejected || (sc.la_hi < 0.f) || (sc.la_lo > thr))) mask |= 1ull << j;
    }
    bvc_walk_bits<unsigned long long>(mask, w0, px, py, ux, uy, walls, best, besti, best_la);
  }
  bvc_walk_end(px, py, ux, uy, walls, besti, best_la, dist, wall_id);
}
// flo_env = 1e-6 * max(1, largest |coordinate| of a wall end) * (longest wall), see bvc_screen
RIAB_DEV void bvc_first_wall(double px, double py, double ux, double uy, const double* __restrict__ walls,
                             const float4* __restrict__ wf, int W, float flo_env, double& dist, int& wall_id) {
  if (W <= 32) bvc_first_wall_impl<uint32_t>(px, py, ux, uy, walls, wf, W, flo_env, dist, wall_id);   // warp-uniform
  else if (W <= 64) bvc_first_wall_impl<unsigned long long>(px, py, ux, uy, walls, wf, W, flo_env, dist, wall_id);
  else bvc_first_wall_many(px, py, ux, uy, walls, wf, W, flo_env, dist, wall_id);
}

// Table screen (at most BVC_NW walls).  A thread keeps ONE agent for all its test angles, so everything that depends on
// (angle, wall) only -- 1 / den, the wall-start term of l_b, the error bounds -- comes from a per-CTA table in shared
// memory built in float64 (bvc_table_entry), and everything that depends on (agent, wall) only -- the numerator of l_a,
// from the float64 position -- sits in registers (numA).  Per (ray, wall):
//   l_a = numA_w * inv,   l_b = Ab - (p x u) * inv      (den = u x sb,  Ab = (a x u) / den,  x = 2D cross product)
// ~12 instructions, then one compare against the bound (min over certainly-scoring walls of l_a + err).
constexpr int BVC_NW = 16;
struct BvcTab { float inv, Ab, kb; };        // kb = margin on l_b;  the floor of l_a's error is BVC_KA_REL * |inv|
RIAB_DEV BvcTab bvc_table_entry(double ux, double uy, const double* __restrict__ wall, float cmax) {
  const double ax = wall[0], ay = wall[1], sbx = wall[2] - ax, sby = wall[3] - ay;
  const double den = ux * sby - uy * sbx;
  const double inv = 1.0 / den;                          // parallel ray: inf -> NaN / inf below, the wall is kept
  BvcTab t;
  t.inv = (float)inv;
  t.Ab = (float)((ax * uy - ay * ux) * inv);
  // float32 rounding of the position and the directions moves (p x u) by < 3e-7 |p|; |p| <= cmax inside the environment
  t.kb = fmaf(4e-6f * cmax, fabsf(t.inv), 1e-3f);
  return t;
}
template <int NW>
RIAB_DEV uint32_t bvc_table_mask(const BvcTab* __restrict__ row, const float (&numA)[NW], int W, float pcr, float ka) {
  float thr = INFINITY, la_lo[NW];
  uint32_t mask = 0;
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    la_lo[w] = INFINITY;
    if (w < W) {
      const BvcTab t = row[w];
      const float la = numA[w] * t.inv, lb = fmaf(-pcr, t.inv, t.Ab);
      const float err = fmaf(1e-5f, fabsf(la), ka * fabsf(t.inv));
      const float off = fabsf(lb - 0.5f) - 0.5f;                       // > 0 outside [0, 1]
      la_lo[w] = la - err;
      if (!((off > t.kb) || (la + err < 0.f))) mask |= 1u << w;        // NaN: kept
      if (off < -t.kb && la_lo[w] > 0.f) thr = fminf(thr, la + err);   // this wall certainly scores 1 / l_a > 0
    }
  }
#pragma unroll
  for (int w = 0; w < NW; ++w)
    if (la_lo[w] > thr) mask &= ~(1u << w);                            // certainly behind a wall that certainly scores
  return mask;
}

struct BvcConst {
  int n_cells, n_pad, T, ego;
  const double* head_dir;    // device (n_rows,2) or NULL (egocentric only)
  float min_fr, span;
  const float* packed;
  const double* test_dirs;   // device (T,2)
};

}  // namespace riab

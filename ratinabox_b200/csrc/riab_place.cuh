// PlaceCells.get_state (ratinabox/Neurons.py:936-981) over an (agents x cells)
// tile, float32, with Environment.get_distances_between___accounting_for_environment
// (ratinabox/Environment.py:677-779) for euclidean / line_of_sight / geodesic.
//
// Layout of the packed per-population block (float32, written by riab_place_pack):
//   cx[Np] | cy[Np] | k[Np] | a[Np] | per inner wall j: fc_j[Np], tc_j[Np] | ce0[Np] | ce1[Np] | cxl[Np] | cyl[Np]
//   cxl, cyl = the float32 residuals (c - box centre) - cx etc., read by the compensated direct form (COMP).
//   a = -k |c|^2 (expanded Gaussian form, see place_rates4), only when all widths are equal.
//   Np = n_cells rounded up to a multiple of 4 (padding cells sit far away, k = 0).
//   Coordinates are relative to the box centre (halves the float32 rounding error).
//   fc_j = signed distance of the centre to wall j's line, tc_j = its parameter
//   along the wall; ce_k = distance centre -> wall end k (geodesic only).
//
// Line-of-sight predicate.  The reference tests segment(centre->pos) against
// each inner wall with utils.vector_intercepts (utils.py:30-118): blocked iff
// 0<l_a<1 and 0<l_b<1.  With f = signed distance to the wall's line and t = the
// parameter along the wall, l_a = f_c/(f_c-f_p) and l_b = (f_c t_p - f_p t_c)/(f_c-f_p),
// so per (agent, cell, wall) the float32 fast path is three scalar FMA-pipe operations on
// per-cell registers and per-agent shared-memory broadcasts and a three-way min; the
// select is arithmetic (the penalty enters the exponent).  Results within an absolute
// band of 0 are re-evaluated in float64 with the reference's exact expression
// (los_blocked_exact), so the decision equals the oracle's.
#pragma once
#include "riab_common.cuh"

namespace riab {

constexpr int PLACE_MAX_WI = 8;      // inner walls held in registers
// Agent record (floats): [px, py, ep0, ep1] [-s t_p/|f_p|, -s (1-t_p)/|f_p|, -f_p * 2^20, band/|f_p|] x PLACE_MAX_WI [float64 px, py]
// with s = sign(f_p): multiplied by the cell's SIGNED f_c these give |f_c| t_p/|f_p| etc. exactly when centre and agent
// lie on opposite sides of the wall's line (the only case in which X and Y matter), with no |.| on the cell side.
constexpr int PLACE_WALL0 = 4;                               // float index of wall 0's float4
// record of a policy with WI inner-wall slots: [px, py, ep0, ep1] [wall float4] x WI [float64 px, py] and, for geodesic
// kernels (GEO), [|e0 - p|, |e1 - p|, 0, 0]: the agent -> wall-end distances of the detour, so that ep0 / ep1 stay free
// for the compensated direct form
constexpr int place_pos64(int wi) { return PLACE_WALL0 + 4 * wi; }   // float index of the float64 position
constexpr int place_geo(int wi) { return place_pos64(wi) + 4; }      // float index of the wall-end distances (GEO)
constexpr int place_rec(int wi, bool geo = false) { return place_pos64(wi) + (geo ? 8 : 4); }   // 16 floats with two walls
constexpr float PLACE_PEN = 1.2676506002282294e30f;          // 2^100: pen * PLACE_PEN is >= 1e24 for every certain blocked pair
constexpr float PLACE_QSCALE = 1048576.0f;                   // 2^20: q' = f_c * (-f_p * 2^20) never enters the band by magnitude

RIAB_HD void wall_coords(double qx, double qy, double ax, double ay, double bx, double by, double& f, double& t) {
  const double sx = bx - ax, sy = by - ay;
  const double n2 = sx * sx + sy * sy;
  f = (sx * (qy - ay) - sy * (qx - ax)) / sqrt(n2);
  t = ((qx - ax) * sx + (qy - ay) * sy) / n2;
}

// The reference's exact float64 test for one (centre, pos, wall) triple:
// a-list = segment centre->pos, b-list = wall  (Environment.py:718-721, utils.py:74-106)
RIAB_DEV bool los_blocked_exact(double cx, double cy, double px, double py, double w0, double w1, double w2, double w3) {
  const D ax(cx), ay(cy), bx(px), by(py);
  const D wx0(w0), wy0(w1), wx1(w2), wy1(w3);
  const D d0x = wx0 - ax, d0y = wy0 - ay;
  const D sax = bx - ax, say = by - ay;
  const D sbx = wx1 - wx0, sby = wy1 - wy0;
  const D sapx = -say, sapy = sax, sbpx = -sby, sbpy = sbx;
  const D la = (d0x * sbpx + d0y * sbpy) / (sax * sbpx + say * sbpy);
  const D lb = ((-d0x) * sapx + (-d0y) * sapy) / (sbx * sapx + sby * sapy);
  return (la.v > 0.0) && (la.v < 1.0) && (lb.v > 0.0) && (lb.v < 1.0);
}
RIAB_DEV bool los_blocked_exact(double cx, double cy, double px, double py, const double* __restrict__ w) {
  return los_blocked_exact(cx, cy, px, py, w[0], w[1], w[2], w[3]);
}

// The reference's float64 geodesic detour centre -> wall end -> pos, the minimum over the ends inside the box
// (ep_valid bit e: end e at (w[2e], w[2e+1])), Environment.py:745-773; INFINITY when no end is inside.
RIAB_DEV double geodesic_detour_exact(double cx, double cy, double px, double py, double w0, double w1, double w2,
                                      double w3, int ep_valid) {
  double via = INFINITY;
  for (int e = 0; e < 2; ++e) {
    if (!((ep_valid >> e) & 1)) continue;
    const D wx(e ? w2 : w0), wy(e ? w3 : w1);
    const D ax = D(cx) - wx, ay = D(cy) - wy, bx = wx - D(px), by = wy - D(py);
    via = fmin(via, (dsqrt(ax * ax + ay * ay) + dsqrt(bx * bx + by * by)).v);
  }
  return via;
}

// Per-agent record for the rate phase, from the float64 position.
// inner = walls + 4*n_boundary (float64 endpoints), cxm/cym = box centre.
// Per-CTA wall invariants of the agent records (shared memory, 2 doubles per inner wall): 1 / |s| and 1 / |s|^2, so that a
// record costs one float64 division per wall (1 / |f_p|) instead of a square root and five divisions -- the records are
// built by the float64 producer warps, whose chain bounds the step once the consumers are fast.
RIAB_DEV void place_wall_invariants(double* __restrict__ aux, const double* __restrict__ inner, int n_inner) {
  for (int j = threadIdx.x; j < n_inner && j < PLACE_MAX_WI; j += blockDim.x) {
    const double sx = inner[4 * j + 2] - inner[4 * j], sy = inner[4 * j + 3] - inner[4 * j + 1];
    const double n2 = sx * sx + sy * sy;
    aux[2 * j] = 1.0 / sqrt(n2);
    aux[2 * j + 1] = 1.0 / n2;
  }
}

// COMP: the compensated direct form -- ep0 / ep1 carry the float32 residuals of the centred position (unused slots there:
// the expanded form does not take COMP).  GEO: the geodesic kernels' wall-end distances at place_geo(WI).
template <int WI, bool COMP = false, bool GEO = false>
RIAB_DEV void place_agent_record(float* __restrict__ rec, double px, double py, const double* __restrict__ inner,
                                 const double* __restrict__ aux,
                                 int n_inner, double cxm, double cym, float band, int expanded, float kx,
                                 float lfold /* log2(span) when the scale is folded into the exponent, else 0 */) {
  float ep0 = 0.f, ep1 = 0.f;
  if (GEO) {
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n_inner >= 1) {
      // utils.get_distances_between(wall_edge, pos2)  (Environment.py:749-751)
      const double e0x = inner[0] - px, e0y = inner[1] - py, e1x = inner[2] - px, e1y = inner[3] - py;
      g.x = (float)sqrt(e0x * e0x + e0y * e0y);
      g.y = (float)sqrt(e1x * e1x + e1y * e1y);
    }
    *reinterpret_cast<float4*>(rec + place_geo(WI)) = g;
  }
  const float pxf = (float)(px - cxm), pyf = (float)(py - cym);
  if (expanded) ep0 = (float)((double)kx * ((double)pxf * pxf + (double)pyf * pyf) + (double)lfold);   // -k |p|^2 [+ log2 span]
  if (COMP) { ep0 = (float)((px - cxm) - (double)pxf); ep1 = (float)((py - cym) - (double)pyf); }
  *reinterpret_cast<float4*>(rec) = make_float4(pxf, pyf, ep0, ep1);
  for (int j = 0; j < WI; ++j) {
    float4 w = make_float4(-1.f, 2.f, -PLACE_QSCALE, 1.0e-6f);    // dummy wall: same side (q' < 0), X = -2, Y = 4
    if (j < n_inner) {
      // wall_coords with the wall's invariants (float32 screen quantities: the last float64 ulp is irrelevant)
      const double ax = inner[4 * j], ay = inner[4 * j + 1], sx = inner[4 * j + 2] - ax, sy = inner[4 * j + 3] - ay;
      const double qx = px - ax, qy = py - ay;
      const double f = (sx * qy - sy * qx) * aux[2 * j], t = (qx * sx + qy * sy) * aux[2 * j + 1];
      const double b = fabs(f);
      if (!(b >= 1e-9)) w = make_float4(0.f, 0.f, 0.f, 3.0e38f);  // agent on the wall's line (or a degenerate wall): exact path
      else {
        const double rb = ((f > 0.0) ? -1.0 : 1.0) / b;            // -sign(f_p) / |f_p|
        w = make_float4((float)(t * rb), (float)((1.0 - t) * rb), (float)(-f) * PLACE_QSCALE, (float)((double)band / b));
      }
    }
    *reinterpret_cast<float4*>(rec + PLACE_WALL0 + 4 * j) = w;
  }
  *reinterpret_cast<double2*>(rec + place_pos64(WI)) = make_double2(px, py);  // exact fall-back only
}

struct PlaceConst {                  // uniform per launch
  int desc, geometry, n_cells, n_pad, n_inner, ep_valid;
  int wall0;                         // index of the first wall the line-of-sight / geodesic tests use (Environment.py:715-717: 4)
  float min_fr, span, top_hat_w2;
  double top_hat_w;
  float eps[PLACE_MAX_WI];
  float band;                        // max of eps[]: one absolute band for all walls
  int expanded;                      // Gaussian with one common width: -k d^2 = a_c + (2k c).p - k|p|^2 (3 FMA-pipe ops)
  float kx;                          // -k = -log2(e)/(2 w^2) of that common width
  int fold;                          // expanded and min_fr == 0: log2(max_fr) is added to the agent's -k|p|^2 term, no final FFMA
  float lspan;                       // log2(max_fr - min_fr)
  const float* packed;               // device
  const double* centres64;           // device (N,2)
  int periodic;                      // wrap centre->agent vectors (Environment.py:670-675)
  int comp;                          // direct form: the host launches the COMP kernels (make_place)
  float scale_f, half_f;
  double scale;
  double cxm, cym;
  float coord_err;                   // float32 error of |c' - p'| from the centres' side (make_place)
  float top_hat_band;                // |d^2 - w^2| below which top_hat decides in float64 (make_place)
  float scale_lo;                    // scale - (float)scale: the compensated periodic wrap
};

// Per-thread cell registers: 4 consecutive cells.
template <int WI>
struct PlaceCellRegs {
  float cx[4], cy[4], k[4];
  float fc[WI > 0 ? WI : 1][4], tc[WI > 0 ? WI : 1][4], tq[WI > 0 ? WI : 1][4];   // tq = 1 - tc
  float ce0[4], ce1[4];
  float cxl[4], cyl[4];              // COMP only: residuals of the centred centres
};

template <int WI, bool COMP = false, bool GEO = false>
RIAB_DEV void place_load_cells(PlaceCellRegs<WI>& r, const PlaceConst& c, int cell0) {
  const float* base = c.packed;
  const int np = c.n_pad;
  ldv(r.cx, base + cell0);
  ldv(r.cy, base + np + cell0);
  ldv(r.k, base + 2 * np + cell0);
  if (c.expanded) {                                      // registers hold (2k cx, 2k cy, -k|c|^2) instead of (cx, cy, k)
    const float k2 = -2.f * c.kx;
#pragma unroll
    for (int i = 0; i < 4; ++i) { r.cx[i] *= k2; r.cy[i] *= k2; }
    ldv(r.k, base + 3 * np + cell0);
  }
#pragma unroll
  for (int j = 0; j < WI; ++j) {
    if (j < c.n_inner) {
      ldv(r.fc[j], base + (4 + 2 * j) * np + cell0);
      ldv(r.tc[j], base + (5 + 2 * j) * np + cell0);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) { r.fc[j][i] = 1.f; r.tc[j][i] = -1.f; }   // dummy wall (see place_agent_record)
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) r.tq[j][i] = 1.f - r.tc[j][i];
  }
  if (GEO) {
    ldv(r.ce0, base + (4 + 2 * c.n_inner) * np + cell0);
    ldv(r.ce1, base + (5 + 2 * c.n_inner) * np + cell0);
  }
  if (COMP) {
    ldv(r.cxl, base + (6 + 2 * c.n_inner) * np + cell0);
    ldv(r.cyl, base + (7 + 2 * c.n_inner) * np + cell0);
  }
}

// Neurons.py:959-976 epilogue on the squared distance (float32).  DESC is a
// compile-time description, or -1 for a run-time switch on c.desc.
template <int DESC>
RIAB_DEV float place_profile(float d2, float k, int desc_rt) {
  const int desc = (DESC >= 0) ? DESC : desc_rt;
  const float g = ex2f(-d2 * k);
  if (desc == RIAB_PC_GAUSSIAN) return g;
  if (desc == RIAB_PC_GAUSSIAN_THRESHOLD)
    return fmaxf(g - 0.60653065971263342f, 0.f) * 2.5414940825367984f;   // exp(-1/2), 1/(1-exp(-1/2))
  // diff_of_gaussians, ratio = 1.5: (g - g2/ratio^2) * ratio^2/(ratio^2-1)
  const float g2 = ex2f(-d2 * k * (1.0f / 2.25f));
  return (g - (1.0f / 2.25f) * g2) * 1.8f;
}

// Exact (float64) line-of-sight flags for this thread's 4 cells: the rare path taken when
// any float32 predicate of the group fell inside its uncertainty band.  Arguments are scalars and
// shared-memory offsets (no generic pointers to materialise in the hot loop).
RIAB_DEV double lds_f64(uint32_t saddr) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(saddr));
  return v;
}
template <int WI>
__device__ __noinline__ unsigned place_blocked_exact4(const double* __restrict__ centres64, int n_cells, int n_inner,
                                                      int cell0, uint32_t rec_s, uint32_t inner_s) {
  const double px = lds_f64(rec_s + 4u * place_pos64(WI)), py = lds_f64(rec_s + 4u * place_pos64(WI) + 8u);
  unsigned m = 0;
  for (int i = 0; i < 4; ++i) {
    const int cell = cell0 + i;
    if (cell >= n_cells) continue;
    const double cx = centres64[2 * cell], cy = centres64[2 * cell + 1];
    bool b = false;
    for (int j = 0; j < WI && j < n_inner; ++j) {
      const uint32_t w = inner_s + 32u * (uint32_t)j;
      b = b || los_blocked_exact(cx, cy, px, py, lds_f64(w), lds_f64(w + 8u), lds_f64(w + 16u), lds_f64(w + 24u));
    }
    m |= b ? (1u << i) : 0u;
  }
  return m;
}

// |p' - c'| along one axis in the periodic box, compensated: s + e = (p - c) exactly up to the residuals' rounding, with
// e the two-difference residual of s = p_hi - c_hi plus lo = p_lo - c_lo; the wrapped (scale - |p - c|) is formed as
// (scale_f - |s|) + (scale_lo - sign(s) e), whose first term is exact near the wrap (Sterbenz).
RIAB_DEV float periodic_comp(float p, float cc, float lo, const PlaceConst& c) {
  const float s = p - cc, b = s - p;
  const float e = ((p - (s - b)) - (cc + b)) + lo;
  const float d = fabsf(s + e);
  return (d > c.half_f) ? (c.scale_f - fabsf(s)) + (c.scale_lo - (s < 0.f ? -e : e)) : d;
}

// Rates of one agent for this thread's 4 cells (branch-free fast path).
//   rec     : the agent's record in shared memory (broadcast reads); holds the float64 position too
//   inner_s : shared-memory offset of the float64 inner walls (exact fall-back only)
//   unsure  : DEFER = true only ORs the band test into it -- the caller redoes the agents it covers
//             later with DEFER = false, which tests per agent and takes the exact float64 path at once.
//   EXP     : 1 = the expanded Gaussian form is known to be on (no branch), 0 = known off, -1 = test c.expanded
//   COMP    : direct form with the float32 residuals of p' (record ep0 / ep1) and c' (cxl / cyl):
//             dx = (px - cx) + (pxl - cxl), so |p'| and |c'| no longer limit the accuracy of d (PlaceConst::comp)
//   GEO     : geodesic detours for blocked pairs (one inner wall, DESC = -1, the record's place_geo block)
template <int WI, int DESC, bool DEFER, int EXP = -1, bool COMP = false, bool GEO = false>
RIAB_DEV void place_rates4(float (&out)[4], const PlaceCellRegs<WI>& r, const PlaceConst& c, int cell0,
                           const float* __restrict__ rec, uint32_t inner_s, bool& unsure_io) {
  const float4 r0 = *reinterpret_cast<const float4*>(rec);          // px, py, ep0 | -k|p|^2, ep1
  // ---- line of sight: pen[i] = 1 if the segment centre_i -> agent crosses an inner wall, else 0
  float pen[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) pen[i] = 0.f;
  if (WI > 0) {
    // With a = |f_c|, b = |f_p| and q' = -f_c f_p 2^20 (> 0 iff the agent is on the other side of the wall's line):
    //   |D| = a + b,  M' = b t_c + a t_p  (a convex combination of t_p, t_c scaled by |D|),
    //   blocked  <=>  q' > 0 and 0 < M' < |D|.
    // Everything is divided by b on the agent side and carries -sign(f_p) (record: -s t_p/b, -s (1-t_p)/b, band/b), so
    //   X = M'/b = fma(f_c, -s t_p/b, t_c),  Y = (|D|-M')/b = fma(f_c, -s (1-t_p)/b, 1-t_c),  q' = f_c (-f_p 2^20)
    // hold whenever q' > 0 (f_c * -s = a then); on the same side q' < 0 decides alone.  m3 = min(X, Y, q'):
    // per cell 2 FFMA + 1 FMUL (agent values from the record) + 2 FMNMX;
    // blocked <=> m3 > 0.
    // |m3| below band/b => the sign of m3 is not certain in float32: re-evaluate in float64.
    // The select is arithmetic: pen = max(0, max_j m3_j) (NaN -> 0) enters the exponent /
    // the squared distance multiplied by 2^100: any pen above the band (>= ~1e-6 / b) makes the rate exactly 0.
    float worst[4], m3_prev[4];                           // worst = max(0, max over walls of m3)
#pragma unroll
    for (int i = 0; i < 4; ++i) { worst[i] = 0.f; m3_prev[i] = 0.f; }
    bool unsure = DEFER ? unsure_io : false;
#pragma unroll
    for (int j = 0; j < WI; ++j) {
      const float4 pw = *reinterpret_cast<const float4*>(rec + PLACE_WALL0 + 4 * j);
      float m3[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float fc = r.fc[j][i];
        const float X = fmaf(fc, pw.x, r.tc[j][i]);
        const float Y = fmaf(fc, pw.y, r.tq[j][i]);
        m3[i] = fminf(fminf(X, Y), fc * pw.z);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if ((j & 1) == 1) worst[i] = fmaxf(fmaxf(worst[i], m3[i]), m3_prev[i]);   // pairs of walls
        else if (j == WI - 1) worst[i] = fmaxf(worst[i], m3[i]);                                    // odd wall count: the last one
        m3_prev[i] = m3[i];
      }
      const float am = fminf(fminf(fminf(fabsf(m3[0]), fabsf(m3[1])), fabsf(m3[2])), fabsf(m3[3]));
      unsure = unsure || (am < pw.w);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) pen[i] = worst[i];
    if (DEFER) unsure_io = unsure;
    else if (unsure) {                                   // rare: redo the group's flags with the reference's float64 test
      const unsigned m = place_blocked_exact4<WI>(c.centres64, c.n_cells, c.n_inner, cell0,
                                                  (uint32_t)__cvta_generic_to_shared(rec), inner_s);
#pragma unroll
      for (int i = 0; i < 4; ++i) pen[i] = ((m >> i) & 1u) ? 1.f : 0.f;
    }
  }
  // ---- Gaussian with one common width, expanded:  -k|c-p|^2 = (-k|c|^2 - k|p|^2) + (2k cx) px + (2k cy) py.
  // 1 FADD + 2 FFMA per rate on per-cell registers (2k cx, 2k cy, -k|c|^2); only used when k * r2_max <= 10,
  // where the cancellation costs < 4e-6 relative (make_place).  Blocked pairs: exponent - 1e5 -> rate 0 (d = 1000).
  if (!COMP && DESC == RIAB_PC_GAUSSIAN && (EXP >= 1 || (EXP < 0 && c.expanded))) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {                         // cell pairs: FADD + 2 (3) FFMA per rate
      float t0 = fmaf(r.cy[2 * h], r0.y, fmaf(r.cx[2 * h], r0.x, r.k[2 * h] + r0.z));
      float t1 = fmaf(r.cy[2 * h + 1], r0.y, fmaf(r.cx[2 * h + 1], r0.x, r.k[2 * h + 1] + r0.z));
      if (WI > 0) { t0 = fmaf(pen[2 * h], -PLACE_PEN, t0); t1 = fmaf(pen[2 * h + 1], -PLACE_PEN, t1); }
      // Neurons.py:978-980; EXP == 2: min_fr == 0 and log2(span) already sits in the agent's -k|p|^2 term
      if (EXP == 2 || (EXP < 0 && c.fold)) { out[2 * h] = ex2f(t0); out[2 * h + 1] = ex2f(t1); }
      else { out[2 * h] = fmaf(ex2f(t0), c.span, c.min_fr); out[2 * h + 1] = fmaf(ex2f(t1), c.span, c.min_fr); }
    }
    return;
  }
  float d2[4];
  if (WI == 0 && c.periodic) {                           // warp-uniform
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float dx, dy;
      if (COMP) {
        // the wrapped distance scale - |dx| is small where |dx| is large: the rounding of px - cx itself counts there, so
        // it is kept as the exact residual of the difference (two-difference), and scale's own float32 residual added
        dx = periodic_comp(r0.x, r.cx[i], r0.z - r.cxl[i], c);
        dy = periodic_comp(r0.y, r.cy[i], r0.w - r.cyl[i], c);
      } else {
        dx = fabsf(r0.x - r.cx[i]); dy = fabsf(r0.y - r.cy[i]);
        dx = (dx > c.half_f) ? c.scale_f - dx : dx;      // the short way round
        dy = (dy > c.half_f) ? c.scale_f - dy : dy;
      }
      d2[i] = fmaf(dy, dy, dx * dx);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float dx = COMP ? (r0.x - r.cx[i]) + (r0.z - r.cxl[i]) : r0.x - r.cx[i];
      const float dy = COMP ? (r0.y - r.cy[i]) + (r0.w - r.cyl[i]) : r0.y - r.cy[i];
      d2[i] = fmaf(dy, dy, dx * dx);
    }
  }
  // final squared distances (blocked pairs get a distance >= 1000, Environment.py:730)
  float dd[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) dd[i] = (WI > 0) ? fmaf(pen[i], PLACE_PEN, d2[i]) : d2[i];
  constexpr bool geodesic = GEO && (DESC < 0) && (WI > 0);
  const int desc = (DESC >= 0) ? DESC : c.desc;
  if (desc != RIAB_PC_TOP_HAT && !geodesic) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      out[i] = fmaf(place_profile<DESC>(dd[i], r.k[i], c.desc), c.span, c.min_fr);   // Neurons.py:978-980
    return;
  }
  const float4 ep = geodesic ? *reinterpret_cast<const float4*>(rec + place_geo(WI)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool blocked = (WI > 0) && (dd[i] != d2[i]);
    float dv = dd[i];
    if (geodesic && blocked) {
      // Environment.py:745-773: min over the wall ends that lie inside the box
      float via = INFINITY;
      if (c.ep_valid & 1) via = r.ce0[i] + ep.x;
      if (c.ep_valid & 2) via = fminf(via, r.ce1[i] + ep.y);
      dv = via * via;
    }
    float v;
    if (desc == RIAB_PC_TOP_HAT) {
      // Neurons.py:975-976: 1*(dist < widths) with the scalar `widths`.  A line-of-sight blocked pair has dv >= 1e24;
      // a geodesic detour's dv = (ce + ep)^2 carries three float32 roundings of the sum and one of the square, under
      // 5e-7 relative, well inside top_hat_band (>= 4e-6 w^2): both forms take the float64 decision near the edge.
      bool in = dv < c.top_hat_w2;
      if (fabsf(dv - c.top_hat_w2) < c.top_hat_band && (geodesic || !blocked)) {
        const int cell = cell0 + i;
        if (cell < c.n_cells) {
          const double2 p64 = *reinterpret_cast<const double2*>(rec + place_pos64(WI));
          const double cx = c.centres64[2 * cell], cy = c.centres64[2 * cell + 1];
          if (geodesic && blocked) {
            in = geodesic_detour_exact(cx, cy, p64.x, p64.y, lds_f64(inner_s), lds_f64(inner_s + 8u),
                                       lds_f64(inner_s + 16u), lds_f64(inner_s + 24u), c.ep_valid) < c.top_hat_w;
          } else {
            D ex = D(cx) - D(p64.x), ey = D(cy) - D(p64.y);
            if (c.periodic) {
              if (fabs(ex.v) > c.scale / 2) ex = D(-copysign(1.0, ex.v)) * (D(c.scale) - D(fabs(ex.v)));
              if (fabs(ey.v) > c.scale / 2) ey = D(-copysign(1.0, ey.v)) * (D(c.scale) - D(fabs(ey.v)));
            }
            in = dsqrt(ex * ex + ey * ey).v < c.top_hat_w;
          }
        }
      }
      v = in ? 1.f : 0.f;
    } else {
      v = place_profile<DESC>(dv, r.k[i], c.desc);
    }
    out[i] = fmaf(v, c.span, c.min_fr);
  }
}

}  // namespace riab

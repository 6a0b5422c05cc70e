// AgentVectorCells.get_state (ratinabox/Neurons.py:2204-2320), float32 rates from float64 agent-partner geometry.
//
//   fr_i = gaussian(d; mu_d_i, sigma_d_i, norm=1) * von_mises(bearing; mu_theta_i, sigma_theta_i, norm=1)
//          * (max_fr - min_fr) + min_fr
//   d       = |pos - partner|, or 1000 when walls_occlude and an inner wall crosses the segment (line_of_sight,
//             Environment.py:710-730)
//   bearing = utils.get_angle(partner - pos) [- utils.get_angle(head_direction) when egocentric]
//
// ObjectVectorCells (riab_ovc.cuh) with one "object", the partner, and no type mask.  The producer reads the partner of
// its row -- row i of the partner Agent, row 0 when the partner has one agent, or the row's own position when the Agent
// is its own partner -- evaluates the geometry in float64 like the reference (np.linalg.norm, the exact
// utils.vector_intercepts test, utils.get_angle with its 1e-6 eps) and publishes
//   (d, cos(b/2), sin(b/2), 0).
// Consumers hold per cell (mu_d, s_d, cos(mu/2), sin(mu/2), k_q) and evaluate, like riab_ovc.cuh,
//   u = (d - mu_d) s_d,  g = (sin(b/2) cos(mu/2) - cos(b/2) sin(mu/2)) k_q,  fr = fma(2^-(u^2 + g^2), max_fr - min_fr, min_fr).
// No partner (tuning_type_agent is None): min_fr = span = 0, so every rate is exactly 0 (Neurons.py:2231-2232).  A NaN
// partner position gives NaN rates, as in the reference (only the own position is masked, Neurons.py:163-164).
#pragma once
#include "riab_common.cuh"
#include "riab_motion.cuh"
#include "riab_place.cuh"

namespace riab {

constexpr int AVC_REC = 4;                        // d, cos(b/2), sin(b/2), unused

struct AvcConst {                                 // uniform per launch
  int n_cells, n_pad, ego, occlude, self, wall0, n_inner;
  float min_fr, span;
  const float* packed;                            // mu_d | s_d | cos(mu/2) | sin(mu/2) | k_q   (Np each)
  const double* other;                            // the partner's positions, NULL: none (or self)
  long long other_ld;                             // 2: row i reads partner row i, 0: every row reads row 0
  const double* head_dir;                         // positions-only launches: (n_pos,2) head directions or NULL = [1,0]
};

struct AvcCellRegs {
  float mu[4], sd[4], cm[4], sm[4], kq[4];
};

RIAB_DEV void avc_load_cells(AvcCellRegs& r, const AvcConst& c, int cell0) {
  const int np = c.n_pad;
  const float* b = c.packed + cell0;
  const float4 a0 = *reinterpret_cast<const float4*>(b), a1 = *reinterpret_cast<const float4*>(b + np),
               a2 = *reinterpret_cast<const float4*>(b + 2 * np), a3 = *reinterpret_cast<const float4*>(b + 3 * np),
               a4 = *reinterpret_cast<const float4*>(b + 4 * np);
  r.mu[0] = a0.x; r.mu[1] = a0.y; r.mu[2] = a0.z; r.mu[3] = a0.w;
  r.sd[0] = a1.x; r.sd[1] = a1.y; r.sd[2] = a1.z; r.sd[3] = a1.w;
  r.cm[0] = a2.x; r.cm[1] = a2.y; r.cm[2] = a2.z; r.cm[3] = a2.w;
  r.sm[0] = a3.x; r.sm[1] = a3.y; r.sm[2] = a3.z; r.sm[3] = a3.w;
  r.kq[0] = a4.x; r.kq[1] = a4.y; r.kq[2] = a4.z; r.kq[3] = a4.w;
}

// Record of row i from its float64 position / head direction.  walls = all walls (W*4 doubles).
RIAB_DEV void avc_agent_record(float* __restrict__ rec, double px, double py, double hdx, double hdy, long long i,
                               const double* __restrict__ walls, const AvcConst& c) {
  double ox = px, oy = py;                                                    // the Agent as its own partner
  if (!c.self) {
    if (c.other == nullptr) {                                                 // no partner: the packed span is 0
      *reinterpret_cast<float4*>(rec) = make_float4(1000.f, 1.f, 0.f, 0.f);
      return;
    }
    ox = c.other[c.other_ld * i];
    oy = c.other[c.other_ld * i + 1];
  }
  const double hb = c.ego ? get_angle(hdx, hdy) : 0.0;                       // Neurons.py:2277-2278
  const D vx = D(px) - D(ox), vy = D(py) - D(oy);                             // pos1 - pos2 (utils.py:213)
  double d = dsqrt(vx * vx + vy * vy).v;                                      // np.linalg.norm
  if (c.occlude) {
    const double* inner = walls + 4 * c.wall0;                                // walls[4:] (Environment.py:715-717)
    bool blocked = false;
    for (int j = 0; j < c.n_inner; ++j) blocked = blocked || los_blocked_exact(px, py, ox, oy, inner + 4 * j);
    if (blocked) d = 1000.0;                                                  // Environment.py:730
  }
  const double b = get_angle(-vx.v, -vy.v) - hb;                              // bearing of partner - pos (Neurons.py:2253-2279)
  double sh, ch;
  sincos(0.5 * b, &sh, &ch);
  *reinterpret_cast<float4*>(rec) = make_float4((float)d, (float)ch, (float)sh, 0.f);
}

RIAB_DEV void avc_rates4(float (&out)[4], const AvcCellRegs& r, const AvcConst& c, const float* __restrict__ rec) {
  const float4 q = *reinterpret_cast<const float4*>(rec);                     // d, cos(b/2), sin(b/2)
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float u = (q.x - r.mu[i]) * r.sd[i];
    const float g = fmaf(q.z, r.cm[i], -q.y * r.sm[i]) * r.kq[i];
    out[i] = fmaf(ex2f(fmaf(-g, g, -u * u)), c.span, c.min_fr);              // Neurons.py:2306-2319
  }
}

}  // namespace riab

// HeadDirectionCells / VelocityCells / SpeedCell.get_state (ratinabox/Neurons.py:2421-2485, :2577-2583, :2632-2651),
// float32 rates from the agent's float64 kinematic state.
//
//   HeadDirectionCells  fr_i = von_mises(get_angle(d), mu_i, sigma_i, norm=1) (max_fr - min_fr) + min_fr
//                       d = head direction, or velocity / |velocity| with use_velocity
//   VelocityCells       the use_velocity HeadDirectionCells rates times |Agent.velocity| / one_sigma_speed
//   SpeedCell           fr = |v| / one_sigma_speed (max_fr - min_fr) + min_fr,   v = the measured velocity
//
// The producer evaluates the angle like the reference, in float64 (utils.get_angle with its 1e-6 eps, after the
// velocity's normalisation), and publishes per agent
//   (cos(theta/2), sin(theta/2), a, b)     a = 1, b = scale (head direction, velocity);  a = scale, b = 1 (speed)
// with scale = |v| inv_one_sigma_speed (velocity, speed) or 1.  Consumers hold per cell (cos(mu/2), sin(mu/2), k_q) and
// evaluate
//   h = sin((theta - mu)/2) = sin(theta/2) cos(mu/2) - cos(theta/2) sin(mu/2),  g = h k_q,  k_q^2 = 2 kappa log2(e)
//   fr = fma(2^-(g^2) a, max_fr - min_fr, min_fr) b
// (von Mises with norm=1 is exp(kappa (cos(theta-mu) - 1)) = exp(-2 kappa sin^2((theta-mu)/2)), the half-angle form of
// riab_ovc.cuh without cancellation for narrow tunings).  A speed cell packs k_q = 0: 2^0 a = scale, so its rate is
// fma(scale, max_fr - min_fr, min_fr) like Neurons.py:2646-2650.  A zero velocity gives NaN (0/0) as in the reference.
#pragma once
#include "riab_common.cuh"
#include "riab_motion.cuh"

namespace riab {

constexpr int KIN_REC = 4;                        // cos(theta/2), sin(theta/2), a, b

struct KinConst {                                 // uniform per launch
  int n_cells, n_pad, variant, use_vel;
  float min_fr, span;
  double inv_oss;                                 // 1 / one_sigma_speed
  double fixed_scale;                             // >= 0 or NaN: VelocityCells' speed factor of every row (get_state away
                                                  // from the agent); negative: |velocity| of the row's own vector
  const float* packed;                            // cos(mu/2) | sin(mu/2) | k_q   (Np each)
  const double* vec;                              // MODE 0: the row's vector (head direction / velocity / measured velocity)
  long long vec_ld;                               // 2: one vector per row, 0: one vector for every row
};

struct KinCellRegs {
  float cm[4], sm[4], kq[4];
};

RIAB_DEV void kin_load_cells(KinCellRegs& r, const KinConst& c, int cell0) {
  const int np = c.n_pad;
  const float* b = c.packed + cell0;
  const float4 a0 = *reinterpret_cast<const float4*>(b), a1 = *reinterpret_cast<const float4*>(b + np),
               a2 = *reinterpret_cast<const float4*>(b + 2 * np);
  r.cm[0] = a0.x; r.cm[1] = a0.y; r.cm[2] = a0.z; r.cm[3] = a0.w;
  r.sm[0] = a1.x; r.sm[1] = a1.y; r.sm[2] = a1.z; r.sm[3] = a1.w;
  r.kq[0] = a2.x; r.kq[1] = a2.y; r.kq[2] = a2.z; r.kq[3] = a2.w;
}

// Per-agent record.  (hdx, hdy): head direction; (vx, vy): velocity; (mvx, mvy): measured velocity (Agent.py:517, the
// history's "vel" that SpeedCell reads).
RIAB_DEV void kin_agent_record(float* __restrict__ rec, double hdx, double hdy, double vx, double vy, double mvx, double mvy,
                               const KinConst& c) {
  if (c.variant == RIAB_KIN_SPEED) {
    const D s = dsqrt(D(mvx) * D(mvx) + D(mvy) * D(mvy)) * D(c.inv_oss);       // np.linalg.norm(vel) / one_sigma_speed
    *reinterpret_cast<float4*>(rec) = make_float4(1.f, 0.f, (float)s.v, 1.f);
    return;
  }
  double dx = hdx, dy = hdy, scale = 1.0;
  if (c.use_vel) {
    const D nv = dsqrt(D(vx) * D(vx) + D(vy) * D(vy));                        // direction = vel / np.linalg.norm(vel)
    dx = (D(vx) / nv).v;
    dy = (D(vy) / nv).v;
    if (c.variant == RIAB_KIN_VELOCITY) scale = (c.fixed_scale < 0.0) ? (nv * D(c.inv_oss)).v : c.fixed_scale;
  }
  double sh, ch;
  sincos(0.5 * get_angle(dx, dy), &sh, &ch);                                  // Neurons.py:2467
  *reinterpret_cast<float4*>(rec) = make_float4((float)ch, (float)sh, 1.f, (float)scale);
}

RIAB_DEV void kin_rates4(float (&out)[4], const KinCellRegs& r, const KinConst& c, const float* __restrict__ rec) {
  const float4 q = *reinterpret_cast<const float4*>(rec);                     // cos(theta/2), sin(theta/2), a, b
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float g = fmaf(q.y, r.cm[i], -q.x * r.sm[i]) * r.kq[i];
    out[i] = fmaf(ex2f(-g * g) * q.z, c.span, c.min_fr) * q.w;
  }
}

}  // namespace riab

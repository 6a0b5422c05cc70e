// DumbAgent (contribs/SubAgent.py:118-179), ShiftAgent (:466-478) and ReplayAgent (:358-431) for ONE agent per thread,
// in float64 with the reference's operation order: the position the SubAgent moves to at this lead step.  The forced
// step of Agent.update that moves it there is the ordinary riab_agent_update_src launch that follows.
//
// ReplayAgent: the reference rolls its sham agent out eagerly, inside the update() that starts a replay, to
// 1.1 replay_speed replay_duration of distance, and interpolates in that rollout on the later steps.  Here the rollout
// advances lazily, only as far as each step's query, keeping the last two samples: the query never decreases within a
// replay and neither does the rollout's distance, so the pair interp1d would pick is the kept pair (as in
// riab_theta.cuh's look ahead).
#pragma once
#include "riab_theta.cuh"

namespace riab {

// utils.py:347-368 for one component with drift 0, the normal drawn with scale=dt: theta (0 - x) dt + sigma (dt n)
// (ou_dx), then the spring -acceleration_scale * displacement * dt (:160) and the two += of :161 and :163.
RIAB_DEV void dumb_spring(double& disp, double& dvel, D dt, D theta, D sigma, D a, D n) {
  const D ou = ou_dx(dt, D(dvel), D(0.0), theta, sigma, n);
  const D spring = (-a) * D(disp) * dt;
  dvel = (D(dvel) + (ou + spring)).v;
  disp = (D(disp) + D(dvel) * dt).v;
}

// :165-173: the displacement cut back to 0.95 of the nearest strict crossing of [lead, lead + disp] with any wall
// (utils.vector_intercepts, utils.py:30-118, with the two divisions NumPy makes: the VALUE of l_b is used).
RIAB_DEV void dumb_wall_cut(double lx, double ly, double& dx, double& dy, const double* __restrict__ walls, int W) {
  const D b0x(lx), b0y(ly);
  const D b1x = b0x + D(dx), b1y = b0y + D(dy);
  const D sbx = b1x - b0x, sby = b1y - b0y;
  const D sbpx = -sby, sbpy = sbx;
  double lmin = INFINITY;
  bool hit = false;
  for (int w = 0; w < W; ++w) {
    const D ax(walls[4 * w]), ay(walls[4 * w + 1]), bx(walls[4 * w + 2]), by(walls[4 * w + 3]);
    const D d0x = b0x - ax, d0y = b0y - ay;
    const D sax = bx - ax, say = by - ay;
    const D sapx = -say, sapy = sax;
    const D la = (d0x * sbpx + d0y * sbpy) / (sax * sbpx + say * sbpy);
    const D lb = ((-d0x) * sapx + (-d0y) * sapy) / (sbx * sapx + sby * sapy);
    if (la.v > 0.0 && la.v < 1.0 && lb.v > 0.0 && lb.v < 1.0) {
      hit = true;
      lmin = fmin(lmin, lb.v);
    }
  }
  if (hit) {
    const D f = D(0.95) * D(lmin);
    dx = (D(dx) * f).v;
    dy = (D(dy) * f).v;
  }
}

// Two uniforms in (0,1) of the Philox counter c (53 bits each; the NumPy mirror reproduces them exactly).
RIAB_DEV void philox_uniforms(uint32_t (&c)[4], uint64_t seed, double& u1, double& u2) {
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  u1 = u01_53(c[0], c[1]);
  u2 = u01_53(c[2], c[3]);
}

RIAB_DEV void subagent_uniforms(uint64_t seed, uint64_t agent, uint32_t sub, uint64_t step, uint32_t stream, double& u1,
                                double& u2) {
  uint32_t c[4];
  philox_ctr(c, agent, sub, step, stream, 0u);
  philox_uniforms(c, seed, u1, u2);
}

// np.random.rayleigh(scale) from a uniform U in (0,1): scale sqrt(-2 log(1 - U))
RIAB_DEV double rayleigh_of(double scale, double u) {
  return (D(scale) * dsqrt(D(-2.0) * D(log((D(1.0) - D(u)).v)))).v;
}

}  // namespace riab

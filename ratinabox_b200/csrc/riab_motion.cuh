// Agent.update (ratinabox/Agent.py:160-242, random-motion branch, 2D solid
// rectangular box) for ONE agent per thread, in float64.  Expressions follow the
// order NumPy evaluates them in the reference (D = non-contracting double) so
// that the wall-collision decisions are bit-identical to the oracle's.
#pragma once
#include "riab_common.cuh"

namespace riab {

struct AgentState {
  double px, py, vx, vy, rot, mvx, mvy, mrot, hdx, hdy, dist, dclose;
};

RIAB_DEV void load_agent(const riab_agents& ag, int64_t i, AgentState& s) {
  const double2 p = reinterpret_cast<const double2*>(ag.pos)[i];
  const double2 v = reinterpret_cast<const double2*>(ag.velocity)[i];
  const double2 mv = reinterpret_cast<const double2*>(ag.measured_velocity)[i];
  const double2 hd = reinterpret_cast<const double2*>(ag.head_direction)[i];
  s.px = p.x; s.py = p.y; s.vx = v.x; s.vy = v.y; s.mvx = mv.x; s.mvy = mv.y; s.hdx = hd.x; s.hdy = hd.y;
  s.rot = ag.rotational_velocity[i];
  s.mrot = ag.measured_rotational_velocity[i];
  s.dist = ag.distance_travelled[i];
  s.dclose = ag.distance_to_closest_wall[i];
}

RIAB_DEV void store_agent(const riab_agents& ag, int64_t i, const AgentState& s) {
  reinterpret_cast<double2*>(ag.pos)[i] = make_double2(s.px, s.py);
  reinterpret_cast<double2*>(ag.velocity)[i] = make_double2(s.vx, s.vy);
  reinterpret_cast<double2*>(ag.measured_velocity)[i] = make_double2(s.mvx, s.mvy);
  reinterpret_cast<double2*>(ag.head_direction)[i] = make_double2(s.hdx, s.hdy);
  ag.rotational_velocity[i] = s.rot;
  ag.measured_rotational_velocity[i] = s.mrot;
  ag.distance_travelled[i] = s.dist;
  ag.distance_to_closest_wall[i] = s.dclose;
}

// Per-call scalars that are the same for every agent, computed once on the host with
// the reference's operation order (plain IEEE double arithmetic, no contraction).
struct MotionDerived {
  double w_theta, w_sigma;      // rotational OU: theta = 1/tau, sigma = sqrt(2 std^2 / (tau dt))   utils.py:364-366
  double v_theta, v_sigma;      // speed OU (noise_scale = 1)
  double two_sm2;               // 2 * speed_mean_kw^2                                          utils.py:418
  double drift_theta;           // 1 / (speed_coherence_time / ratio)                           Agent.py:340
  double v0, k, d, d2;          // wall_repel_strength * speed_mean, v0^2/d^2, d, d*d           Agent.py:367-389
  double cv, cp;                // 3 (1-thig)^2, 6 thig^2                                       Agent.py:399,415
  double hd_a, hd_b;            // 1 - dt/tau, dt/tau                                           Agent.py:498
  double half_sm;               // 0.5 * speed_mean                                             Agent.py:439
};

inline void derive_motion(const riab_motion_params& p, MotionDerived& m) {
  const double dt = p.dt;
  m.w_theta = 1.0 / p.rotational_velocity_coherence_time_kw;
  m.w_sigma = sqrt((2.0 * (p.rotational_velocity_std_kw * p.rotational_velocity_std_kw)) /
                   (p.rotational_velocity_coherence_time_kw * dt));
  m.v_theta = 1.0 / p.speed_coherence_time_kw;
  m.v_sigma = sqrt((2.0 * (1.0 * 1.0)) / (p.speed_coherence_time_kw * dt));
  m.two_sm2 = 2.0 * (p.speed_mean_kw * p.speed_mean_kw);
  m.drift_theta = 1.0 / (p.speed_coherence_time / p.drift_to_random_strength_ratio);
  m.d = p.wall_repel_distance_kw;
  m.v0 = p.wall_repel_strength_kw * p.speed_mean;
  m.d2 = m.d * m.d;
  m.k = (m.v0 * m.v0) / m.d2;
  m.cv = 3.0 * ((1.0 - p.thigmotaxis_kw) * (1.0 - p.thigmotaxis_kw));
  m.cp = 6.0 * (p.thigmotaxis_kw * p.thigmotaxis_kw);
  m.hd_b = dt / p.head_direction_smoothing_timescale;
  m.hd_a = 1.0 - m.hd_b;
  m.half_sm = 0.5 * p.speed_mean;
}

// utils.ornstein_uhlenbeck (utils.py:347-368): returns dx; `n` is the standard
// normal, np.random.normal(scale=dt) == dt*n.
RIAB_DEV D ou_dx(D dt, D x, D drift, D theta, D sigma, D n) {
  return theta * (drift - x) * dt + sigma * (dt * n);
}

// 0 < num/den < 1 decided without the division.  Exactly the IEEE result: for finite
// operands fl(num/den) > 0 <=> num, den share a sign (num != 0), and fl(num/den) < 1 <=>
// |num| < |den|; NaN / zero denominators compare false like the reference's NaN / inf.
RIAB_DEV bool unit_open(D num, D den) {
  const bool same = (num.v > 0.0 && den.v > 0.0) || (num.v < 0.0 && den.v < 0.0);
  return same && (fabs(num.v) < fabs(den.v));
}

// utils.get_angle for a 2-vector (utils.py:231-273): atan2(y, x+1e-6) mod 2pi
RIAB_DEV double get_angle(double x, double y) {
  return np_mod(atan2(y, __dadd_rn(x, 1e-6)), 2.0 * M_PI);
}

// Even-odd ray cast over `count` polygon edges stored as walls (wall i = [v_{i+1}, v_i], Environment.py:137-144):
// strictly inside <=> odd number of crossings and not on an edge (shapely `contains`, Environment.py:810-817).
RIAB_DEV bool edges_contain(double x, double y, const double* __restrict__ w, int count) {
  bool inside = false;
  for (int i = 0; i < count; ++i) {
    const D x1(w[4 * i]), y1(w[4 * i + 1]), x0(w[4 * i + 2]), y0(w[4 * i + 3]);
    const D cross = (x1 - x0) * (D(y) - y0) - (y1 - y0) * (D(x) - x0);
    if (cross.v == 0.0 && fmin(x0.v, x1.v) <= x && x <= fmax(x0.v, x1.v) && fmin(y0.v, y1.v) <= y && y <= fmax(y0.v, y1.v))
      return false;                                                   // on an edge or a vertex: not inside
    if ((y0.v > y) != (y1.v > y)) {
      const D xi = x0 + (D(y) - y0) * (x1 - x0) / (y1 - y0);
      if (x < xi.v) inside = !inside;
    }
  }
  return inside;
}
// In the environment: inside the boundary polygon (first n_poly walls) and in no hole (walls [hole0, hole0+n_hole)).
RIAB_DEV bool env_contains(double x, double y, const double* __restrict__ walls, int n_poly, int hole0, int n_hole) {
  if (!edges_contain(x, y, walls, n_poly)) return false;
  // the holes are disjoint polygons: strictly inside one of them <=> odd crossings over all their edges.
  // A point on a hole's edge is not in that hole (nor in another one), so it is in the environment.
  return (n_hole == 0) || !edges_contain(x, y, walls + 4 * hole0, n_hole);
}

// Environment.apply_boundary_conditions (Environment.py:855-894) for a position that may have left the environment.
// Polygon or holes: "just resample random position" (:890-893) -- uniform in the extent until inside, draw(t, u1, u2)
// giving the t-th pair of uniforms (the position is kept if 1024 draws miss).  Rectangle: pos % extent when periodic
// (:877-879), else clamped 0.01 inside (:880-889).
template <class Draw>
RIAB_DEV void apply_boundary(D& px, D& py, const double* __restrict__ ext, const double* __restrict__ walls, bool periodic,
                             bool polygon, int n_poly, int hole0, int n_hole, Draw draw) {
  if (polygon) {
    if (!env_contains(px.v, py.v, walls, n_poly, hole0, n_hole)) {
      for (uint32_t t = 0; t < 1024u; ++t) {
        double u1, u2;
        draw(t, u1, u2);
        const double qx = ext[0] + u1 * (ext[1] - ext[0]);
        const double qy = ext[2] + u2 * (ext[3] - ext[2]);
        if (env_contains(qx, qy, walls, n_poly, hole0, n_hole)) { px = D(qx); py = D(qy); break; }
      }
    }
  } else if (!((px.v > ext[0]) && (px.v < ext[1]) && (py.v > ext[2]) && (py.v < ext[3]))) {
    if (periodic) {
      px = D(np_mod(px.v, ext[1]));
      py = D(np_mod(py.v, ext[3]));
    } else {
      px = D(fmin(fmax(px.v, ext[0] + 0.01), ext[1] - 0.01));
      py = D(fmin(fmax(py.v, ext[2] + 0.01), ext[3] - 0.01));
    }
  }
}

// A pos / prev_pos pair's displacement; through the boundary when periodic (Environment.py:670-675)
RIAB_DEV void step_displacement(D px, D py, D ppx, D ppy, bool periodic, double scale, D& stx, D& sty) {
  stx = px - ppx; sty = py - ppy;
  if (periodic) {
    const double half = scale / 2;
    if (fabs(stx.v) > half) stx = D(-copysign(1.0, stx.v)) * (D(scale) - D(fabs(stx.v)));
    if (fabs(sty.v) > half) sty = D(-copysign(1.0, sty.v)) * (D(scale) - D(fabs(sty.v)));
  }
}

// A8-A10 of Agent.update, after the position of the step is known: measured velocity / rotational velocity, head
// direction and distance travelled from the step's displacement (stx, sty) and the previous measured velocity.
// Writes s.mrot, s.hdx, s.hdy, s.dist and returns the measured velocity in (mvx, mvy); the caller stores it.  SOURCE:
// the imported / forced branches (_measure_velocity_of_step_taken(overwrite_velocity=True), Agent.py:444-472): a NaN
// in pos or prev_pos (nan_step) makes the measured velocities NaN and adds 0 to the distance travelled.
template <bool SOURCE>
RIAB_DEV void measure_tail(AgentState& s, D stx, D sty, double pmvx, double pmvy, D dt, const riab_motion_params& p,
                           const MotionDerived& m, double fallback_n1, double fallback_n2, D& mvx, D& mvy,
                           bool nan_step = false) {
  // ---- A8: measured velocity / rotational velocity (Agent.py:444-472)
  mvx = stx / dt; mvy = sty / dt;
  if (SOURCE && nan_step) { mvx = D(__longlong_as_double(0x7ff8000000000000ll)); mvy = mvx; }     // Agent.py:451-454
  if (dsqrt(mvx * mvx + mvy * mvy).v == 0.0) {
    // 1e-8 * randn(2) in the reference; here a Philox draw keyed by the (bit-cast) seed / step^agent words
    uint32_t c[4] = {(uint32_t)__double_as_longlong(fallback_n2), (uint32_t)(__double_as_longlong(fallback_n2) >> 32),
                     0x4d454153u, RIAB_STREAM_MEASURE << 24};
    philox4x32_10(c, (uint32_t)__double_as_longlong(fallback_n1), (uint32_t)(__double_as_longlong(fallback_n1) >> 32));
    mvx = D(1e-8 * (2.0 * u01_53(c[0], c[1]) - 1.0));
    mvy = D(1e-8 * (2.0 * u01_53(c[2], c[3]) - 1.0));
  }
  {
    // utils.pi_domain(get_angle(now) - get_angle(before)) (utils.py:231-273, :331-341).  get_angle is
    // atan2(y, x + 1e-6) mod 2pi; the wrapped difference of the two angles equals the signed angle
    // between the eps-shifted vectors, atan2(cross, dot): one atan2 instead of two plus three fmods
    // (identical up to rounding; pi_domain maps to (-pi, pi] like atan2).
    const double x1 = __dadd_rn(pmvx, 1e-6), y1 = pmvy, x2 = __dadd_rn(mvx.v, 1e-6), y2 = mvy.v;
    const double ang = atan2(x1 * y2 - y1 * x2, x1 * x2 + y1 * y2);
    s.mrot = __ddiv_rn(ang, dt.v);
  }

  // ---- A9: head direction low-pass (Agent.py:474-500)
  {
    const D nmv = dsqrt(mvx * mvx + mvy * mvy);
    const D ix = mvx / nmv, iy = mvy / nmv;
    const D tau(p.head_direction_smoothing_timescale);
    if (tau.v <= dt.v) { s.hdx = ix.v; s.hdy = iy.v; }
    else {
      const D a(m.hd_a), b(m.hd_b);
      const D hx = D(s.hdx) * a + b * ix, hy = D(s.hdy) * a + b * iy;
      const D nh = dsqrt(hx * hx + hy * hy);
      s.hdx = (hx / nh).v; s.hdy = (hy / nh).v;
    }
  }

  // ---- A10: distance travelled (Agent.py:502-507; a NaN in pos or prev_pos adds 0)
  if (!SOURCE || !nan_step) {
    s.dist = (D(s.dist) + dsqrt(stx * stx + sty * sty)).v;
  }
}

// walls: shared/global array of W*(ax,ay,bx,by) doubles.
// REC: write the per-iteration collision masks (parity taps).
template <bool REC>
RIAB_DEV void motion_step(AgentState& s, const double* __restrict__ walls, int W, const riab_motion_params& p,
                          const MotionDerived& m, const double* __restrict__ ext, bool periodic, double scale,
                          bool polygon, int n_poly, int hole0, int n_hole, double xi1, double xi2, bool has_drift, double drx,
                          double dry, double fallback_n1, double fallback_n2, uint8_t* __restrict__ mask,
                          int32_t* __restrict__ first_hit, int32_t* __restrict__ n_iters_out) {
  const D dt(p.dt);
  const D ppx(s.px), ppy(s.py);          // prev_pos           Agent.py:199
  const double pmvx = s.mvx, pmvy = s.mvy;  // prev_measured_velocity :201

  // ---- A1: rotational velocity OU + rotation (Agent.py:289-296, utils.py:293-301)
  D rot(s.rot);
  rot = rot + ou_dx(dt, rot, D(p.rotational_velocity_drift_kw), D(m.w_theta), D(m.w_sigma), D(xi1));
  double sn, cs;
  sincos((rot * dt).v, &sn, &cs);
  D vx = D(cs) * D(s.vx) + D(-sn) * D(s.vy);
  D vy = D(sn) * D(s.vx) + D(cs) * D(s.vy);

  // ---- A2: speed, Rayleigh <-> normal OU (Agent.py:298-312, utils.py:409-421)
  D speed = dsqrt(vx * vx + vy * vy);
  if (speed.v == 0.0) { vx = D(1e-8); vy = D(0.0); speed = D(1e-8); }
  {
    const D sm(p.speed_mean_kw);
    double u = (D(1.0) - D(exp((-(speed * speed) / D(m.two_sm2)).v))).v;
    u = fmin(fmax(1e-6, u), 1.0 - 1e-6);
    D z(normcdfinv(u));
    z = z + ou_dx(dt, z, D(0.0), D(m.v_theta), D(m.v_sigma), D(xi2));
    const D cdf(normcdf(z.v));
    D speed_new = sm * dsqrt(D(-2.0) * D(log((D(1.0) - cdf).v)));
    if (p.speed_std == 0.0) speed_new = sm;
    const D f = speed_new / speed;
    vx = f * vx; vy = f * vy;
  }

  // ---- A3: drift towards drift_velocity (Agent.py:324-341; noise_scale = 0)
  if (has_drift) {
    const D theta(m.drift_theta);
    vx = vx + (theta * (D(drx) - vx) * dt + D(0.0));
    vy = vy + (theta * (D(dry) - vy) * dt + D(0.0));
  }

  // ---- A4: wall repulsion (Agent.py:343-421, utils.py:121-184; zero jitter)
  D px(s.px), py(s.py);
  if (p.wall_repel_strength_kw != 0.0 && W > 0) {
    const D d(m.d), v0(m.v0), k(m.k), dd2(m.d2);
    D accx(0.0), accy(0.0), spx(0.0), spy(0.0);
    double dmin2 = INFINITY;
    const double near2 = m.d2 * (1.0 + 1e-9);          // conservative pre-filter for x <= d
    for (int w = 0; w < W; ++w) {
      const D ax(walls[4 * w]), ay(walls[4 * w + 1]), bx(walls[4 * w + 2]), by(walls[4 * w + 3]);
      const D ddx = px - ax, ddy = py - ay, sx = bx - ax, sy = by - ay;
      const D s2 = sx * sx + sy * sy;
      D l = (ddx * sx + ddy * sy) / s2;
      // a zero-length wall (the reference's own tests/test_environment.py:20-23 adds one) is a point: the reference's 1e-6
      // jitter (utils.py:143-144) turns it into a ~1e-6 m segment; with zero jitter its 0/0 would poison the state with NaN
      if (s2.v == 0.0) l = D(0.0);
      if (l.v > 1.0) l = D(1.0);
      if (l.v < 0.0) l = D(0.0);
      const D qx = px - (ax + l * sx), qy = py - (ay + l * sy);
      const D x2 = qx * qx + qy * qy;
      dmin2 = (x2.v < dmin2 || x2.v != x2.v) ? x2.v : dmin2;     // min of the distances == sqrt(min x^2)
      if (x2.v <= near2 || x2.v != x2.v) {
        // only walls within wall_repel_distance contribute (the others add exact zeros, Agent.py:390-393)
        const D x = dsqrt(x2);
        // x == 0: the agent sits exactly on the wall (e.g. Ag.pos = [0.5, 0.5] with a wall at x = 0.5).  The reference's jitter
        // gives that case a random 1e-6 m offset; without it the unit normal is 0/0, so the wall is skipped for this step
        if (x <= d && x.v > 0.0) {
          const D ux = qx / x, uy = qy / x;
          const D acc = k * (d - x);
          const D dx2 = (d - x) * (d - x);
          const D spd = v0 * (D(1.0) - dsqrt(D(1.0) - dx2 / dd2));
          accx = accx + acc * ux; accy = accy + acc * uy;
          spx = spx + spd * ux; spy = spy + spd * uy;
        }
      }
    }
    s.dclose = __dsqrt_rn(dmin2);
    const D cv(m.cv), cp(m.cp);
    vx = vx + cv * (accx * dt);
    vy = vy + cv * (accy * dt);
    px = px + cp * (spx * dt);
    py = py + cp * (spy * dt);
  }

  // ---- A5: integrate (Agent.py:216)
  px = px + vx * dt;
  py = py + vy * dt;

  // ---- A6: collision loop (Agent.py:423-441, Environment.py:820-841, utils.py:30-118)
  int iters = 0;
  for (; iters < RIAB_MAX_BOUNCE_ITERS; ++iters) {
    const D sbx = px - ppx, sby = py - ppy;         // step segment (b list): prev_pos -> pos
    const D sbpx = -sby, sbpy = sbx;
    int first = -1;
    for (int w = 0; w < W; ++w) {
      const D ax(walls[4 * w]), ay(walls[4 * w + 1]), bx(walls[4 * w + 2]), by(walls[4 * w + 3]);
      const D d0x = ppx - ax, d0y = ppy - ay;       // b0 - a0
      const D sax = bx - ax, say = by - ay;
      const D sapx = -say, sapy = sax;
      // 0 < l_a < 1 and 0 < l_b < 1 (utils.py:96-106) without the two divisions (unit_open is exact)
      const bool hit = unit_open(d0x * sbpx + d0y * sbpy, sax * sbpx + say * sbpy) &&
                       unit_open((-d0x) * sapx + (-d0y) * sapy, sbx * sapx + sby * sapy);
      if (REC && mask != nullptr && iters < RIAB_MAX_REC_ITERS) mask[iters * W + w] = hit ? 1 : 0;
      if (hit && first < 0) first = w;
    }
    if (REC && first_hit != nullptr && iters < RIAB_MAX_REC_ITERS) first_hit[iters] = first;
    if (first < 0) { ++iters; break; }
    // utils.wall_bounce (utils.py:304-328) + rescale to 0.5*speed_mean (Agent.py:439)
    const double* wl = walls + 4 * first;
    D parx = D(wl[2]) - D(wl[0]), pary = D(wl[3]) - D(wl[1]);
    D perx = -pary, pery = parx;
    if ((perx * vx + pery * vy).v <= 0.0) { perx = -perx; pery = -pery; }
    if ((parx * vx + pary * vy).v <= 0.0) { parx = -parx; pary = -pary; }
    const D npar = dsqrt(parx * parx + pary * pary), nper = dsqrt(perx * perx + pery * pery);
    parx = parx / npar; pary = pary / npar; perx = perx / nper; pery = pery / nper;
    const D dpar = vx * parx + vy * pary, dper = vx * perx + vy * pery;
    D nvx = parx * dpar - perx * dper, nvy = pary * dpar - pery * dper;
    const D f = D(m.half_sm) / dsqrt(nvx * nvx + nvy * nvy);
    vx = f * nvx; vy = f * nvy;
    px = ppx + vx * dt; py = ppy + vy * dt;
  }
  if (REC && n_iters_out != nullptr) *n_iters_out = iters;

  // ---- A7: still inside? else clamp (Environment.py:781-818, :880-889)
  {
    // (the reference re-draws from np.random; a Philox stream keyed like the zero-displacement fall-back here)
    const long long k1 = __double_as_longlong(fallback_n1), k2 = __double_as_longlong(fallback_n2);
    apply_boundary(px, py, ext, walls, periodic, polygon, n_poly, hole0, n_hole, [&](uint32_t t, double& u1, double& u2) {
      uint32_t c[4] = {(uint32_t)k2, (uint32_t)(k2 >> 32), 0x52534d50u + t, RIAB_STREAM_MEASURE << 24};
      philox4x32_10(c, (uint32_t)k1, (uint32_t)(k1 >> 32));
      u1 = u01_53(c[0], c[1]);
      u2 = u01_53(c[2], c[3]);
    });
  }
  D stx, sty, mvx, mvy;
  step_displacement(px, py, ppx, ppy, periodic, scale, stx, sty);
  measure_tail<false>(s, stx, sty, pmvx, pmvy, dt, p, m, fallback_n1, fallback_n2, mvx, mvy);
  s.px = px.v; s.py = py.v; s.vx = vx.v; s.vy = vy.v; s.rot = rot.v; s.mvx = mvx.v; s.mvy = mvy.v;
}

// Agent.save_to_history row (Agent.py:509-521) as 8 float32
RIAB_DEV void store_history_row(float* __restrict__ row, const AgentState& s) {
  float4* r = reinterpret_cast<float4*>(row);
  r[0] = make_float4((float)s.px, (float)s.py, (float)s.mvx, (float)s.mvy);
  r[1] = make_float4((float)s.hdx, (float)s.hdy, (float)s.mrot, (float)s.dist);
}

}  // namespace riab

// libriab_b200.so -- kernels + C ABI (include/riab_b200.h).  sm_90a (H100) only.
//
// Kernel inventory
//   k_agent_update      Agent.update, one agent per thread (float64)
//   k_agent_update_src  Agent.update from an imported trajectory / forced positions, one agent per thread (float64)
//   k_traj_build        not-a-knot spline of imported trajectories, one thread per (trajectory, axis) column
//   k_step<P,MODE,..>   persistent warp-specialised step kernel for PlaceCells / GridCells / ObjectVectorCells /
//                       head direction, velocity and speed cells / AgentVectorCells / PhasePrecessingPlaceCells /
//                       PlaneWaveNeurons:
//                       producer warps run Agent.update (float64) and publish per-agent float32
//                       records through an mbarrier ring; consumer warps keep 4 cells per thread
//                       in registers and stream float4 rate rows (+ OU noise, + bit-packed spikes)
//   k_bvc_rays<TABLE>   BVC phase A (float64 rays)
//   k_bvc_integrate     BVC phase B (float32 angular integral, TMA-staged tables)
//   k_td_*              TD learning of ValueNeuron / SuccessorFeatures (riab_td.cuh)
//   k_nnn<BN>           NeuralNetworkNeurons: a Linear / activation chain over the input rows, one launch (riab_nnn.cu)
//   k_theta_seq         ThetaSequenceAgent sweep positions over a lead Agent's batch, one agent per thread (float64)
//   k_subagent          DumbAgent / ShiftAgent / ReplayAgent positions over a lead Agent's batch, one agent per thread (float64)
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#include "riab_bvc.cuh"
#include "riab_ffl.cuh"
#include "riab_ovc.cuh"
#include "riab_avc.cuh"
#include "riab_grid.cuh"
#include "riab_kin.cuh"
#include "riab_motion.cuh"
#include "riab_nnn.cuh"
#include "riab_place.cuh"
#include "riab_pppc.cuh"
#include "riab_pwn.cuh"
#include "riab_rsn.cuh"
#include "riab_traj.cuh"
#include "riab_td.cuh"
#include "riab_theta.cuh"
#include "riab_subagent.cuh"

using namespace riab;

namespace {

thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define RIAB_CUDA_OK(expr)                                                                   \
  do {                                                                                       \
    cudaError_t e__ = (expr);                                                                \
    if (e__ != cudaSuccess) return fail(RIAB_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(e__)); \
  } while (0)

constexpr int TA = 32;      // agents per tile (one warp runs their motion)
constexpr int NT = 256;     // threads per CTA in the tile kernels
constexpr int MAXW = RIAB_MAX_STEP_WALLS;    // walls the rate kernels stage in static shared memory
// The motion kernels (k_agent_update, k_subagent, k_theta_seq) stage all RIAB_MAX_WALLS walls in dynamic shared memory,
// W * 32 bytes: within the 48 KB every kernel may use without an opt-in.
static_assert(RIAB_MAX_WALLS * 32 <= 48 * 1024, "motion wall staging needs no dynamic shared memory opt-in");
constexpr int CELL_PAD = 128;  // packed per-cell arrays are padded to 4 cells x 32 lanes

struct EnvK {
  const double* walls;
  int W, nb, aligned, periodic;
  int polygon, nh, h0;      // RIAB_BOUNDARY_POLYGON: even-odd in-environment test over walls [0,nb) and [h0,h0+nh)
  double ext[4];
  double cxm, cym, scale;
};

struct OutK {
  float* rates;
  long long ld;
  uint32_t* spikes;
  long long spike_ld;       // words per row
  float* noise;
  float dt, noise_decay, noise_sig;   // n <- n + (-n*dt/tau) + sig*xi ; decay = dt/tau
  unsigned long long seed, step;
  long long id_offset;
  int pop, vec_ok;
  uint32_t rk7[14];         // Philox4x32-7 round keys of the spike stream (host-computed, constant bank)
  // thinned spikes (thin_block): candidates at rate p' = dt * (an upper bound of the rate), accepted with rate / bound
  int tile_agents;          // agents per ring slot of k_step (<= TA, even): launch_tile shrinks the tiles of small batches so
                            // that every (CTA, consumer group) gets an equal share (strong scaling: a batch of fewer than
                            // 4 full slots per group would otherwise leave part of the last wave idle)
  int thin;                 // 1: the population's rates are bounded and p' = dt * bound <= 1/16 (thin_block)
  uint32_t thin_cdf[32];    // cdf[k] = floor(2^32 P(Binomial(128, p') <= k)): candidates of a (row, 128-cell block) = #{k: word >= cdf[k]}
  float thin_c1, thin_c0;   // accept <=> fma(float(20-bit uniform), c1, c0) < rate;  c1 = 2^-20 bound, c0 = 2^-21 bound
};

// MODE 3 of k_step: the whole riab_run loop of a single Place / Grid / PlaneWave population in ONE launch.  Agents are independent and
// the tile -> CTA assignment is static, so a CTA can run all n_steps for its own agents with no grid-wide synchronisation:
// the producers keep advancing their tiles into the next step while the consumers still write the rates of this one, and
// the per-launch ramp (wall staging, cell registers, first records) and tail are paid once per run instead of once per step.
struct RunK {
  long long n_steps;
  float* rates_ring;            // (ring_rows, A, ld): step s writes row (ring_next + s) % ring_rows
  uint32_t* spikes_ring;        // (ring_rows, A, spike_ld) or NULL
  long long ring_rows, ring_next;
  float* hist_ring;             // (hist_rows, A, 8) agent history rows or NULL
  long long hist_rows, hist_next;
  SrcK src;                     // MODE 4: the motion source that replaces the random motion (riab_run_src)
};

// ---------------------------------------------------------------------------
// walls -> shared memory through a 1-D TMA bulk copy when 16-byte aligned.
__device__ __forceinline__ void stage_walls(double* s_walls, uint64_t* bar, const EnvK& env) {
  const uint32_t bytes = (uint32_t)env.W * 32u;
  if (env.aligned) {
    if (threadIdx.x == 0) {
      mbar_init(bar, 1);
      mbar_fence_init();
      mbar_expect_tx(bar, bytes);
      tma_bulk_g2s(s_walls, env.walls, bytes, bar);
    }
    __syncthreads();
    mbar_wait(bar, 0);
  } else {
    for (int i = threadIdx.x; i < env.W * 4; i += blockDim.x) s_walls[i] = env.walls[i];
    __syncthreads();
  }
}

// One agent's Agent.update inside a kernel (loads/stores its state).
template <bool REC>
__device__ __forceinline__ void agent_update_one(const riab_agents& ag, const riab_motion_params& mp,
                                                 const MotionDerived& md, const riab_step_io& io, const EnvK& env,
                                                 const double* s_walls, long long i, AgentState& s) {
  load_agent(ag, i, s);
  double n1, n2;
  const unsigned long long gid = (unsigned long long)(ag.id_offset + i);
  if (io.xi != nullptr) { n1 = io.xi[2 * i]; n2 = io.xi[2 * i + 1]; }
  else agent_normals(io.seed, io.step, gid, n1, n2);
  const bool has_drift = io.drift_velocity != nullptr;
  double drx = 0.0, dry = 0.0;
  if (has_drift) { drx = io.drift_velocity[2 * i]; dry = io.drift_velocity[2 * i + 1]; }
  // exactly-zero displacement (Agent.py:460-461) draws from a separate Philox stream, lazily
  const double f1 = __longlong_as_double((long long)io.seed), f2 = __longlong_as_double((long long)(io.step ^ (gid << 20)));
  uint8_t* mask = (REC && io.collision_mask) ? io.collision_mask + (size_t)i * RIAB_MAX_REC_ITERS * env.W : nullptr;
  int32_t* fh = (REC && io.first_hit) ? io.first_hit + (size_t)i * RIAB_MAX_REC_ITERS : nullptr;
  int32_t* ni = (REC && io.n_iters) ? io.n_iters + i : nullptr;
  motion_step<REC>(s, s_walls, env.W, mp, md, env.ext, env.periodic != 0, env.scale, env.polygon != 0, env.nb, env.h0, env.nh,
                   n1, n2, has_drift, drx, dry, f1, f2,
                   mask, fh, ni);
  store_agent(ag, i, s);
  if (io.pos_mirror != nullptr) *reinterpret_cast<double2*>(io.pos_mirror + 2 * (size_t)i) = make_double2(s.px, s.py);
  if (io.history_row != nullptr) store_history_row(io.history_row + 8 * (size_t)i, s);
}

// One agent's imported / forced Agent.update at time t (step io.step; same zero-displacement keys as the random branch).
__device__ __forceinline__ void agent_update_src_one(const riab_agents& ag, const riab_motion_params& mp,
                                                     const MotionDerived& md, const riab_step_io& io, const SrcK& src,
                                                     double t, const EnvK& env, long long i, AgentState& s) {
  load_agent(ag, i, s);
  const unsigned long long gid = (unsigned long long)(ag.id_offset + i);
  const double f1 = __longlong_as_double((long long)io.seed), f2 = __longlong_as_double((long long)(io.step ^ (gid << 20)));
  source_step(s, src, i, t, mp, md, env.periodic != 0, env.scale, f1, f2);
  store_agent(ag, i, s);
  if (io.pos_mirror != nullptr) *reinterpret_cast<double2*>(io.pos_mirror + 2 * (size_t)i) = make_double2(s.px, s.py);
  if (io.history_row != nullptr) store_history_row(io.history_row + 8 * (size_t)i, s);
}

__global__ void __launch_bounds__(128) k_agent_update_src(const riab_agents ag, const riab_motion_params mp,
                                                          const MotionDerived md, const riab_step_io io, const SrcK src,
                                                          const EnvK env) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ag.n_agents) return;
  AgentState s;
  agent_update_src_one(ag, mp, md, io, src, src.t, env, i, s);
}

// dynamic shared memory: env.W * 32 bytes of walls (motion_walls_bytes)
template <bool REC>
__global__ void __launch_bounds__(128) k_agent_update(const riab_agents ag, const riab_motion_params mp,
                                                      const MotionDerived md, const riab_step_io io, const EnvK env) {
  extern __shared__ __align__(128) unsigned char dyn[];
  double* s_walls = reinterpret_cast<double*>(dyn);
  __shared__ uint64_t s_bar;
  stage_walls(s_walls, &s_bar, env);
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ag.n_agents) return;
  AgentState s;
  agent_update_one<REC>(ag, mp, md, io, env, s_walls, i, s);
}

// ---------------------------------------------------------------------------
// Neurons.update tail for 4 consecutive cells of one agent: OU noise
// (Neurons.py:153-160,168), rate store, spikes (Neurons.py:681-684).
// `full4`: all 4 cells exist and the row is 16-byte aligned (vector store).
// Per-thread constants of the rate tail (4 consecutive cells).
struct TailCtx {
  int cell0, n_cells;
  unsigned vmask;          // which of the 4 cells exist
  bool full4;              // all 4 exist and rows are 16-byte aligned -> one vector store
  uint32_t sub;            // Philox counter word 1: cell group index
  uint32_t c2, c3_spk;     // Philox counter words 2,3 (step, stream | population)
};

// Row cursor of one thread: pointers into the current agent's rows, advanced per agent.
struct RowCursor {
  float* dst;              // rates row + cell0
  float* nz;               // noise-state row + cell0 (or NULL)
  uint32_t* spk;           // spikes row + 4 * (cell0 / 128): the 4 ballot words of this warp's 128 cells
  unsigned long long gid;  // global agent id
};

__device__ __forceinline__ void tail_init(TailCtx& t, const OutK& out, int cell0, int n_cells, unsigned long long step) {
  t.cell0 = cell0; t.n_cells = n_cells;
  t.vmask = 0u;
#pragma unroll
  for (int i = 0; i < 4; ++i) t.vmask |= (cell0 + i < n_cells) ? (1u << i) : 0u;
  t.full4 = out.vec_ok && (t.vmask == 0xfu);
  t.sub = (uint32_t)(cell0 >> 2);
  t.c2 = (uint32_t)step;
  const uint32_t hi = ((uint32_t)(step >> 32) & 0xffffu) | (((uint32_t)out.pop & 0xffu) << 16);
  t.c3_spk = hi | (RIAB_STREAM_SPIKES << 24);
}

__device__ __forceinline__ void cursor_init(RowCursor& rc, const OutK& out, const TailCtx& t, long long row) {
  rc.dst = out.rates + row * out.ld + t.cell0;
  rc.nz = out.noise ? out.noise + row * out.ld + t.cell0 : nullptr;
  rc.spk = out.spikes ? out.spikes + row * out.spike_ld + ((t.cell0 >> 7) << 2) : nullptr;
  rc.gid = (unsigned long long)(out.id_offset + row);
}
struct RowStride { long long rate, spk; int rows; };      // element strides for `rows` agents (warp-uniform)
__device__ __forceinline__ RowStride make_stride(const OutK& out, int rows) {
  RowStride st;
  st.rate = (long long)rows * out.ld; st.spk = (long long)rows * out.spike_ld; st.rows = rows;
  return st;
}
__device__ __forceinline__ void cursor_advance(RowCursor& rc, const RowStride& st) {
  rc.dst += st.rate;
  if (rc.nz) rc.nz += st.rate;
  if (rc.spk) rc.spk += st.spk;
  rc.gid += (unsigned long long)st.rows;
}

// Neurons.update tail for 4 consecutive cells of one agent, part 1: OU noise
// (Neurons.py:153-160,168) and the rate store.
template <bool NOISE>
__device__ __forceinline__ void store4(float (&o)[4], const OutK& out, const TailCtx& t, const RowCursor& rc,
                                       long long row_off /* extra rows, in elements of ld */) {
  if (NOISE && rc.nz != nullptr) {
    uint32_t c[4];
    philox_ctr(c, rc.gid + (row_off != 0 ? 1ull : 0ull), t.sub, out.step, RIAB_STREAM_CELL_NOISE, (uint32_t)out.pop);
    philox4x32_10(c, (uint32_t)out.seed, (uint32_t)(out.seed >> 32));
    float z[4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float u1 = u01_24(c[2 * h]), u2 = u01_24(c[2 * h + 1]);
      const float r = sqrtf(-2.0f * __logf(u1));
      float sn, cs;
      __sincosf(6.2831853071795865f * u2, &sn, &cs);
      z[2 * h] = r * cs; z[2 * h + 1] = r * sn;
    }
    float* nzp = rc.nz + row_off;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if ((t.vmask >> i) & 1u) {
        float n = nzp[i];
        n = n + (-n * out.noise_decay) + out.noise_sig * z[i];
        nzp[i] = n;
        o[i] += n;
      }
    }
  }
  float* dst = rc.dst + row_off;
  if (t.full4) {
    st_cs_f4(dst, o[0], o[1], o[2], o[3]);
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if ((t.vmask >> i) & 1u) st_cs_f1(dst + i, o[i]);
  }
}

// Part 2: spikes (Neurons.py:681-684), spike <=> uniform < dt * rate.
// One Philox4x32-7 call serves the 4 cells of TWO agents (global ids 2k, 2k+1):
//   r = Philox7(ctr = (gid >> 1, cell group, step, stream|population), key = seed)
//   agent half h = gid & 1 takes words r[2h], r[2h+1]: four 16-bit integers m_i (cell i = half-word i);
//   all eight share the dither v = ((r0^r2) >> 8) * 2^-24; uniform_i = (m_i + v) * 2^-16, and
//   spike_i <=> m_i < fma(rate_i, dt*65536, -v)      (one FFMA, one I2F, one FSETP per rate).
// (m_i + v) is uniform on [0, 65536) with 40 random bits and v is independent of every single m_i;
// sharing v only correlates the sub-2^-16 fractions of the eight uniforms (covariance < 6e-11).
// Layout of a spike row: a warp owns 128 consecutive cells (lane L holds cells 128B+4L .. +3) and
// writes the four ballots of its cell slots as one 16-byte store:
//   bit L of word 4B+i  =  spike of cell 128B + 4L + i.
__device__ __forceinline__ void spike_words(uint32_t (&c)[4], const OutK& out, const TailCtx& t, unsigned long long gid) {
  const unsigned long long pair = gid >> 1;
  c[0] = (uint32_t)pair; c[1] = t.sub ^ ((uint32_t)(pair >> 32) << 24); c[2] = t.c2; c[3] = t.c3_spk;
  philox_keyed<7>(c, out.rk7);
}
__device__ __forceinline__ float spike_neg_dither(const uint32_t (&c)[4]) {
  return (float)((c[0] ^ c[2]) >> 8) * -5.9604644775390625e-08f;
}
// ballots of one agent's 4 cell slots; `ok` = this thread's cells exist (all 4 or none) when !MASKED.
template <bool MASKED>
__device__ __forceinline__ void spike_ballots(uint32_t (&b)[4], uint32_t w0, uint32_t w1, float nv, const float (&o)[4],
                                              float q /* dt * 65536 */, unsigned vmask, bool ok) {
  float m0, m1, m2, m3;           // the four 16-bit integers as floats (I2F.U16 reads either half-word directly)
  asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.rn.f32.u16 %0, l;\n\tcvt.rn.f32.u16 %1, h;\n\t}" : "=f"(m0), "=f"(m1) : "r"(w0));
  asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.rn.f32.u16 %0, l;\n\tcvt.rn.f32.u16 %1, h;\n\t}" : "=f"(m2), "=f"(m3) : "r"(w1));
  bool s0 = m0 < fmaf(o[0], q, nv);
  bool s1 = m1 < fmaf(o[1], q, nv);
  bool s2 = m2 < fmaf(o[2], q, nv);
  bool s3 = m3 < fmaf(o[3], q, nv);
  if (MASKED) { s0 = s0 && (vmask & 1u); s1 = s1 && (vmask & 2u); s2 = s2 && (vmask & 4u); s3 = s3 && (vmask & 8u); }
  else { s0 = s0 && ok; s1 = s1 && ok; s2 = s2 && ok; s3 = s3 && ok; }
  b[0] = __ballot_sync(0xffffffffu, s0);
  b[1] = __ballot_sync(0xffffffffu, s1);
  b[2] = __ballot_sync(0xffffffffu, s2);
  b[3] = __ballot_sync(0xffffffffu, s3);
}
__device__ __forceinline__ void spike_store(const uint32_t (&b)[4], uint32_t* spk) {
  // every lane holds the same four words: one elected lane stores them (whole warp must call)
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "@p st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};\n\t}" ::"l"(spk), "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3])
      : "memory");
}
// A position in a ring slot's spike staging block (shared memory, same layout as the global rows; see k_step): the whole
// run's consumers store their ballot words there, and the slot's producer writes the block to HBM as whole lines.
struct SmemSpk { uint32_t addr; };
__device__ __forceinline__ SmemSpk operator+(const SmemSpk p, const long long words) { return {p.addr + 4u * (uint32_t)words}; }
__device__ __forceinline__ SmemSpk& operator+=(SmemSpk& p, const long long words) { p.addr += 4u * (uint32_t)words; return p; }
__device__ __forceinline__ void spike_store(const uint32_t (&b)[4], const SmemSpk spk) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "@p st.shared.v4.u32 [%0], {%1,%2,%3,%4};\n\t}" ::"r"(spk.addr), "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3])
      : "memory");
}
// one agent (whole warp must call); SP: uint32_t* (global row) or SmemSpk (staging block)
template <class SP>
__device__ __forceinline__ void spikes1(const float (&o)[4], const OutK& out, const TailCtx& t, const unsigned long long gid,
                                        const SP spk) {
  uint32_t c[4], b[4];
  spike_words(c, out, t, gid);
  const float nv = spike_neg_dither(c);
  const unsigned h = (unsigned)(gid & 1ull);
  spike_ballots<true>(b, h ? c[2] : c[0], h ? c[3] : c[1], nv, o, out.dt * 65536.0f, t.vmask, true);
  spike_store(b, spk);
}
// agents gid and, if has_b, gid + 1 of the general path (whole warp must call): one Philox call for a complete pair
// that starts on an even id, else one per agent
template <class SP>
__device__ __forceinline__ void spikes_pair(const float (&oa)[4], const float (&ob)[4], const bool has_b, const bool even,
                                            const OutK& out, const TailCtx& t, const unsigned long long gid, const SP spk,
                                            const float q16) {
  if (has_b && even) {
    uint32_t c[4], bl[4];
    spike_words(c, out, t, gid);
    const float nv = spike_neg_dither(c);
    spike_ballots<true>(bl, c[0], c[1], nv, oa, q16, t.vmask, true);
    spike_store(bl, spk);
    spike_ballots<true>(bl, c[2], c[3], nv, ob, q16, t.vmask, true);
    spike_store(bl, spk + out.spike_ld);
  } else {
    spikes1(oa, out, t, gid, spk);
    if (has_b) spikes1(ob, out, t, gid + 1ull, spk + out.spike_ld);
  }
}

template <bool SPIKES, bool NOISE>
__device__ __forceinline__ void finish4(float (&o)[4], const OutK& out, const TailCtx& t, const RowCursor& rc) {
  store4<NOISE>(o, out, t, rc, 0);
  if (SPIKES && (!NOISE || rc.spk != nullptr)) spikes1(o, out, t, rc.gid, rc.spk);
}

// ---------------------------------------------------------------------------
// Cell-type policies for the step kernel.
// COMP: the compensated direct form (PlaceConst::comp, riab_place.cuh): kernels of their own, chosen by the host, so the
// expanded kernels keep their code and registers.  GEO: the geodesic kernel (one inner wall, run-time profile, COMP), whose
// record carries the agent -> wall-end distances as well.
template <int WI, int DESC, bool COMP = false, bool GEO = false>
struct PlacePolicy {
  using Const = PlaceConst;
  using Regs = PlaceCellRegs<WI>;
  static constexpr int REC = place_rec(WI, GEO);
  static constexpr bool LIGHT = (WI == 0) && (DESC >= 0) && !COMP;   // few instructions per rate: HBM-bound consumers
  // rates lie in [min_fr, max_fr], so the thinned spike stream applies, but it measured slower for place cells: the
  // Euclidean Gaussian loop is HBM-bound and hides the dense stream's instructions under its stores, the line-of-sight
  // loop with the post-pass needs 8 producer warps and loses next to them.  The dense stream stays.
  static constexpr bool THIN = false;
  static constexpr bool POSITIONAL = true;
  static __device__ __forceinline__ void given_dir(const Const&, long long, double&, double&) {}
  static __device__ __forceinline__ void prepare(double* aux, const double* s_walls, const Const& c) {
    place_wall_invariants(aux, s_walls + 4 * c.wall0, WI > 0 ? c.n_inner : 0);
  }
  static __device__ __forceinline__ void record(float* rec, long long, double px, double py, double, double, double, double, double, double,
                                                const double* s_walls, const double* aux, const Const& c, const EnvK& env) {
    place_agent_record<WI, COMP, GEO>(rec, px, py, s_walls + 4 * c.wall0, aux, WI > 0 ? c.n_inner : 0, env.cxm, env.cym, c.band, c.expanded, c.kx, c.fold ? c.lspan : 0.f);
  }
  static __device__ __forceinline__ void load(Regs& r, const Const& c, int cell0) { place_load_cells<WI, COMP, GEO>(r, c, cell0); }
  template <bool DEFER, int EXP = -1>
  static __device__ __forceinline__ void rates4(float (&o)[4], const Regs& r, const Const& c, int cell0,
                                                const float* rec, uint32_t inner_s, bool& unsure) {
    place_rates4<WI, DESC, DEFER, EXP, COMP, GEO>(o, r, c, cell0, rec, inner_s, unsure);
  }
  // 0: direct form, 1: expanded exponent, 2: expanded with the [0, max_fr] scale folded into the exponent
  static __device__ __forceinline__ int expanded(const Const& c) {
    return (!COMP && DESC == RIAB_PC_GAUSSIAN && c.expanded) ? 1 + c.fold : 0;
  }
  static __device__ __forceinline__ int wall0(const Const& c) { return c.wall0; }
};

// TURNS = 1: the block holds turns (riab_grid_cells::phase_turns) and the rates take the compensated phase.  A kernel of
// its own, chosen by the host: the radian kernels keep their code and registers.
template <int TURNS>
struct GridPolicy {
  using Const = GridConst;
  using Regs = GridCellRegs;
  static constexpr int REC = 4;
  static constexpr bool LIGHT = false;    // 36 cell registers per thread do not fit StepCfg<8>'s 56-register consumers
  static constexpr bool THIN = true;      // bounded rates, consumer-bound loop: thinned spikes
  static constexpr bool POSITIONAL = true;
  static __device__ __forceinline__ void given_dir(const Const&, long long, double&, double&) {}
  static __device__ __forceinline__ void prepare(double*, const double*, const Const&) {}
  static __device__ __forceinline__ void record(float* rec, long long, double px, double py, double, double, double, double, double, double,
                                                const double*, const double*, const Const&, const EnvK& env) {
    rec[0] = (float)(px - env.cxm);
    rec[1] = (float)(py - env.cym);
  }
  static __device__ __forceinline__ void load(Regs& r, const Const& c, int cell0) { grid_load_cells(r, c, cell0); }
  template <bool DEFER, int EXP = -1>
  static __device__ __forceinline__ void rates4(float (&o)[4], const Regs& r, const Const& c, int, const float* rec,
                                                uint32_t, bool&) {
    grid_rates4<TURNS>(o, r, c, rec);
  }
  static __device__ __forceinline__ int expanded(const Const&) { return 0; }
  static __device__ __forceinline__ int wall0(const Const&) { return 0; }
};

struct OvcPolicy {
  using Const = OvcConst;
  using Regs = OvcCellRegs;
  static constexpr int REC = OVC_REC;
  static constexpr bool LIGHT = false;
  static constexpr bool THIN = false;     // sums over objects: no a-priori rate bound
  static constexpr bool POSITIONAL = true;
  // egocentric cells evaluated at given positions: their head directions
  static __device__ __forceinline__ void given_dir(const Const& c, long long i, double& x, double& y) {
    if (c.head_dir != nullptr) { x = c.head_dir[2 * i]; y = c.head_dir[2 * i + 1]; }
  }
  static __device__ __forceinline__ void prepare(double*, const double*, const Const&) {}
  static __device__ __forceinline__ void record(float* rec, long long, double px, double py, double hdx, double hdy, double, double,
                                                double, double, const double* s_walls, const double*, const Const& c,
                                                const EnvK&) {
    ovc_agent_record(rec, px, py, hdx, hdy, s_walls, c);
  }
  static __device__ __forceinline__ void load(Regs& r, const Const& c, int cell0) { ovc_load_cells(r, c, cell0); }
  template <bool DEFER, int EXP = -1>
  static __device__ __forceinline__ void rates4(float (&o)[4], const Regs& r, const Const& c, int, const float* rec,
                                                uint32_t, bool&) {
    ovc_rates4(o, r, c, rec);
  }
  static __device__ __forceinline__ int expanded(const Const&) { return 0; }
  static __device__ __forceinline__ int wall0(const Const&) { return 0; }
};

// Head direction / velocity / speed cells: the record is the agent's kinematic state, not its position.  MODE 0 takes the
// state from KinConst::vec (the agents' arrays, or get_state's vectors with no positions at all: pos_in may be NULL).
struct KinPolicy {
  using Const = KinConst;
  using Regs = KinCellRegs;
  static constexpr int REC = KIN_REC;
  static constexpr bool LIGHT = true;     // one ex2 per rate, 12 cell registers: HBM-bound consumers
  static constexpr bool THIN = false;     // velocity and speed rates have no a-priori bound: dense spike stream
  static constexpr bool POSITIONAL = false;
  static __device__ __forceinline__ void given_dir(const Const& c, long long i, double& x, double& y) {
    if (c.vec != nullptr) { x = c.vec[c.vec_ld * i]; y = c.vec[c.vec_ld * i + 1]; }
  }
  static __device__ __forceinline__ void prepare(double*, const double*, const Const&) {}
  static __device__ __forceinline__ void record(float* rec, long long, double, double, double hdx, double hdy, double vx, double vy,
                                                double mvx, double mvy, const double*, const double*, const Const& c,
                                                const EnvK&) {
    kin_agent_record(rec, hdx, hdy, vx, vy, mvx, mvy, c);
  }
  static __device__ __forceinline__ void load(Regs& r, const Const& c, int cell0) { kin_load_cells(r, c, cell0); }
  template <bool DEFER, int EXP = -1>
  static __device__ __forceinline__ void rates4(float (&o)[4], const Regs& r, const Const& c, int, const float* rec,
                                                uint32_t, bool&) {
    kin_rates4(o, r, c, rec);
  }
  static __device__ __forceinline__ int expanded(const Const&) { return 0; }
  static __device__ __forceinline__ int wall0(const Const&) { return 0; }
};

// AgentVectorCells: OvcPolicy's geometry for one "object", the partner Agent's position of the record's row.
struct AvcPolicy {
  using Const = AvcConst;
  using Regs = AvcCellRegs;
  static constexpr int REC = AVC_REC;
  // 20 cell registers: as a LIGHT policy, ptxas -v reports 56-60 spill bytes in its StepCfg<8> instantiations (KinPolicy's
  // 12 registers: 28-32), so the consumers keep the 96-register configurations like OvcPolicy
  static constexpr bool LIGHT = false;
  static constexpr bool THIN = false;     // the dense spike stream, as for OVC (a NaN partner gives NaN rates)
  static constexpr bool POSITIONAL = true;
  static __device__ __forceinline__ void given_dir(const Const& c, long long i, double& x, double& y) {
    if (c.head_dir != nullptr) { x = c.head_dir[2 * i]; y = c.head_dir[2 * i + 1]; }
  }
  static __device__ __forceinline__ void prepare(double*, const double*, const Const&) {}
  static __device__ __forceinline__ void record(float* rec, long long i, double px, double py, double hdx, double hdy, double,
                                                double, double, double, const double* s_walls, const double*, const Const& c,
                                                const EnvK&) {
    avc_agent_record(rec, px, py, hdx, hdy, i, s_walls, c);
  }
  static __device__ __forceinline__ void load(Regs& r, const Const& c, int cell0) { avc_load_cells(r, c, cell0); }
  template <bool DEFER, int EXP = -1>
  static __device__ __forceinline__ void rates4(float (&o)[4], const Regs& r, const Const& c, int, const float* rec,
                                                uint32_t, bool&) {
    avc_rates4(o, r, c, rec);
  }
  static __device__ __forceinline__ int expanded(const Const&) { return 0; }
  static __device__ __forceinline__ int wall0(const Const&) { return 0; }
};

// PhasePrecessingPlaceCells: PlacePolicy's record, cells and rates (direct exponent form), times the theta modulation
// factor of riab_pppc.cuh.  MODE 0 reads the rows' velocities from Const::vel (given_dir: the one given vector stands for
// every kinematic input).
template <int WI, int DESC, bool COMP = false, bool GEO = false>
struct PppcPolicy {
  using Place = PlacePolicy<WI, DESC, COMP, GEO>;
  using Const = PppcConst;
  using Regs = PppcCellRegs<WI>;
  static constexpr int REC = pppc_rec(WI, GEO);
  static constexpr bool LIGHT = false;    // ~10 more instructions per rate and 12 more cell registers than PlacePolicy
  static constexpr bool THIN = false;     // the factor has no a-priori bound below M max_fr: dense spike stream
  static constexpr bool POSITIONAL = true;
  static __device__ __forceinline__ void given_dir(const Const& c, long long i, double& x, double& y) {
    if (c.vel != nullptr) { x = c.vel[2 * i]; y = c.vel[2 * i + 1]; }
  }
  static __device__ __forceinline__ void prepare(double* aux, const double* s_walls, const Const& c) {
    Place::prepare(aux, s_walls, c);
  }
  static __device__ __forceinline__ void record(float* rec, long long i, double px, double py, double hdx, double hdy,
                                                double vx, double vy, double mvx, double mvy, const double* s_walls,
                                                const double* aux, const Const& c, const EnvK& env) {
    Place::record(rec, i, px, py, hdx, hdy, vx, vy, mvx, mvy, s_walls, aux, c, env);
    pppc_direction_record(rec + pppc_dir(WI, GEO), px, py, vx, vy, env.cxm, env.cym);
  }
  static __device__ __forceinline__ void load(Regs& r, const Const& c, int cell0) {
    Place::load(r.p, c, cell0);
    pppc_load_phase<WI>(r, c);
  }
  template <bool DEFER, int EXP = -1>
  static __device__ __forceinline__ void rates4(float (&o)[4], const Regs& r, const Const& c, int cell0,
                                                const float* rec, uint32_t inner_s, bool& unsure) {
    Place::template rates4<DEFER, 0>(o, r.p, c, cell0, rec, inner_s, unsure);
    pppc_modulate4<WI>(o, r, c, rec + pppc_dir(WI, GEO));
  }
  static __device__ __forceinline__ int expanded(const Const&) { return 0; }
  static __device__ __forceinline__ int wall0(const Const& c) { return c.wall0; }
};

// PlaneWaveNeurons (riab_pwn.cuh): one cosine per rate.  The phase form (radians, or compensated turns) is a uniform
// run-time branch of one kernel, so the population costs 15 k_step instantiations, not 30.
struct PwnPolicy {
  using Const = PwnConst;
  using Regs = PwnCellRegs;
  static constexpr int REC = 4;
  // Chosen with scripts/bench_pwn.py (65 536 agents x 1 024 cells, whole run, compensated phase; H100 80GB HBM3, 700 W):
  // spikes on, the dense stream in StepCfg<4> ran 119.6 us / step against 134.1 with the thinned stream and 135.3 with
  // LIGHT's dense StepCfg<12>, so THIN = false and LIGHT = false; without spikes LIGHT's StepCfg<8> would save 3 us
  // (90.3 against 93.4), less than it costs with spikes, which the reference records by default.
  static constexpr bool LIGHT = false;
  static constexpr bool THIN = false;
  static constexpr bool POSITIONAL = true;
  static __device__ __forceinline__ void given_dir(const Const&, long long, double&, double&) {}
  static __device__ __forceinline__ void prepare(double*, const double*, const Const&) {}
  static __device__ __forceinline__ void record(float* rec, long long, double px, double py, double, double, double, double, double, double,
                                                const double*, const double*, const Const&, const EnvK& env) {
    pwn_agent_record(rec, px, py, env.cxm, env.cym);
  }
  static __device__ __forceinline__ void load(Regs& r, const Const& c, int cell0) { pwn_load_cells(r, c, cell0); }
  template <bool DEFER, int EXP = -1>
  static __device__ __forceinline__ void rates4(float (&o)[4], const Regs& r, const Const& c, int, const float* rec,
                                                uint32_t, bool&) {
    pwn_rates4(o, r, c, rec);
  }
  static __device__ __forceinline__ int expanded(const Const&) { return 0; }
  static __device__ __forceinline__ int wall0(const Const&) { return 0; }
};

// ---------------------------------------------------------------------------
// k_step: persistent, warp-specialised step kernel (one CTA per SM).
//   warps [0, MW)        producers: each takes a tile of 32 agents, runs Agent.update for its
//                        lane's agent in float64 (MOTION) or just reads the position, writes the
//                        agent state back, and publishes a float32 "rate record" per agent into a
//                        shared-memory ring slot (mbarrier full[slot]).
//   warps [MW, MW+RW)    consumers: every thread keeps 4 consecutive cells in registers, waits for
//                        a slot, streams the slot's agents through the rate evaluator and writes
//                        float4 rate rows (+ noise + bit-packed spikes), then frees the slot
//                        (mbarrier empty[slot]).
// The float64 motion latency (a ~2.5k-instruction dependent chain) is thereby hidden behind the
// HBM-bound rate writes of earlier tiles instead of idling the CTA.
// Warp-role configuration.  The register file is re-balanced between the roles with setmaxnreg (the float64 motion code wants
// ~130 registers, the consumers 56..104).  Three splits, all 16 consumer warps:
//   StepCfg<4>:  4 producers x 64 registers (spilling), consumers x 104 (640 threads x 96 at launch).  Pair loops with
//                spikes or OU noise: the consumers set the pace and want the registers.
//   StepCfg<8>:  8 producers x 128, consumers x 56 (768 threads x 80): light consumers without spikes (Euclidean Gaussian
//                place cells) run at the HBM write rate, so the float64 motion chain needs the producer warps and the
//                registers to keep up.
//   StepCfg<12>: 8 producers x 48 (spilling), consumers x 96 (768 threads x 80): heavier loops WITHOUT spikes (line of sight,
//                grid cells) and the light loop WITH the dense spike stream, where 4 producers leave the consumers waiting
//                for records.
// A split that exceeds a sub-partition's launch allocation hangs (step_cfg_fits below).
constexpr int RW = 16;    // consumer warps
template <int ID>
struct StepCfg {
  static_assert(ID == 4 || ID == 8 || ID == 12, "unknown warp-role configuration");
  static constexpr int MW = (ID == 4) ? 4 : 8;                     // producer warps
  static constexpr int CTAS = 1;                                  // CTAs per SM
  static constexpr int NS = (ID == 8) ? MW : 2 * MW;              // ring slots (multiple of MW; static smem <= 48 KB)
  static constexpr int THREADS = (MW + RW) * 32;
  // what __launch_bounds__(THREADS, 1) allocates: the register file is per SM sub-partition (16384 registers, warp w on
  // sub-partition w % 4), so ptxas sizes for the fullest one -- 704 threads (22 warps, 6 on one sub-partition) get 80, not 88
  static constexpr int WARPS_SP = (MW + RW + 3) / 4;
  static constexpr int REGS_LAUNCH = (16384 / (WARPS_SP * 32)) / 8 * 8;
  static constexpr int REGS_PRODUCER = (ID == 4) ? 64 : (ID == 8) ? 128 : 48;
  static constexpr int REGS_CONSUMER = (ID == 4) ? 104 : (ID == 8) ? 56 : 96;
};
// setmaxnreg only moves registers WITHIN the launch allocation of a sub-partition (its warps x REGS_LAUNCH): an .inc blocks
// until enough warps have released theirs with .dec.  A split whose total exceeds the allocation therefore never
// completes -- the hang of round 1's 112 / 56 experiment (4 x 32 x 112 + 32 x 56 = 16128 > 5 x 32 x 96 = 15360) and of a
// 6-producer variant with 96-register consumers in round 2 (4 x 32 x 96 + 2 x 32 x 64 = 16384 > 6 x 32 x 80).
template <class C>
constexpr bool step_cfg_fits() {
  return (RW / 4) * 32 * C::REGS_CONSUMER + ((C::MW + 3) / 4) * 32 * C::REGS_PRODUCER <= C::WARPS_SP * 32 * C::REGS_LAUNCH;
}
static_assert(step_cfg_fits<StepCfg<4>>() && step_cfg_fits<StepCfg<8>>() && step_cfg_fits<StepCfg<12>>(),
              "setmaxnreg split exceeds the CTA's register allocation: the kernel would hang");
// setmaxnreg towards N registers from the launch allocation L (inc when N > L, dec when N < L)
template <int N, int L> __device__ __forceinline__ void reg_set() {
  if (N > L) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
  else if (N < L) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// ring slots of a (policy, configuration): the configuration's count, halved for the fat records (8 inner walls, object
// vector cells: 160 B per agent) while the ring would not fit in 40 KB of the 48 KB static shared memory
template <class P, class C>
constexpr int ring_slots() {
  int ns = C::NS;
  while (ns >= 2 * C::MW && ns * (TA * P::REC * 4 + 16) > 40 * 1024) ns /= 2;
  return ns;
}

// Consumer groups of the lean slot loop: each ring slot is consumed by ONE group, slot q by group q % G.  A group must see
// every phase of the slots it waits on (an mbarrier parity wait cannot skip a phase), so G has to divide the ring size.
__host__ __device__ constexpr int lean_groups(int cell_threads, int ring) {
  int g = (RW * 32) / (cell_threads > 0 ? cell_threads : 1);
  if (g < 1) g = 1;
  if (g > ring) g = ring;
  while (ring % g != 0) --g;
  return g;
}

template <int REC>
struct __align__(16) StepSlot {
  float rec[TA][REC];
  int na;
  unsigned nanmask;         // bit a: agent a's position is NaN -> its rates are zero (Neurons.py:163-164)
  uint32_t* spk_rows;       // whole run, dense spikes: the tile's first spike row, where its staging block goes (k_step)
};

// The consumers' hot loop: n2 consecutive agent pairs (2p, 2p+1) of one ring slot, no OU noise, 16-byte aligned rows
// (ld floats apart), every thread's 4 cells exist or none (`act`).  recp and d (the first agent's record, rate row + cell0)
// advance past the pairs, with DENSE also spk and pair (spike row + ballot words, global id / 2).  The line-of-sight band
// test is deferred: a pair whose float32 decision fell inside the band only sets its bit in `redo`; the caller redoes
// those pairs through the general path (per-agent exact float64 fall-back) after the loop -- no call, no branch in here.
// DENSE: the dense spike stream (one Philox4x32-7 call per pair, a threshold test per rate; needs an even first global
// id) runs in the loop; thinned spikes are a post-pass over the slot (thin_block) and leave this loop spike-free.
template <class P, bool DENSE, int EXP, class SP>
__device__ __forceinline__ void consume_pairs(const int n2, const typename P::Regs& regs, const typename P::Const& pc,
                                              const OutK& out, const TailCtx& tc, const int cell0, const float*& recp,
                                              const uint32_t inner_s, const long long ld, float*& d, SP& spk,
                                              unsigned long long& pair, const bool act, const float q16, uint32_t& redo) {
  for (int it = 0; it < n2; ++it) {
    float o[4];
    uint32_t c[4], bl[4];
    bool unsure = false;
    P::template rates4<true, EXP>(o, regs, pc, cell0, recp, inner_s, unsure);
    if (act) st_cs_f4(d, o);
    float nv = 0.f;
    if constexpr (DENSE) {
      c[0] = (uint32_t)pair; c[1] = tc.sub ^ ((uint32_t)(pair >> 32) << 24); c[2] = tc.c2; c[3] = tc.c3_spk;
      philox_keyed<7>(c, out.rk7);
      nv = spike_neg_dither(c);
      spike_ballots<false>(bl, c[0], c[1], nv, o, q16, 0u, act);
      spike_store(bl, spk);
    }
    P::template rates4<true, EXP>(o, regs, pc, cell0, recp + P::REC, inner_s, unsure);
    if (act) st_cs_f4(d + ld, o);
    if constexpr (DENSE) {
      spike_ballots<false>(bl, c[2], c[3], nv, o, q16, 0u, act);
      spike_store(bl, spk + out.spike_ld);
      spk += 2 * out.spike_ld;
      pair += 1ull;
    }
    redo |= (unsure ? 1u : 0u) << it;
    d += 2 * ld;
    recp += 2 * P::REC;
  }
}

// ---------------------------------------------------------------------------
// Thinned spikes (Neurons.py:681-684: spike <=> uniform < dt * rate) for populations whose rates are bounded by `bound`
// with p' = dt * bound <= 1/16 (the usual case: dt = 10 ms, max_fr = 1 Hz gives p' = 0.01).  Exact Bernoulli(dt * rate) by
// thinning: every (agent, cell) is a CANDIDATE with probability p', a candidate spikes with probability rate / bound.
// Candidates are drawn per (agent row gid, 128-cell block B) -- the 32 x 128 rates one consumer warp has just stored for a
// ring slot, lane = row -- so that the result does not depend on tiles, shards or the launch path:
//   call n = 0, 1, ...:  R = Philox7(ctr = (gid, B | n << 16, step, THIN | population))
//   K       = #{k < 32 : R_0[0] >= cdf[k]},  cdf[k] = floor(2^32 P(Binomial(128, p') <= k))        (call 0 only)
//   draws   d = 4 n + j, j = 0..3:  position pos_d = (R_n[1] >> 7 j) & 127,
//                                   20-bit uniform x_d = (half-word j of (R_n[2], R_n[3])) << 4 | R_n[1] >> 28
//   the candidates are the first K DISTINCT positions of the draw sequence (a draw that repeats an earlier position is
//   skipped: sampling without replacement, i.e. a uniform K-subset, i.e. 128 independent Bernoulli(p') cells);
//   candidate at pos_d spikes  <=>  fma(float(x_d), c1, c0) < rate[gid, 128 B + pos_d]      (c1 = 2^-20 bound, c0 = 2^-21 bound).
// The pair loop does nothing for spikes.  After a slot's rates are stored the warp runs this once: ~1.3 candidates per
// lane at p' = 0.01, one Philox call per lane serves four of them; the rates are read back from L2 (this warp stored them),
// accepted bits go into the spike rows the producer cleared with RED.OR.  NumPy mirror: tests/philox_np.py (expected_spikes_thin).
// An out-of-line call (like slot_fixups): inlined, its ~40 live registers made ptxas park cell registers of the pair loop in
// local memory (8 LDL per pair iteration: the pass then cost more than the dense stream it replaces).  `out` is the kernel's
// __grid_constant__ parameter, so its address can be passed without a local copy.
__device__ __noinline__ void thin_block(const OutK* __restrict__ outp, const int cell0, const int n_cells, const uint32_t c2,
                                        const uint32_t c3_spk, const float* __restrict__ rates, uint32_t* __restrict__ spikes,
                                        const long long row_lo, const int rows) {
  const OutK& out = *outp;
  const int lane = threadIdx.x & 31;
  const int blk0 = cell0 - 4 * lane;                      // first cell of the warp's block (warp-uniform)
  const int cells_left = n_cells - blk0;
  if (lane >= rows || cells_left <= 0 || spikes == nullptr) return;   // (lanes leave independently: no warp-wide operation in here)
  const uint32_t B = (uint32_t)(blk0 >> 7);
  const long long row = row_lo + lane;
  const unsigned long long gid = (unsigned long long)(out.id_offset + row);
  const uint32_t c1w = B ^ ((uint32_t)(gid >> 32) << 24);
  const uint32_t c3w = (c3_spk & 0x00ffffffu) | (RIAB_STREAM_THIN << 24);
  uint32_t rk[14];
#pragma unroll
  for (int i = 0; i < 14; ++i) rk[i] = out.rk7[i];
  uint32_t R[4] = {(uint32_t)gid, c1w, c2, c3w};
  philox_keyed<7>(R, rk);
  int K = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) K += (R[0] >= out.thin_cdf[k]) ? 1 : 0;        // independent compares
  if (K == 8) while (K < 32 && R[0] >= out.thin_cdf[K]) ++K;
  if (K == 0) return;
  const float c1 = out.thin_c1, c0 = out.thin_c0;
  const float* rrow = rates + row * out.ld + blk0;
  uint32_t* srow = spikes + row * out.spike_ld + 4u * B;
  unsigned long long occ_lo = 0ull, occ_hi = 0ull;
  int cnt = 0;
  for (uint32_t n = 0u;;) {
    uint32_t take = 0u;
    int pos[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      pos[j] = (int)((R[1] >> (7 * j)) & 127u);
      const unsigned long long oh_lo = (pos[j] < 64) ? (1ull << pos[j]) : 0ull;
      const unsigned long long oh_hi = (pos[j] < 64) ? 0ull : (1ull << (pos[j] - 64));
      const bool fresh = (cnt < K) && (((occ_lo & oh_lo) | (occ_hi & oh_hi)) == 0ull);
      if (fresh) { occ_lo |= oh_lo; occ_hi |= oh_hi; ++cnt; }
      if (fresh && pos[j] < cells_left) take |= 1u << j;   // candidates on padding cells count, but have no rate
    }
    float rate[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      rate[j] = 0.f;
      if ((take >> j) & 1u) asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(rate[j]) : "l"(rrow + pos[j]));
    }
    const uint32_t dith = R[1] >> 28;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t m = ((j < 2 ? R[2] : R[3]) >> (16 * (j & 1))) & 0xffffu;
      const float x = (float)((m << 4) | dith);
      if (((take >> j) & 1u) && fmaf(x, c1, c0) < rate[j]) atomicOr(srow + (pos[j] & 3), 1u << (pos[j] >> 2));
    }
    if (cnt >= K || ++n >= 256u) break;
    R[0] = (uint32_t)gid; R[1] = c1w ^ (n << 16); R[2] = c2; R[3] = c3w;
    philox_keyed<7>(R, rk);
  }
}

// The consumers' slot loop (see k_step).  EXP: exponent form of the fast pair loop (PlacePolicy::expanded).
template <class P, int SPK, bool NOISE, class C, int EXP>
__device__ __forceinline__ void consumer_slots(const typename P::Const& pc, const OutK& out, StepSlot<P::REC>* s_slot,
                                               uint64_t* s_full, uint64_t* s_empty, const double* s_walls,
                                               const long long nq, const int ctid, const int lane,
                                               const long long n_rows) {
  constexpr int NS = ring_slots<P, C>();
  constexpr int NC = RW * 32;
  constexpr bool DENSE = (SPK == 1);
  const int CT = pc.n_pad / 4;                        // cell-threads needed (multiple of 32)
  const int chunks = (CT + NC - 1) / NC;
  const int G = (chunks == 1) ? (NC / CT) : 1;        // agent groups when the cells need fewer threads
  const int grp = (chunks == 1) ? (ctid / CT) : 0;
  const bool idle = (chunks == 1) && (grp >= G);
  // group `grp` takes the consecutive agents [2 grp PPG, 2 (grp+1) PPG) of a slot (PPG pairs)
  const int PPG = (TA / 2 + G - 1) / G;
  typename P::Regs regs;
  int cell0 = (chunks == 1) ? (ctid % CT) * 4 : 0;
  TailCtx tc;
  if (chunks == 1 && !idle) {
    P::load(regs, pc, cell0);
    tail_init(tc, out, cell0, pc.n_cells, out.step);
  }
  const uint32_t inner_s = smem_u32(s_walls) + 32u * (uint32_t)P::wall0(pc);   // float64 inner walls (exact fall-back)
  // Fast pair loop: rows are 16-byte aligned and every thread owns 4 existing cells or none, the
  // tile starts on an even global id (one Philox call per agent pair) and there is no OU noise.
  const bool fast = !NOISE && out.vec_ok && ((pc.n_cells & 3) == 0) && ((out.id_offset & 1ll) == 0 || SPK != 1);
  const float q16 = out.dt * 65536.0f;
  for (long long q = 0; q < nq; ++q) {
    const int s = (int)(q % NS);
    mbar_wait(&s_full[s], (uint32_t)((q / NS) & 1));
    const long long a0 = ((long long)blockIdx.x + q * gridDim.x) * out.tile_agents;
    const int na = s_slot[s].na;
    const int a_lo = 2 * grp * PPG;
    const int a_hi = (a_lo + 2 * PPG < na) ? a_lo + 2 * PPG : na;       // this group's agents of the slot: [a_lo, a_hi)
    // chunks == 1: the cell registers loaded above serve every slot; more than 2048 cells: the 16 warps walk
    // the cells in chunks of 2048 and reload their registers per chunk (G = 1, all warps on the same agents)
    for (int ch = 0; ch < chunks; ++ch) {
      if (chunks > 1) {
        cell0 = (ch * NC + ctid) * 4;
        if (cell0 >= pc.n_pad) continue;              // warp-uniform (n_pad is a multiple of 128)
        P::load(regs, pc, cell0);
        tail_init(tc, out, cell0, pc.n_cells, out.step);
      } else if (idle) {
        continue;
      }
      if (a_lo >= a_hi) continue;                     // warp-uniform
      const bool act = cell0 < pc.n_cells;
      {
        // agents are taken in pairs (2p, 2p+1) so that one Philox call feeds the (dense) spikes of both
        RowCursor rc;
        cursor_init(rc, out, tc, a0 + a_lo);
        const float* recp = s_slot[s].rec[a_lo];
        int a = a_lo;
        uint32_t only = 0xffffffffu;       // pairs (by iteration index) the general loop below evaluates
        if (fast) {
          uint32_t redo = 0u;
          const int n2 = (a_hi - a_lo) >> 1;
          unsigned long long pair = rc.gid >> 1;
          consume_pairs<P, DENSE, EXP>(n2, regs, pc, out, tc, cell0, recp, inner_s, out.ld, rc.dst, rc.spk, pair, act, q16, redo);
          a += 2 * n2;
          rc.gid = pair << 1;                      // rc.spk / rc.gid advance with DENSE, the only case that reads them below
          redo = __reduce_or_sync(0xffffffffu, redo);
          if (const unsigned nm = s_slot[s].nanmask; nm != 0u)          // pairs with a NaN position: zero rates below
            for (int it = 0; a_lo + 2 * it < a_hi; ++it)
              if ((nm >> (a_lo + 2 * it)) & 3u) redo |= 1u << it;
          if (redo != 0u) {
            // some float32 line-of-sight decision was inside the band: redo those pairs through the
            // general path (the stores are idempotent); complete pairs not in `redo` are skipped
            only = redo;
            a = a_lo;
            cursor_init(rc, out, tc, a0 + a_lo);
            recp = s_slot[s].rec[a_lo];
          }
        }
        // general path: the last agent of an odd tile, odd shard offsets, OU noise, ragged cell counts
        const RowStride stride = make_stride(out, 2);
        const bool even = ((rc.gid & 1ull) == 0ull);      // uniform: a0 and a_lo are even
        for (uint32_t it = (uint32_t)((a - a_lo) >> 1); a < a_hi; a += 2, ++it) {
          float oa[4], ob[4];
          const bool has_b = (a + 1 < a_hi);
          if (has_b && !((only >> (it & 31u)) & 1u)) {      // warp-uniform
            cursor_advance(rc, stride);
            recp += 2 * P::REC;
            continue;
          }
          bool dummy = false;
          P::template rates4<false>(oa, regs, pc, cell0, recp, inner_s, dummy);
          if (has_b) P::template rates4<false>(ob, regs, pc, cell0, recp + P::REC, inner_s, dummy);
          if (const unsigned nm = s_slot[s].nanmask; nm != 0u) {        // NaN position -> zero rates (Neurons.py:163-164)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              if ((nm >> a) & 1u) oa[i] = 0.f;
              if (has_b && ((nm >> (a + 1)) & 1u)) ob[i] = 0.f;
            }
          }
          store4<NOISE>(oa, out, tc, rc, 0);
          if (has_b) store4<NOISE>(ob, out, tc, rc, out.ld);
          if (DENSE && (!NOISE || rc.spk != nullptr)) spikes_pair(oa, ob, has_b, even, out, tc, rc.gid, rc.spk, q16);
          cursor_advance(rc, stride);
          recp += 2 * P::REC;
        }
        if (SPK == 2) {
          __syncwarp();      // orders this warp's rate stores before the read-back
          thin_block(&out, tc.cell0, tc.n_cells, tc.c2, tc.c3_spk, out.rates, out.spikes, a0 + a_lo, a_hi - a_lo);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&s_empty[s]);
  }
}

// Repairs of one ring slot for consumer_fast, after its pair loop (rare): pairs whose float32 line-of-sight decision fell
// inside the band (bit `it` of redo) are re-evaluated with the exact float64 fall-back, and an odd last agent gets its row.
// Inlined like the pair loop; only the float64 fall-back (place_blocked_exact4) is an out-of-line call.  spk: this warp's
// ballot words in the tile's first spike row (global, or the slot's staging block: the pair loop's words are overwritten there).
template <class P, bool DENSE, class SP>
__device__ __forceinline__ void slot_fixups(const typename P::Regs& regs, const typename P::Const& pc, const OutK& out,
                                            const TailCtx& tc, const float* rec, const uint32_t inner_s, float* d,
                                            const SP spk, const long long a0, const int n_agents, const uint32_t redo,
                                            const bool act) {
  for (int a = 0; a < n_agents; a += 2, d += 2 * out.ld, rec += 2 * P::REC) {
    const bool has_b = a + 1 < n_agents;
    if (has_b && !((redo >> (a >> 1)) & 1u)) continue;              // warp-uniform
    float oa[4], ob[4];
    bool dummy = false;
    P::template rates4<false>(oa, regs, pc, tc.cell0, rec, inner_s, dummy);
    if (has_b) P::template rates4<false>(ob, regs, pc, tc.cell0, rec + P::REC, inner_s, dummy);
    if (act) {
      st_cs_f4(d, oa);
      if (has_b) st_cs_f4(d + out.ld, ob);
    }
    if constexpr (DENSE)                                            // whole warp: ballots; even: consumer_fast's tiles start on even ids
      spikes_pair(oa, ob, has_b, true, out, tc, (unsigned long long)(out.id_offset + a0 + a), spk + a * out.spike_ld, out.dt * 65536.0f);
  }
}

// The consumers' slot loop for the common case: no OU noise, vector-aligned rows, whole 4-cell groups, all cells resident
// in one set of registers (n_pad <= 2048), an even first global id when there are spikes.  Pointers advance incrementally,
// the rare repairs run after the pair loop (slot_fixups), thinned spikes are a post-pass per slot (thin_block).  The whole
// run's dense spike words go to the slot's staging block at `stage` (shared address, see k_step), the stepped paths' to HBM.
template <class P, int SPK, class C, int EXP, bool MULTI>
__device__ __forceinline__ void consumer_fast(const typename P::Const& pc, const OutK& out, const RunK& run, StepSlot<P::REC>* s_slot,
                                              uint64_t* s_full, uint64_t* s_empty, const double* s_walls, const long long nq,
                                              const int ctid, const int lane, const long long n_rows, const uint32_t stage) {
  constexpr int NS = ring_slots<P, C>(), MW = C::MW, NSP = NS / MW;
  constexpr bool STAGED = MULTI && SPK == 1;
  using SP = std::conditional_t<STAGED, SmemSpk, uint32_t*>;
  const int CT = pc.n_pad / 4;                        // cell-threads needed (multiple of 32, <= RW * 32)
  const int G = lean_groups(CT, NS), grp = ctid / CT; // groups of CT threads; group g consumes the tiles q = g, g + G, ...
  if (grp >= G) return;                               // spare warps (the slots' release count is one group's warps)
  constexpr int a_lo = 0;
  typename P::Regs regs;
  const int cell0 = (ctid % CT) * 4;
  TailCtx tc;
  P::load(regs, pc, cell0);
  tail_init(tc, out, cell0, pc.n_cells, out.step);
  const bool act = cell0 < pc.n_cells;                // all 4 cells exist or none (n_cells % 4 == 0)
  const uint32_t inner_s = smem_u32(s_walls) + 32u * (uint32_t)P::wall0(pc);
  const long long ld = out.ld;
  const float q16 = out.dt * 65536.0f;
  const long long a_first = ((long long)blockIdx.x + (long long)grp * gridDim.x) * out.tile_agents;   // first row of the group's first tile
  const long long a_step = (long long)G * gridDim.x * out.tile_agents, slot_step = a_step * ld;
  const long long n_steps = MULTI ? run.n_steps : 1;
  for (long long st = 0; st < n_steps; ++st) {
    // this step's rows: the caller's (single step) or the rings' row (ring_next + st) % ring_rows
    float* rates = out.rates;
    uint32_t* spikes = out.spikes;
    if (MULTI) {
      const long long slot = (run.ring_next + st) % run.ring_rows;
      rates = run.rates_ring + slot * n_rows * ld;
      spikes = run.spikes_ring ? run.spikes_ring + slot * n_rows * out.spike_ld : nullptr;
      tail_init(tc, out, cell0, pc.n_cells, out.step + (unsigned long long)st);
    }
    long long a0 = a_first;
    float* dst0 = rates + a0 * ld + cell0;
    for (long long q = grp; q < nq; q += G, dst0 += slot_step, a0 += a_step) {
      // tile q is produced by warp q % MW as its n-th tile overall: slot and phase of that producer's private ring
      const int pw = (int)(q % MW);
      const long long npw = (nq - pw + MW - 1) / MW;    // tiles of that producer per step
      const long long n = st * npw + q / MW;
      const int s = pw + MW * (int)(n % NSP);
      mbar_wait(&s_full[s], (uint32_t)((n / NSP) & 1));
      const int a_hi = s_slot[s].na;
      if (a_lo < a_hi) {
        const float* recp = s_slot[s].rec[a_lo];
        float* d = dst0;
        uint32_t redo = 0u;
        const int n2 = (a_hi - a_lo) >> 1;
        const auto first_spk = [&]() -> SP {                             // this warp's words in the tile's first spike row
          if constexpr (STAGED) return SmemSpk{stage + 4u * (uint32_t)(s * TA * out.spike_ld + ((cell0 >> 7) << 2))};
          else if constexpr (SPK == 1) return spikes + a0 * out.spike_ld + ((cell0 >> 7) << 2);
          else return nullptr;
        };
        SP spk{};
        unsigned long long pair = 0ull;
        if constexpr (SPK == 1) {
          spk = first_spk();
          pair = (unsigned long long)(out.id_offset + a0) >> 1;          // even first global id: rows (2p, 2p+1) are one pair
        }
        consume_pairs<P, SPK == 1, EXP>(n2, regs, pc, out, tc, cell0, recp, inner_s, ld, d, spk, pair, act, q16, redo);
        redo = __reduce_or_sync(0xffffffffu, redo);
        if (redo != 0u || ((a_hi - a_lo) & 1)) {
          // copies: passing regs / pc themselves leaves every kernel's register and stack use as it is, but ptxas then
          // schedules 65 of the k_step instantiations differently; they stay until a measurement says which is faster
          const typename P::Regs rcopy = regs;
          const typename P::Const pcopy = pc;
          slot_fixups<P, SPK == 1>(rcopy, pcopy, out, tc, s_slot[s].rec[a_lo], inner_s, dst0, first_spk(), a0, a_hi - a_lo, redo, act);
        }
        if (const unsigned nm = s_slot[s].nanmask; nm != 0u && act) {     // NaN position -> zero rates (Neurons.py:163-164)
          for (int a = a_lo; a < a_hi; ++a)
            if ((nm >> a) & 1u) st_cs_f4(dst0 + (long long)(a - a_lo) * ld, 0.f, 0.f, 0.f, 0.f);
        }
        if constexpr (SPK == 2) {
          __syncwarp();                                  // this warp's rate stores before the read-back
          thin_block(&out, tc.cell0, tc.n_cells, tc.c2, tc.c3_spk, rates, spikes, a0 + a_lo, a_hi - a_lo);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&s_empty[s]);
    }
  }
}

// A producer warp publishes the records its lanes < na have written into ring slot `slot`: lane 0 stores the count and the
// NaN-position mask (Neurons.py:163-164: those agents get zero rates), then the warp arrives on the slot's full barrier.
template <int REC>
__device__ __forceinline__ void publish_slot(StepSlot<REC>& slot, uint64_t* full, const int lane, const int na, const bool nanpos) {
  const unsigned nanmask = __ballot_sync(0xffffffffu, nanpos);
  if (lane == 0) { slot.na = na; slot.nanmask = nanmask; }
  __syncwarp();
  if (lane == 0) mbar_arrive(full);
}

// Thinned spikes: a producer lane clears its agent's spike row before the tile is published; the consumers OR accepted bits
// in after that (the mbarrier release / acquire orders these stores before their RED.ORs).
__device__ __forceinline__ void clear_spike_row(uint32_t* row, const long long words) {
  for (long long w = 0; w < words; w += 4)
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%1,%1,%1};" ::"l"(row + w), "r"(0u) : "memory");
}

// Whole run with the dense stream: a producer writes the staging block of a consumed tile (`words` words from shared address
// `src`) to its spike rows at `dst`.  Rows of consecutive agents are contiguous, so the block is one range of whole lines:
// 512 B per warp instruction, instead of the 16-byte pieces each consumer warp would store into every row.
__device__ __forceinline__ void flush_spike_block(uint32_t* dst, const uint32_t src, const int words, const int lane) {
#pragma unroll 4
  for (int w = 4 * lane; w < words; w += 128) {
    uint32_t v0, v1, v2, v3;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3) : "r"(src + 4u * (uint32_t)w) : "memory");
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(dst + w), "r"(v0), "r"(v1), "r"(v2), "r"(v3) : "memory");
  }
}

// bytes of dynamic shared memory k_step needs: the whole run's dense spike staging, one block of TA rows per ring slot
__host__ __device__ constexpr long long spike_stage_bytes(int ring, long long spike_ld) { return (long long)ring * TA * spike_ld * 4; }

// SPK: 0 no spikes, 1 dense spike stream (in the loops), 2 thinned spikes (thin_block per ring slot)
template <class P, int MODE, int SPK, bool NOISE, class C>
__global__ void __launch_bounds__(C::THREADS, C::CTAS) k_step(const EnvK env, const riab_agents ag,
                                                          const riab_motion_params mp, const MotionDerived md,
                                                          const riab_step_io io, const typename P::Const pc, const __grid_constant__ OutK out,
                                                          const double* __restrict__ pos_in, const long long n_rows,
                                                          const RunK run) {
  __shared__ __align__(16) double s_walls[MAXW * 4];
  constexpr int MW = C::MW, NS = ring_slots<P, C>();
  __shared__ StepSlot<P::REC> s_slot[NS];
  __shared__ uint64_t s_bar, s_full[NS], s_empty[NS];
  // whole run, dense spikes: slot s's spike words are assembled in s_stage[s * TA * spike_ld ..] (rows of the tile, laid out
  // like the global rows) and written to HBM by the slot's producer once the consumers have released the slot
  constexpr bool STAGED = MODE >= 3 && SPK == 1 && !NOISE;
  extern __shared__ __align__(128) unsigned char dyn[];
  const uint32_t s_stage = smem_u32(dyn);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // lean consumers (consumer_fast): every ring slot is consumed by ONE group of warps (n_pad / 4 threads), the general
  // loop (consumer_slots) by all RW consumer warps
  bool lean = false;
  if constexpr (!NOISE)
    lean = out.vec_ok && ((pc.n_cells & 3) == 0) && (pc.n_pad <= RW * 32 * 4) && (out.spikes == nullptr || ((out.id_offset & 1ll) == 0));
  if (threadIdx.x == 0) {
    const uint32_t n_release = lean ? (uint32_t)((pc.n_pad / 4) >> 5) : (uint32_t)RW;
    for (int i = 0; i < NS; ++i) { mbar_init(&s_full[i], 1); mbar_init(&s_empty[i], n_release); }
    mbar_fence_init();
  }
  stage_walls(s_walls, &s_bar, env);     // includes __syncthreads()
  __shared__ double s_aux[2 * PLACE_MAX_WI];             // per-wall invariants of the agent records (policy-specific)
  P::prepare(s_aux, s_walls, pc);
  __syncthreads();

  const int ta = out.tile_agents;
  const long long n_tiles = (n_rows + ta - 1) / ta;
  const long long nq = (n_tiles > (long long)blockIdx.x) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  // producers take the HIGHEST warp ids: the issue arbiter prefers higher warp ids among eligible warps, and
  // the float64 motion chain (one instruction every ~20 cycles) must not wait behind 4 busy consumers
  const int pw = warp - RW;
  if (warp >= RW) {
    // ------------------------------------------------------------- producers
    reg_set<C::REGS_PRODUCER, C::REGS_LAUNCH>();
    if constexpr (MODE >= 3) {
      // whole run (MODE 4: following run.src instead of the random motion): this warp advances ITS tiles (q = pw, pw + MW, ...) step after step -- the same warp for every step of a
      // tile, so a tile's steps are ordered -- and publishes each (step, tile) record into its private ring (slots
      // pw + MW * i): the n-th record it produces goes to slot i = n % NSP in phase n / NSP
      constexpr int NSP = NS / MW;
      // its clear of a tile's spike rows for step s+1 may overlap the ORs of up to NSP - 1 earlier steps of that tile, so
      // those steps must have other rows: riab_run launches whole runs with spikes only for ring_rows >= 2 >= NSP
      static_assert(NSP <= 2, "riab_run launches whole runs with spike rings of 2 rows");
      long long n = 0;
      double t_st = run.src.t;                           // MODE 4: Agent.t of step st, advanced by `t += dt` like the host's
      for (long long st = 0; st < run.n_steps; ++st) {
        riab_step_io io_st = io;
        io_st.step = io.step + (unsigned long long)st;
        io_st.history_row = run.hist_ring ? run.hist_ring + ((run.hist_next + st) % run.hist_rows) * n_rows * 8 : nullptr;
        uint32_t* const spikes_st = run.spikes_ring ? run.spikes_ring + ((run.ring_next + st) % run.ring_rows) * n_rows * out.spike_ld : nullptr;
        for (long long q = pw; q < nq; q += MW, ++n) {
          const int s = pw + MW * (int)(n % NSP);
          mbar_wait(&s_empty[s], (uint32_t)(((n / NSP) & 1) ^ 1));
          // the wait acquired the consumers' staging stores of the tile this slot held (record n - NSP): write them out
          if constexpr (STAGED)
            if (n >= NSP) flush_spike_block(s_slot[s].spk_rows, s_stage + (uint32_t)spike_stage_bytes(s, out.spike_ld), s_slot[s].na * (int)out.spike_ld, lane);
          const long long a0 = ((long long)blockIdx.x + q * gridDim.x) * ta;
          const int na = (int)((n_rows - a0) < ta ? (n_rows - a0) : ta);
          if (SPK == 2 && lane < na && spikes_st != nullptr) clear_spike_row(spikes_st + (a0 + lane) * out.spike_ld, out.spike_ld);
          if (STAGED && lane == 0) s_slot[s].spk_rows = spikes_st + a0 * out.spike_ld;     // (publish_slot's __syncwarp orders it)
          bool nanpos = false;
          if (lane < na) {
            AgentState as;
            if constexpr (MODE == 4) agent_update_src_one(ag, mp, md, io_st, run.src, t_st, env, a0 + lane, as);
            else agent_update_one<false>(ag, mp, md, io_st, env, s_walls, a0 + lane, as);
            nanpos = (as.px != as.px);
            P::record(s_slot[s].rec[lane], a0 + lane, as.px, as.py, as.hdx, as.hdy, as.vx, as.vy, as.mvx, as.mvy, s_walls, s_aux, pc, env);
          }
          publish_slot(s_slot[s], &s_full[s], lane, na, nanpos);
        }
        if constexpr (MODE == 4) t_st = t_st + mp.dt;
      }
      if constexpr (STAGED) {
        // the blocks of this warp's last NSP records i: their consumers complete phase i / NSP of s_empty, the phase a
        // refill (record i + NSP) would wait for with parity ((i + NSP) / NSP & 1) ^ 1 = (i / NSP) & 1
        for (long long i = (n > NSP ? n - NSP : 0); i < n; ++i) {
          const int s = pw + MW * (int)(i % NSP);
          mbar_wait(&s_empty[s], (uint32_t)((i / NSP) & 1));
          flush_spike_block(s_slot[s].spk_rows, s_stage + (uint32_t)spike_stage_bytes(s, out.spike_ld), s_slot[s].na * (int)out.spike_ld, lane);
        }
      }
    } else {
      for (long long q = pw; q < nq; q += MW) {
        const int s = (int)(q % NS);
        const uint32_t k = (uint32_t)(q / NS);
        mbar_wait(&s_empty[s], (k & 1u) ^ 1u);
        const long long tile = (long long)blockIdx.x + q * gridDim.x;
        const long long a0 = tile * ta;
        const int na = (int)((n_rows - a0) < ta ? (n_rows - a0) : ta);
        if (SPK == 2 && lane < na) clear_spike_row(out.spikes + (a0 + lane) * out.spike_ld, out.spike_ld);
        if (MODE == 2) {
          // skewed: publish the records of the CURRENT positions first, then advance the agents
          // (the next launch's rates) -- consumers never wait for the float64 motion chain.
          bool nanpos = false;
          if (lane < na) {
            const long long i = a0 + lane;
            const double px = ag.pos[2 * i], py = ag.pos[2 * i + 1];
            nanpos = (px != px);
            P::record(s_slot[s].rec[lane], i, px, py, ag.head_direction[2 * i], ag.head_direction[2 * i + 1], ag.velocity[2 * i],
                      ag.velocity[2 * i + 1], ag.measured_velocity[2 * i], ag.measured_velocity[2 * i + 1], s_walls, s_aux, pc, env);
          }
          publish_slot(s_slot[s], &s_full[s], lane, na, nanpos);
          if (lane < na) {
            AgentState st;
            agent_update_one<false>(ag, mp, md, io, env, s_walls, a0 + lane, st);
          }
          continue;
        }
        bool nanpos = false;
        if (lane < na) {
          const long long i = a0 + lane;
          double px = 0.0, py = 0.0, hdx = 1.0, hdy = 0.0, vx, vy, mvx, mvy;
          if (MODE == 1) {
            AgentState st;
            agent_update_one<false>(ag, mp, md, io, env, s_walls, i, st);
            px = st.px; py = st.py; hdx = st.hdx; hdy = st.hdy; vx = st.vx; vy = st.vy; mvx = st.mvx; mvy = st.mvy;
          } else {
            if (P::POSITIONAL || pos_in != nullptr) { px = pos_in[2 * i]; py = pos_in[2 * i + 1]; }
            P::given_dir(pc, i, hdx, hdy);                      // the one given vector stands for every kinematic input
            vx = mvx = hdx; vy = mvy = hdy;
          }
          nanpos = (px != px);
          P::record(s_slot[s].rec[lane], i, px, py, hdx, hdy, vx, vy, mvx, mvy, s_walls, s_aux, pc, env);
        }
        publish_slot(s_slot[s], &s_full[s], lane, na, nanpos);
      }
    }
  } else {
    // ------------------------------------------------------------- consumers
    reg_set<C::REGS_CONSUMER, C::REGS_LAUNCH>();
    const int ctid = threadIdx.x;
    // one copy of the slot loop per exponent form (0: direct, 1: expanded, 2: expanded + folded scale), chosen once:
    // the cell registers then stay in registers across slots (a run-time switch inside the loop made ptxas park them
    // in local memory around every slot)
    const int ex = P::expanded(pc);
    if constexpr (!NOISE) {
      if (lean) {
        if (ex == 2) consumer_fast<P, SPK, C, 2, (MODE >= 3)>(pc, out, run, s_slot, s_full, s_empty, s_walls, nq, ctid, lane, n_rows, s_stage);
        else if (ex == 1) consumer_fast<P, SPK, C, 1, (MODE >= 3)>(pc, out, run, s_slot, s_full, s_empty, s_walls, nq, ctid, lane, n_rows, s_stage);
        else consumer_fast<P, SPK, C, 0, (MODE >= 3)>(pc, out, run, s_slot, s_full, s_empty, s_walls, nq, ctid, lane, n_rows, s_stage);
        return;
      }
    }
    if constexpr (MODE >= 3) return;                    // (the host launches whole runs only where the lean loop applies)
    if (ex == 2) consumer_slots<P, SPK, NOISE, C, 2>(pc, out, s_slot, s_full, s_empty, s_walls, nq, ctid, lane, n_rows);
    else if (ex == 1) consumer_slots<P, SPK, NOISE, C, 1>(pc, out, s_slot, s_full, s_empty, s_walls, nq, ctid, lane, n_rows);
    else consumer_slots<P, SPK, NOISE, C, 0>(pc, out, s_slot, s_full, s_empty, s_walls, nq, ctid, lane, n_rows);
  }
}

// ---------------------------------------------------------------------------
// PlaceCells description "one_hot" (Neurons.py:972-974): rate = 1 for the cell with the smallest
// distance (np.argmin: first index of the minimum), 0 elsewhere.  One warp per position.  Pass 1 finds the
// minimum float32 squared distance (line-of-sight flags from the same float32 predicate as the rate
// kernels; pairs inside the predicate's uncertainty band count with their unblocked distance); pass 2
// re-evaluates every cell within a relative 1e-5 of that minimum in float64 exactly like the reference
// (np.linalg.norm, utils.vector_intercepts) and keeps the smallest (distance, index).
__device__ __forceinline__ double onehot_exact_dist(const PlaceConst& c, int cell, double px, double py,
                                                    const double* __restrict__ inner64) {
  const double cx = c.centres64[2 * cell], cy = c.centres64[2 * cell + 1];
  bool blocked = false;
  for (int j = 0; j < c.n_inner; ++j) blocked = blocked || los_blocked_exact(cx, cy, px, py, inner64 + 4 * j);
  D ex = D(cx) - D(px), ey = D(cy) - D(py);
  if (c.periodic) {
    if (fabs(ex.v) > c.scale / 2) ex = D(-copysign(1.0, ex.v)) * (D(c.scale) - D(fabs(ex.v)));
    if (fabs(ey.v) > c.scale / 2) ey = D(-copysign(1.0, ey.v)) * (D(c.scale) - D(fabs(ey.v)));
  }
  const double d = dsqrt(ex * ex + ey * ey).v;
  if (!blocked) return d;
  if (c.geometry == RIAB_GEOM_GEODESIC)
    return geodesic_detour_exact(cx, cy, px, py, inner64[0], inner64[1], inner64[2], inner64[3], c.ep_valid);
  return 1000.0;
}

__global__ void __launch_bounds__(NT) k_place_onehot(const EnvK env, const PlaceConst pc, const double* __restrict__ pos,
                                                     const long long n_rows, const OutK out) {
  __shared__ __align__(16) double s_walls[MAXW * 4];
  __shared__ uint64_t s_bar;
  stage_walls(s_walls, &s_bar, env);
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  const double px = pos[2 * row], py = pos[2 * row + 1];
  const double* inner = s_walls + 4 * pc.wall0;
  const float pxf = (float)(px - env.cxm), pyf = (float)(py - env.cym);
  float fp[PLACE_MAX_WI], tp[PLACE_MAX_WI];
  for (int j = 0; j < PLACE_MAX_WI; ++j) {
    fp[j] = 1.f; tp[j] = 0.f;
    if (j < pc.n_inner) {
      double f, t;
      wall_coords(px, py, inner[4 * j], inner[4 * j + 1], inner[4 * j + 2], inner[4 * j + 3], f, t);
      fp[j] = (float)f; tp[j] = (fabs(f) < 1e-9) ? nanf("") : (float)t;
    }
  }
  const int np = pc.n_pad;
  auto d2_of = [&](int cell, bool& unsure) -> float {          // optimistic float32 squared distance of one cell
    float dx = fabsf(pxf - pc.packed[cell]), dy = fabsf(pyf - pc.packed[np + cell]);
    if (pc.periodic) {
      dx = (dx > pc.half_f) ? pc.scale_f - dx : dx;
      dy = (dy > pc.half_f) ? pc.scale_f - dy : dy;
    }
    float d2 = fmaf(dy, dy, dx * dx);
    bool hit = false;
    for (int j = 0; j < pc.n_inner; ++j) {
      const float fc = pc.packed[(size_t)(4 + 2 * j) * np + cell], tcv = pc.packed[(size_t)(5 + 2 * j) * np + cell];
      const float afp = fabsf(fp[j]);
      const float Mp = fmaf(afp, tcv, fabsf(fc) * tp[j]);
      const float mn = fminf(Mp, (fabsf(fc) + afp) - Mp);
      const bool u = !(fabsf(mn) >= pc.eps[j]);
      unsure = unsure || u;
      hit = hit || (((fc * fp[j]) < 0.f) && (mn > 0.f) && !u);
    }
    return hit ? 1.0e6f : d2;
  };
  float best = INFINITY;
  for (int cell = lane; cell < pc.n_cells; cell += 32) {
    bool u = false;
    best = fminf(best, d2_of(cell, u));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = fminf(best, __shfl_xor_sync(0xffffffffu, best, o));
  // Every cell whose true distance ties the true minimum passes the screen: with E a bound on |d_f - d| (the float32
  // rounding of the centred coordinates, coord_err from make_place plus this row's |p'|), the true minimum is at most
  // sqrt(best) + E and such a cell's float32 square at most (sqrt(best) + 2E)^2, both up to the float32 rounding of d^2.
  // Geodesic detours are shorter than 1000: every blocked cell is a candidate there.
  const double E = (double)pc.coord_err + 1.2e-7 * ((double)fabsf(pxf) + (double)fabsf(pyf));
  const double sb = sqrt((double)best) * (1.0 + 1e-6) + 2.0 * E;
  const float thr = (pc.geometry == RIAB_GEOM_GEODESIC && pc.n_inner > 0) ? INFINITY
                    : fmaxf(best * (1.0f + 1e-5f) + 1e-12f, (float)(sb * sb * (1.0 + 1e-6)));
  double bd = INFINITY;
  int bi = 0x7fffffff;
  for (int cell = lane; cell < pc.n_cells; cell += 32) {
    bool u = false;
    const float d2 = d2_of(cell, u);
    if (d2 <= thr || u) {
      const double d = onehot_exact_dist(pc, cell, px, py, inner);
      if (d < bd || (d == bd && cell < bi)) { bd = d; bi = cell; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double od = __shfl_xor_sync(0xffffffffu, bd, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
  }
  const float lo = pc.min_fr, hi = pc.min_fr + pc.span;
  float* dst = out.rates + row * out.ld;
  for (int cell = lane; cell < pc.n_cells; cell += 32) st_cs_f1(dst + cell, cell == bi ? hi : lo);
}

// Noise + spikes post-pass over rate rows that a kernel without finish4 produced (BVC).
__global__ void __launch_bounds__(NT) k_finish_rows(const OutK out, const int n_cells, const int n_pad128,
                                                    const long long n_rows) {
  const long long row = blockIdx.x;                        // rows on x: gridDim.y stops at 65535
  const int cell0 = (blockIdx.y * NT + threadIdx.x) * 4;
  if (row >= n_rows || cell0 >= n_pad128) return;          // warp-uniform: a warp covers 128 consecutive cells
  float o[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) o[i] = (cell0 + i < n_cells) ? out.rates[row * out.ld + cell0 + i] : 0.f;
  TailCtx tc;
  tail_init(tc, out, cell0, n_cells, out.step);
  tc.full4 = false;
  RowCursor rc;
  cursor_init(rc, out, tc, row);
  finish4<true, true>(o, out, tc, rc);
}

// ---------------------------------------------------------------------------
// BVC phase A: one CTA per tile of 32 agents.  Dynamic shared memory: the T directions, then (TABLE) the float32
// directions and the (angle, wall) table of at most BVC_NW walls next to the static wall block, or (!TABLE) the env.W
// float64 walls and their float32 copies (launch_bvc), up to RIAB_MAX_WALLS.
template <bool TABLE>
__global__ void __launch_bounds__(NT, TABLE ? 4 : 1) k_bvc_rays(const EnvK env, const BvcConst bc,
                                                 const double* __restrict__ pos_in, const long long n_rows,
                                                 float* __restrict__ scratch, int32_t* __restrict__ first_wall,
                                                 uint32_t* __restrict__ spikes_zero, const long long spike_ld) {
  extern __shared__ __align__(128) unsigned char dyn[];
  double* s_dirs = reinterpret_cast<double*>(dyn);                 // T*2
  __shared__ __align__(16) double s_walls_tab[TABLE ? MAXW * 4 : 2];
  __shared__ __align__(16) float4 s_wf_tab[TABLE ? MAXW : 1];
  double* s_walls = TABLE ? s_walls_tab : s_dirs + 2 * bc.T;         // 16-byte aligned: T * 16 bytes of directions
  float4* s_wf = TABLE ? s_wf_tab : reinterpret_cast<float4*>(s_walls + 4 * env.W);
  __shared__ __align__(16) double s_pos[TA][2];
  __shared__ uint64_t s_bar;
  stage_walls(s_walls, &s_bar, env);
  for (int i = threadIdx.x; i < 2 * bc.T; i += blockDim.x) s_dirs[i] = bc.test_dirs[i];
  for (int w = threadIdx.x; w < env.W; w += blockDim.x)
    s_wf[w] = make_float4((float)s_walls[4 * w], (float)s_walls[4 * w + 1], (float)(s_walls[4 * w + 2] - s_walls[4 * w]),
                          (float)(s_walls[4 * w + 3] - s_walls[4 * w + 1]));

  const long long a0 = (long long)blockIdx.x * TA;
  const int na = (int)((n_rows - a0) < TA ? (n_rows - a0) : TA);
  if (threadIdx.x < TA) {
    double px = 0.5 * (env.ext[0] + env.ext[1]), py = 0.5 * (env.ext[2] + env.ext[3]);   // padding rows: box centre
    if ((int)threadIdx.x < na) {
      const long long i = a0 + threadIdx.x;
      px = pos_in[2 * i]; py = pos_in[2 * i + 1];
    }
    s_pos[threadIdx.x][0] = px;
    s_pos[threadIdx.x][1] = py;
  }
  __syncthreads();
  if (spikes_zero != nullptr) {
    // the integration kernel ORs this step's spikes into the tile's (contiguous) spike rows: clear them here
    uint4* z = reinterpret_cast<uint4*>(spikes_zero + a0 * spike_ld);
    for (long long w = threadIdx.x; w < (long long)na * spike_ld / 4; w += blockDim.x) z[w] = make_uint4(0u, 0u, 0u, 0u);
  }
  float* tile = scratch + (size_t)blockIdx.x * bc.T * BVC_AT;
  float cmax = 1.f, lmax = 0.f;                         // error floors of the float32 screens (riab_bvc.cuh)
  for (int w = 0; w < env.W; ++w) {
    const float4 wl = s_wf[w];
    cmax = fmaxf(cmax, fmaxf(fmaxf(fabsf(wl.x), fabsf(wl.y)), fmaxf(fabsf(wl.x + wl.z), fabsf(wl.y + wl.w))));
    lmax = fmaxf(lmax, fabsf(wl.z) + fabsf(wl.w));
  }
  if (TABLE) {
    // (angle, wall) table + float32 directions, then one agent per thread for all its angles (idx & 31 is constant)
    float2* s_dirf = reinterpret_cast<float2*>(s_dirs + 2 * bc.T);
    BvcTab* s_tab = reinterpret_cast<BvcTab*>(s_dirf + bc.T);
    const int W = env.W;
    for (int e = threadIdx.x; e < bc.T * W; e += blockDim.x) {
      const int th = e / W, w = e - th * W;
      s_tab[e] = bvc_table_entry(s_dirs[2 * th], s_dirs[2 * th + 1], s_walls + 4 * w, cmax);
    }
    for (int th = threadIdx.x; th < bc.T; th += blockDim.x) s_dirf[th] = make_float2((float)s_dirs[2 * th], (float)s_dirs[2 * th + 1]);
    __syncthreads();
    const int a = threadIdx.x & 31;
    const double px = s_pos[a][0], py = s_pos[a][1];
    const float pxf = (float)px, pyf = (float)py;
    const float ka = 1e-9f * cmax * lmax;
    float numA[BVC_NW];
#pragma unroll
    for (int w = 0; w < BVC_NW; ++w) {
      numA[w] = 0.f;
      if (w < W) {
        const double ax = s_walls[4 * w], ay = s_walls[4 * w + 1];
        numA[w] = (float)((ax - px) * (s_walls[4 * w + 3] - ay) - (ay - py) * (s_walls[4 * w + 2] - ax));   // (a - p) x sb
      }
    }
    for (int th = threadIdx.x >> 5; th < bc.T; th += NT / 32) {
      const float2 u = s_dirf[th];
      uint32_t mask = bvc_table_mask<BVC_NW>(s_tab + th * W, numA, W, pxf * u.y - pyf * u.x, ka);
      if (!(fabsf(pxf) + fabsf(pyf) <= 4.f * cmax)) mask = 0xffffffffu >> (32 - W);   // far outside (or NaN): no screen
      double d;
      int wid;
      bvc_walk<uint32_t>(mask, px, py, s_dirs[2 * th], s_dirs[2 * th + 1], s_walls, d, wid);
      tile[th * BVC_AT + a] = (float)d;
      if (first_wall != nullptr && a < na) first_wall[(a0 + a) * bc.T + th] = wid;
    }
    return;
  }
  const float flo_env = 1e-6f * cmax * lmax;
  for (int idx = threadIdx.x; idx < bc.T * BVC_AT; idx += blockDim.x) {
    const int th = idx >> 5, a = idx & 31;
    double d;
    int wid;
    bvc_first_wall(s_pos[a][0], s_pos[a][1], s_dirs[2 * th], s_dirs[2 * th + 1], s_walls, s_wf, env.W, flo_env, d, wid);
    tile[idx] = (float)d;
    if (first_wall != nullptr && a < na) first_wall[(a0 + a) * bc.T + th] = wid;
  }
}

// BVC phase B: grid.x = cell tiles, grid.y = agent-tile lanes; 256 threads:
// cell = tid & 63, agent group g = tid >> 6 handles agents 8g..8g+7 of the tile.
// Neurons.save_to_history spikes (Neurons.py:681-684) of one cell for 8 consecutive agents (rows r0 .. r0+7, r0 even, even
// shard offset), the dense stream of spike_words / spike_ballots: one Philox4x32-7 call per (agent pair, 4-cell group) --
// every thread of a group repeats it for its own cell, 4 calls per 180 x 8 integrand terms -- and RED.OR into the rows
// k_bvc_rays cleared.
__device__ __forceinline__ void bvc_spikes8(const OutK& out, const float (&v)[8], const long long r0, const long long n_rows,
                                            const int cell) {
  const int i = cell & 3;
  const uint32_t sub = (uint32_t)(cell >> 2);
  const uint32_t hi = ((uint32_t)(out.step >> 32) & 0xffffu) | (((uint32_t)out.pop & 0xffu) << 16) | (RIAB_STREAM_SPIKES << 24);
  const float q16 = out.dt * 65536.0f;
  const uint32_t bit = 1u << ((cell >> 2) & 31);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const long long row = r0 + 2 * k;
    if (row >= n_rows) break;
    const unsigned long long pair = (unsigned long long)(out.id_offset + row) >> 1;
    uint32_t c[4];
    c[0] = (uint32_t)pair; c[1] = sub ^ ((uint32_t)(pair >> 32) << 24); c[2] = (uint32_t)out.step; c[3] = hi;
    philox_keyed<7>(c, out.rk7);
    const float nv = spike_neg_dither(c);
    const uint32_t wa = (i < 2) ? c[0] : c[1], wb = (i < 2) ? c[2] : c[3];
    const float ma = (float)((wa >> (16 * (i & 1))) & 0xffffu), mb = (float)((wb >> (16 * (i & 1))) & 0xffffu);
    uint32_t* w = out.spikes + row * out.spike_ld + ((cell >> 7) << 2) + i;
    if (ma < fmaf(v[2 * k], q16, nv)) atomicOr(w, bit);
    if (row + 1 < n_rows && mb < fmaf(v[2 * k + 1], q16, nv)) atomicOr(w + out.spike_ld, bit);
  }
}

__global__ void __launch_bounds__(NT) k_bvc_integrate(const BvcConst bc, const float* __restrict__ scratch,
                                                      const long long n_rows, const long long n_tiles,
                                                      const OutK out, const int fold_spikes) {
  extern __shared__ __align__(128) unsigned char dyn[];
  const int T = bc.T;
  float* s_vm = reinterpret_cast<float*>(dyn);                     // [T][64]
  float* s_d0 = s_vm + (size_t)T * BVC_CT;                         // [T][32] x 2 buffers
  float* s_d1 = s_d0 + (size_t)T * BVC_AT;
  __shared__ uint64_t bar_vm, bar_d[2];
  const int ct = blockIdx.x;
  const int tid = threadIdx.x, cl = tid & 63, g = tid >> 6;
  const int slot = ct * BVC_CT + cl;
  // slot -> cell and this warp's angular window (riab_bvc_pack): outside [th0, th0 + tlen) mod T all 32 von Mises weights
  // are < 2^-30 of their peak
  const int32_t* perm = reinterpret_cast<const int32_t*>(bc.packed + 6 * (size_t)bc.n_pad + (size_t)bc.n_pad * T + 2 * (size_t)T);
  const int cell = perm[slot];
  const int th0 = perm[bc.n_pad + 2 * (slot >> 5)], tlen = perm[bc.n_pad + 2 * (slot >> 5) + 1];
  const uint32_t vm_bytes = (uint32_t)T * BVC_CT * 4u, d_bytes = (uint32_t)T * BVC_AT * 4u;
  const float* vm_src = bc.packed + 3 * (size_t)bc.n_pad + (size_t)ct * T * BVC_CT;
  if (tid == 0) {
    mbar_init(&bar_vm, 1); mbar_init(&bar_d[0], 1); mbar_init(&bar_d[1], 1);
    mbar_fence_init();
    mbar_expect_tx(&bar_vm, vm_bytes);
    tma_bulk_g2s(s_vm, vm_src, vm_bytes, &bar_vm);
    long long t0 = blockIdx.y;
    if (t0 < n_tiles) { mbar_expect_tx(&bar_d[0], d_bytes); tma_bulk_g2s(s_d0, scratch + (size_t)t0 * T * BVC_AT, d_bytes, &bar_d[0]); }
  }
  __syncthreads();
  const float sc = bc.packed[cell], mc = bc.packed[bc.n_pad + cell], scale = bc.packed[2 * bc.n_pad + cell];
  mbar_wait(&bar_vm, 0);
  uint32_t phase[2] = {0u, 0u};
  int buf = 0;
  for (long long t = blockIdx.y; t < n_tiles; t += gridDim.y, buf ^= 1) {
    const long long tn = t + gridDim.y;
    if (tid == 0 && tn < n_tiles) {          // prefetch the next agent tile into the other buffer
      mbar_expect_tx(&bar_d[buf ^ 1], d_bytes);
      tma_bulk_g2s(buf ? s_d0 : s_d1, scratch + (size_t)tn * T * BVC_AT, d_bytes, &bar_d[buf ^ 1]);
    }
    mbar_wait(&bar_d[buf], phase[buf]);
    phase[buf] ^= 1u;
    const float* sd = (buf ? s_d1 : s_d0) + 8 * g;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    // the window [th0, th0 + tlen) mod T as two plain segments (no wrap test in the loop); 4 angles in flight per thread:
    // the loop is bound by MUFU.EX2 (one warp instruction per 8 cycles), whose queue has to be kept fed across the
    // LDS -> FFMA -> FMUL head of every angle
    const int n0 = min(tlen, T - th0);
#pragma unroll 1
    for (int seg = 0; seg < 2; ++seg) {
      const int tb = seg ? 0 : th0, tn = seg ? tlen - n0 : n0;
      const float* pv = s_vm + tb * BVC_CT + cl;
      const float* pd = sd + tb * BVC_AT;
#pragma unroll 4
      for (int j = 0; j < tn; ++j, pv += BVC_CT, pd += BVC_AT) {
        const float vm = *pv;
        const float4 da = *reinterpret_cast<const float4*>(pd);
        const float4 db = *reinterpret_cast<const float4*>(pd + 4);
        const float dv[8] = {da.x, da.y, da.z, da.w, db.x, db.y, db.z, db.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float u = fmaf(dv[i], sc, -mc);                    // (d - mu_d) * s
          // gaussian * von Mises.  Moving some of the eight exponentials to an 11-instruction FMA-pipe polynomial gained
          // in one build and lost in another (register allocation of the unrolled loop decides): all eight stay on MUFU.
          const float e = ex2f(-u * u);
          acc[i] = fmaf(e, vm, acc[i]);
        }
      }
    }
    if (cell < bc.n_cells) {
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const long long row = t * BVC_AT + 8 * g + i;
        // a NaN position makes every distance NaN: the reference returns zero rates for it (Neurons.py:163-164)
        v[i] = (acc[i] != acc[i]) ? 0.f : fmaf(acc[i] * scale, bc.span, bc.min_fr);
        if (row < n_rows) st_cs_f1(out.rates + row * out.ld + cell, v[i]);
      }
      if (fold_spikes) bvc_spikes8(out, v, t * BVC_AT + 8 * g, n_rows, cell);
    }
    __syncthreads();   // everyone done with this buffer before it is refilled two iterations later
  }
}

// BVC phase B, egocentric frame: same tiling as k_bvc_integrate, no von Mises table.
__global__ void __launch_bounds__(NT) k_bvc_integrate_ego(const BvcConst bc, const float* __restrict__ scratch,
                                                          const long long n_rows, const long long n_tiles,
                                                          const OutK out, const int fold_spikes) {
  extern __shared__ __align__(128) unsigned char dyn[];
  const int T = bc.T;
  float2* s_th = reinterpret_cast<float2*>(dyn);                    // [T] (cos, sin) of the test angles
  float* s_d0 = reinterpret_cast<float*>(dyn) + 2 * (size_t)((T + 1) / 2 * 2);   // [T][32] x 2 buffers
  float* s_d1 = s_d0 + (size_t)T * BVC_AT;
  __shared__ uint64_t bar_d[2];
  const int ct = blockIdx.x;
  const int tid = threadIdx.x, cl = tid & 63, g = tid >> 6;
  const int cell = ct * BVC_CT + cl;
  const uint32_t d_bytes = (uint32_t)T * BVC_AT * 4u;
  const float* base = bc.packed;
  const size_t np = (size_t)bc.n_pad;
  const float* ext = base + 3 * np + np * (size_t)T;               // kap | cmu | smu | cth | sth
  for (int i = tid; i < T; i += blockDim.x) s_th[i] = make_float2(ext[3 * np + i], ext[3 * np + T + i]);
  if (tid == 0) {
    mbar_init(&bar_d[0], 1); mbar_init(&bar_d[1], 1);
    mbar_fence_init();
    long long t0 = blockIdx.y;
    if (t0 < n_tiles) { mbar_expect_tx(&bar_d[0], d_bytes); tma_bulk_g2s(s_d0, scratch + (size_t)t0 * T * BVC_AT, d_bytes, &bar_d[0]); }
  }
  __syncthreads();
  const float sc = base[cell], mc = base[np + cell], scale = base[2 * np + cell];
  const float kap = ext[cell], cmu = ext[np + cell], smu = ext[2 * np + cell];
  uint32_t phase[2] = {0u, 0u};
  int buf = 0;
  for (long long t = blockIdx.y; t < n_tiles; t += gridDim.y, buf ^= 1) {
    const long long tn = t + gridDim.y;
    if (tid == 0 && tn < n_tiles) {
      mbar_expect_tx(&bar_d[buf ^ 1], d_bytes);
      tma_bulk_g2s(buf ? s_d0 : s_d1, scratch + (size_t)tn * T * BVC_AT, d_bytes, &bar_d[buf ^ 1]);
    }
    // (cos, sin)(head bearing + mu_theta) for this thread's 8 agents
    float cph[8], sph[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const long long row = t * BVC_AT + 8 * g + i;
      float hx = 1.0f + 1e-6f, hy = 0.f;                            // default head direction [1,0] (Neurons.py:1703)
      if (bc.head_dir != nullptr && row < n_rows) {
        hx = (float)(bc.head_dir[2 * row] + 1e-6);                  // utils.get_angle: atan2(y, x + eps)
        hy = (float)bc.head_dir[2 * row + 1];
      }
      const float rn = rsqrtf(fmaf(hx, hx, hy * hy));
      const float ch = hx * rn, sh = hy * rn;
      cph[i] = fmaf(-sh, smu, ch * cmu);
      sph[i] = fmaf(ch, smu, sh * cmu);
    }
    mbar_wait(&bar_d[buf], phase[buf]);
    phase[buf] ^= 1u;
    const float* sd = (buf ? s_d1 : s_d0) + 8 * g;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll 2
    for (int th = 0; th < T; ++th) {
      const float2 cs = s_th[th];
      const float4 da = *reinterpret_cast<const float4*>(sd + th * BVC_AT);
      const float4 db = *reinterpret_cast<const float4*>(sd + th * BVC_AT + 4);
      const float dv[8] = {da.x, da.y, da.z, da.w, db.x, db.y, db.z, db.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float u = fmaf(dv[i], sc, -mc);                       // (d - mu_d) * s
        const float c = fmaf(cs.y, sph[i], cs.x * cph[i]);          // cos(theta - bearing - mu_theta)
        acc[i] += ex2f(fmaf(kap, c - 1.0f, -u * u));                // gaussian * von Mises in one ex2
      }
    }
    if (cell < bc.n_cells) {
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const long long row = t * BVC_AT + 8 * g + i;
        // a NaN position makes every distance NaN: the reference returns zero rates for it (Neurons.py:163-164)
        v[i] = (acc[i] != acc[i]) ? 0.f : fmaf(acc[i] * scale, bc.span, bc.min_fr);
        if (row < n_rows) st_cs_f1(out.rates + row * out.ld + cell, v[i]);
      }
      if (fold_spikes) bvc_spikes8(out, v, t * BVC_AT + 8 * g, n_rows, cell);
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// History analytics: occupancy and rate-weighted histograms of the agents' positions (utils.py:544-589).
// np.histogram2d with explicit edges: bin = searchsorted(edges, x, 'right') - 1, the right-most edge belongs to
// the last bin, samples outside are dropped.  Counts are 64-bit integers and rate sums float64: a default Agent ring of
// 65 536 agents holds 2^26 samples, a float32 count stops at 2^24 and a float32 running sum of millions of rates drifts
// by about 1e-2 relative, while any order of a float64 sum of n float32 rates agrees to about n * 2^-53 relative.
__device__ __forceinline__ int hist_bin(const double* __restrict__ e, int n_edges, double x) {
  if (!(x >= e[0]) || !(x <= e[n_edges - 1])) return -1;
  if (x == e[n_edges - 1]) return n_edges - 2;
  int lo = 0, hi = n_edges;                       // first edge > x
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (e[mid] <= x) lo = mid + 1; else hi = mid;
  }
  return lo - 1;
}
__global__ void __launch_bounds__(NT) k_history_maps(const riab_history_view h, const double* __restrict__ ex, int nex,
                                                     const double* __restrict__ ey, int ney, double* __restrict__ sum,
                                                     unsigned long long* __restrict__ count) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (NT / 32);
  const long long n_samples = h.n_steps * h.n_agents;
  const int ny = ney - 1;
  for (long long w = (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5); w < n_samples; w += warps) {
    const long long step = w / h.n_agents, agent = w - step * h.n_agents;
    const long long arow = (h.agent_row0 + step) % h.agent_ring_rows;
    const float* p = h.agent_ring + (arow * h.n_agents + agent) * 8;
    const int ix = hist_bin(ex, nex, (double)p[0]), iy = hist_bin(ey, ney, (double)p[1]);
    if (ix < 0 || iy < 0) continue;                              // warp-uniform
    const long long bin = (long long)ix * ny + iy;
    if (lane == 0) atomicAdd(count + bin, 1ull);
    if (h.rates_ring != nullptr) {
      const long long rrow = (h.rates_row0 + step) % h.rates_ring_rows;
      const float* r = h.rates_ring + (rrow * h.n_agents + agent) * h.ld;
      double* dst = sum + bin * h.ld;
      for (int c = lane; c < h.n_cells; c += 32) atomicAdd(dst + c, (double)r[c]);
    }
  }
}

// ---------------------------------------------------------------------------
// host helpers
int make_env(const riab_env* env, EnvK& k) {
  if (env == nullptr || (env->walls_dev == nullptr && env->n_walls > 0)) return fail(RIAB_ERR_INVALID, "env / walls_dev is NULL");
  if (env->n_walls < 0 || env->n_walls > RIAB_MAX_WALLS)
    return fail(RIAB_ERR_UNSUPPORTED, "n_walls=%d exceeds %d", env->n_walls, RIAB_MAX_WALLS);
  if (env->n_boundary_walls < 0 || env->n_boundary_walls > env->n_walls)
    return fail(RIAB_ERR_INVALID, "n_boundary_walls=%d out of range", env->n_boundary_walls);
  k.walls = env->walls_dev; k.W = env->n_walls; k.nb = env->n_boundary_walls;
  k.aligned = (((uintptr_t)env->walls_dev) % 16 == 0) && env->n_walls > 0;
  for (int i = 0; i < 4; ++i) k.ext[i] = env->extent[i];
  k.cxm = 0.5 * (env->extent[0] + env->extent[1]);
  k.cym = 0.5 * (env->extent[2] + env->extent[3]);
  if (env->boundary_mode < 0 || env->boundary_mode > RIAB_BOUNDARY_POLYGON) return fail(RIAB_ERR_INVALID, "bad boundary_mode %d", env->boundary_mode);
  k.periodic = env->boundary_mode == RIAB_BOUNDARY_PERIODIC_BOX ? 1 : 0;
  k.polygon = env->boundary_mode == RIAB_BOUNDARY_POLYGON ? 1 : 0;
  k.nh = k.polygon ? env->n_hole_walls : 0;
  k.h0 = k.polygon ? env->hole_wall0 : 0;
  if (k.nh < 0 || k.h0 < 0 || (k.nh > 0 && (k.h0 < k.nb || k.h0 + k.nh > k.W)))
    return fail(RIAB_ERR_INVALID, "hole walls [%d, %d) out of range", env->hole_wall0, env->hole_wall0 + env->n_hole_walls);
  if (k.polygon && k.nb < 3) return fail(RIAB_ERR_INVALID, "a polygon boundary needs at least 3 boundary walls");
  k.scale = env->scale;
  if (k.periodic && !(env->scale > 0.0)) return fail(RIAB_ERR_INVALID, "periodic environment needs scale > 0");
  return 0;
}

// Dynamic shared memory of the motion kernels: every wall in float64
size_t motion_walls_bytes(const EnvK& env) { return (size_t)env.W * 4 * sizeof(double); }

// Whether the motion step can run inside a rate kernel (k_step MODE 1 / 2 / 3 / 4), whose static wall block holds MAXW
// walls; with more, the stand-alone motion kernel takes every step.
bool step_kernel_walls(const EnvK& env) { return env.W <= MAXW; }

// The environment without its walls, for rate kernels that read none: k_step MODE 0 and k_place_onehot then stage
// nothing, whatever the wall count.
EnvK without_walls(const EnvK& env) {
  EnvK k = env;
  k.walls = nullptr; k.W = 0; k.nb = 0; k.nh = 0; k.h0 = 0; k.aligned = 0;
  return k;
}

int check_agents(const riab_agents* a) {
  if (a == nullptr) return fail(RIAB_ERR_INVALID, "agents is NULL");
  if (a->n_agents < 0) return fail(RIAB_ERR_INVALID, "n_agents < 0");
  if (a->n_agents > 0 && (!a->pos || !a->velocity || !a->rotational_velocity || !a->measured_velocity ||
                          !a->measured_rotational_velocity || !a->head_direction || !a->distance_travelled ||
                          !a->distance_to_closest_wall))
    return fail(RIAB_ERR_INVALID, "agents: NULL state array");
  return 0;
}

int check_motion(const riab_motion_params* p) {
  if (p == nullptr) return fail(RIAB_ERR_INVALID, "motion params NULL");
  if (!(p->dt > 0.0)) return fail(RIAB_ERR_INVALID, "dt must be > 0");
  return 0;
}

// fr_bound: an upper bound of the population's rates (thinned spikes), negative when there is none
int make_out(const riab_rates_out* o, const riab_neuron_noise* nz, int n_cells, double dt, long long id_offset, OutK& k,
             double fr_bound = -1.0) {
  if (o == nullptr || o->rates_row == nullptr) return fail(RIAB_ERR_INVALID, "rates_row is NULL");
  if (o->ld < n_cells) return fail(RIAB_ERR_INVALID, "ld (%lld) < n_cells (%d)", (long long)o->ld, n_cells);
  memset(&k, 0, sizeof(k));
  k.rates = o->rates_row; k.ld = o->ld;
  k.spikes = o->spikes_row; k.spike_ld = 4 * ((n_cells + 127) / 128);     // 4 ballot words per 128 cells
  if (k.spikes != nullptr && (((uintptr_t)k.spikes) % 16 != 0)) return fail(RIAB_ERR_INVALID, "spikes_row must be 16-byte aligned");
  k.noise = nullptr;
  k.dt = (float)dt;
  k.id_offset = id_offset;
  if (nz != nullptr) {
    k.seed = nz->seed; k.step = nz->step; k.pop = nz->population_id;
    if (nz->noise_std != 0.f) {
      if (o->noise_state == nullptr) return fail(RIAB_ERR_INVALID, "noise_std != 0 needs noise_state");
      k.noise = o->noise_state;
      const double tau = nz->noise_coherence_time;
      k.noise_decay = (float)(dt / tau);
      k.noise_sig = (float)(sqrt(2.0 * (double)nz->noise_std * nz->noise_std / (tau * dt)) * dt);
    }
  } else if (o->spikes_row != nullptr) {
    return fail(RIAB_ERR_INVALID, "spikes need a riab_neuron_noise (seed/step)");
  }
  k.vec_ok = (o->ld % 4 == 0) && (((uintptr_t)o->rates_row) % 16 == 0);
  {
    uint32_t k0 = (uint32_t)k.seed, k1 = (uint32_t)(k.seed >> 32);
    for (int i = 0; i < 7; ++i) { k.rk7[2 * i] = k0; k.rk7[2 * i + 1] = k1; k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
  }
  // thinned spikes (thin_block): p' = dt * bound * (1 + 2^-10) -- the margin covers the rates' float32 rounding above `bound`.
  // The default for bounded populations without OU noise when p' <= 1/16 (beyond that the candidates are no rarer than the
  // dense stream's work); RIAB_DENSE_SPIKES=1 in the environment keeps the dense stream everywhere.
  k.thin = 0;
  if (k.spikes != nullptr && k.noise == nullptr && fr_bound >= 0.0 && getenv("RIAB_DENSE_SPIKES") == nullptr) {
    const double bound = fr_bound * (1.0 + 1.0 / 1024.0), p = dt * bound;
    if (p > 0.0 && p <= 0.0625) {
      k.thin = 1;
      // Binomial(128, p) by the pmf recurrence, IEEE operations in this order (tests/philox_np.py: thin_tables repeats them)
      const double q = 1.0 - p, r = p / q;
      double pmf = q;
      for (int i = 0; i < 7; ++i) pmf = pmf * pmf;                       // q^128
      double cdf = 0.0;
      for (int i = 0; i < 32; ++i) {
        cdf = cdf + pmf;
        const double t = floor(4294967296.0 * cdf);
        k.thin_cdf[i] = (t >= 4294967295.0) ? 4294967295u : (uint32_t)t;
        pmf = pmf * ((double)(128 - i) * r) / (double)(i + 1);
      }
      k.thin_c1 = (float)(bound * (1.0 / 1048576.0));
      k.thin_c0 = (float)(bound * (1.0 / 2097152.0));
    }
  }
  return 0;
}

int make_place(const riab_place_cells* pc, const EnvK& env, PlaceConst& c) {
  if (pc == nullptr || pc->packed_dev == nullptr) return fail(RIAB_ERR_INVALID, "place cells / packed_dev NULL");
  if (pc->description < 0 || pc->description > RIAB_PC_ONE_HOT) return fail(RIAB_ERR_INVALID, "bad description %d", pc->description);
  if (pc->wall_geometry < 0 || pc->wall_geometry > RIAB_GEOM_GEODESIC) return fail(RIAB_ERR_INVALID, "bad wall_geometry");
  // Environment.py:715-717 hard-codes `walls[4:]`: with a polygon boundary the walls after the first FOUR count as
  // "inner" walls whatever the polygon's vertex count; the box has exactly its 4 boundary walls first
  const int skip = env.polygon ? (env.W < 4 ? env.W : 4) : env.nb;
  const int n_inner = env.W - skip;
  c.wall0 = skip;
  if (pc->wall_geometry != RIAB_GEOM_EUCLIDEAN) {
    if (pc->n_inner_walls != n_inner) return fail(RIAB_ERR_INVALID, "packed for %d inner walls, env has %d (re-pack after add_wall)", pc->n_inner_walls, n_inner);
    if (n_inner > PLACE_MAX_WI) return fail(RIAB_ERR_UNSUPPORTED, "line_of_sight supports at most %d inner walls (got %d)", PLACE_MAX_WI, n_inner);
    if (pc->centres_dev == nullptr) return fail(RIAB_ERR_INVALID, "centres_dev NULL");
    if (pc->wall_geometry == RIAB_GEOM_GEODESIC && n_inner > 1)
      return fail(RIAB_ERR_INVALID, "geodesic geometry is only defined with one additional wall (Environment.py:736-739)");
    // the reference's np.amin over the detours via the ends inside the box has nothing to reduce (Environment.py:769-773)
    if (pc->wall_geometry == RIAB_GEOM_GEODESIC && n_inner == 1 && pc->ep_valid == 0)
      return fail(RIAB_ERR_INVALID, "geodesic geometry needs an end of the additional wall strictly inside the box");
  }
  if ((pc->description == RIAB_PC_TOP_HAT || pc->description == RIAB_PC_ONE_HOT) && pc->centres_dev == nullptr)
    return fail(RIAB_ERR_INVALID, "centres_dev NULL");
  c.desc = pc->description; c.geometry = pc->wall_geometry; c.n_cells = pc->n_cells; c.n_pad = pc->n_pad;
  c.n_inner = (pc->wall_geometry == RIAB_GEOM_EUCLIDEAN) ? 0 : n_inner;
  c.ep_valid = pc->ep_valid;
  c.min_fr = pc->min_fr; c.span = pc->max_fr - pc->min_fr;
  c.top_hat_w = pc->top_hat_width; c.top_hat_w2 = (float)(pc->top_hat_width * pc->top_hat_width);
  c.band = 0.f;
  for (int j = 0; j < PLACE_MAX_WI; ++j) { c.eps[j] = pc->eps[j]; c.band = fmaxf(c.band, pc->eps[j]); }
  c.packed = pc->packed_dev; c.centres64 = pc->centres_dev;
  c.cxm = env.cxm; c.cym = env.cym;
  // expanded Gaussian (place_rates4): one common width, plain Gaussian, no wrap-around, and small enough
  // exponents at the far corner that the float32 cancellation stays below 4e-6 relative
  c.expanded = (pc->description == RIAB_PC_GAUSSIAN && pc->wall_geometry != RIAB_GEOM_GEODESIC && !env.periodic &&
                pc->k_uniform > 0.f && pc->k_uniform * pc->r2_max <= 10.0f) ? 1 : 0;
  c.kx = -pc->k_uniform;
  c.fold = (c.expanded && pc->min_fr == 0.f && c.span > 0.f) ? 1 : 0;
  c.lspan = c.fold ? log2f(c.span) : 0.f;
  // The direct form rounds p' and c' to float32 separately, |d_f - d| ~ 2^-24 (|p'| + |c'|): a relative rate error of
  // ~ d |d_f - d| / w^2, 2.5e-5 at 3.7 w with w = 0.05 in a 10 m box and near 1e-5 already at w = 0.05 in the unit box.
  // Every direct-form launch therefore takes the compensated kernels, geodesic included: its record holds the agent ->
  // wall-end distances in a block of their own (place_geo), so ep0 / ep1 carry the residuals there too.
  c.comp = (!c.expanded && pc->description != RIAB_PC_ONE_HOT) ? 1 : 0;
  c.periodic = env.periodic; c.scale = env.scale; c.scale_f = (float)env.scale; c.half_f = (float)(env.scale / 2);
  c.scale_lo = (float)(env.scale - (double)c.scale_f);
  {
    // Float32 error of a centre -> position distance, |d_f - d| <= 2^-23 (|p'|_1 + |c'|_1 [+ 2 scale when wrapped]):
    // each coordinate is rounded once (2^-24 |.|), the difference once more (2^-24 |dx| <= 2^-24 (|p'x| + |c'x|)), and
    // the wrap adds the rounding of scale and of scale - dx.  |c'|_1 <= sqrt(2 r2_max).
    const double u = 1.1920928955078125e-07;                          // 2^-23
    const double c1 = sqrt(2.0 * (double)pc->r2_max), per = env.periodic ? 2.0 * env.scale : 0.0;
    c.coord_err = (float)(u * (c1 + per) * 1.001);                     // one_hot adds its row's |p'|_1 (k_place_onehot)
    // top_hat: d^2 near w^2 is known to within 2 w E + E^2 + 2^-23 w^2, with |p'|_1 <= |c'|_1 + sqrt(2) w on the edge;
    // pairs inside twice that band take the float64 distance (the scale-1 band 4e-6 (w^2 + 1e-3) stays the floor)
    const double w = pc->top_hat_width, E = u * (2.0 * c1 + 1.4142135623730951 * w + per);
    c.top_hat_band = (float)fmax(4e-6 * (w * w + 1e-3), 2.0 * (2.0 * w * E + E * E + u * w * w));
  }
  if (env.periodic && pc->wall_geometry != RIAB_GEOM_EUCLIDEAN)
    return fail(RIAB_ERR_INVALID, "line_of_sight / geodesic wall geometry only possible when the boundary conditions are solid (Neurons.py:907-921)");
  return 0;
}

int make_grid(const riab_grid_cells* gc, const EnvK& env, GridConst& c) {
  if (gc == nullptr || gc->packed_dev == nullptr) return fail(RIAB_ERR_INVALID, "grid cells / packed_dev NULL");
  c.n_cells = gc->n_cells; c.n_pad = gc->n_pad;
  if (gc->description == RIAB_GC_RECTIFIED_COSINES) {
    if (!(gc->width_ratio > 0.0 && gc->width_ratio <= 1.0)) return fail(RIAB_ERR_INVALID, "width_ratio must be between 0 and 1");
    const double full = (1.0 / 3.0) * (2.0 * cos(sqrt(3.0) * M_PI * gc->width_ratio / 2.0) + 1.0);   // Neurons.py:1211
    c.A = (float)((1.0 / 3.0) / (1.0 - full));
    c.B = (float)(-full / (1.0 - full));
    c.rectify = 1;
  } else if (gc->description == RIAB_GC_SHIFTED_COSINES) {
    c.A = (float)(2.0 / 9.0); c.B = (float)(1.0 / 3.0); c.rectify = 0;                                 // Neurons.py:1216-1218
  } else return fail(RIAB_ERR_INVALID, "bad grid description %d", gc->description);
  c.min_fr = gc->min_fr; c.span = gc->max_fr - gc->min_fr;
  c.As = c.A * c.span; c.Bs = fmaf(c.B, c.span, c.min_fr);
  c.clamp = c.rectify ? (c.span >= 0.f ? 1 : 2) : 0;
  c.packed = gc->packed_dev; c.cxm = env.cxm; c.cym = env.cym;
  c.turns = gc->phase_turns ? 1 : 0;
  return 0;
}

int make_ovc(const riab_ovc_cells* oc, const EnvK& env, const double* head_dir, OvcConst& c) {
  if (oc == nullptr || oc->packed_dev == nullptr) return fail(RIAB_ERR_INVALID, "object vector cells / packed_dev NULL");
  if (oc->n_objects < 0 || oc->n_objects > RIAB_MAX_OBJECTS)
    return fail(RIAB_ERR_UNSUPPORTED, "n_objects=%d exceeds %d", oc->n_objects, RIAB_MAX_OBJECTS);
  if (env.periodic) return fail(RIAB_ERR_UNSUPPORTED, "object vector cells need solid boundary conditions here");
  memset(&c, 0, sizeof(c));
  c.n_cells = oc->n_cells; c.n_pad = oc->n_pad; c.n_obj = oc->n_objects;
  c.ego = oc->egocentric ? 1 : 0; c.occlude = oc->walls_occlude ? 1 : 0;
  c.wall0 = env.W < 4 ? env.W : 4;                       // Environment.py:715-717: walls[4:]
  c.n_inner = env.W - c.wall0;
  c.min_fr = oc->min_fr; c.span = oc->max_fr - oc->min_fr;
  c.packed = oc->packed_dev; c.head_dir = head_dir;
  for (int o = 0; o < oc->n_objects; ++o) {
    c.obj[2 * o] = oc->objects[2 * o]; c.obj[2 * o + 1] = oc->objects[2 * o + 1];
    c.type[o] = (float)oc->object_types[o];
  }
  return 0;
}

// Kinematic cells at the agents: the vector their variant reads, one per agent (Neurons.py:2430, :2448, :2642).
int make_kin(const riab_kin_cells* kc, const riab_agents& ag, KinConst& c) {
  if (kc == nullptr || kc->packed_dev == nullptr) return fail(RIAB_ERR_INVALID, "kinematic cells / packed_dev NULL");
  if (kc->variant < RIAB_KIN_HEAD_DIRECTION || kc->variant > RIAB_KIN_SPEED) return fail(RIAB_ERR_INVALID, "bad kinematic variant %d", kc->variant);
  if (kc->n_cells <= 0 || kc->n_pad != (kc->n_cells + CELL_PAD - 1) / CELL_PAD * CELL_PAD)
    return fail(RIAB_ERR_INVALID, "kinematic cells: n_cells %d / n_pad %d (pack with riab_kin_pack)", kc->n_cells, kc->n_pad);
  if (((uintptr_t)kc->packed_dev) % 16 != 0) return fail(RIAB_ERR_INVALID, "kinematic cells: packed_dev must be 16-byte aligned");
  memset(&c, 0, sizeof(c));
  c.n_cells = kc->n_cells; c.n_pad = kc->n_pad; c.variant = kc->variant;
  c.use_vel = (kc->variant == RIAB_KIN_VELOCITY || kc->use_velocity) ? 1 : 0;
  c.min_fr = kc->min_fr; c.span = kc->max_fr - kc->min_fr;
  c.inv_oss = kc->inv_one_sigma_speed;
  c.fixed_scale = -1.0;
  c.packed = kc->packed_dev;
  c.vec = kc->variant == RIAB_KIN_SPEED ? ag.measured_velocity : (c.use_vel ? ag.velocity : ag.head_direction);
  c.vec_ld = 2;
  return 0;
}

// AgentVectorCells over n_rows rows (the agents, or get_state's positions): the partner of each row (riab_avc_cells).
int make_avc(const riab_avc_cells* vc, const EnvK& env, const double* head_dir, long long n_rows, AvcConst& c) {
  if (vc == nullptr || vc->packed_dev == nullptr) return fail(RIAB_ERR_INVALID, "agent vector cells / packed_dev NULL");
  if (vc->n_cells <= 0 || vc->n_pad != (vc->n_cells + CELL_PAD - 1) / CELL_PAD * CELL_PAD)
    return fail(RIAB_ERR_INVALID, "agent vector cells: n_cells %d / n_pad %d (pack with riab_avc_pack)", vc->n_cells, vc->n_pad);
  if (((uintptr_t)vc->packed_dev) % 16 != 0) return fail(RIAB_ERR_INVALID, "agent vector cells: packed_dev must be 16-byte aligned");
  if (env.periodic) return fail(RIAB_ERR_UNSUPPORTED, "agent vector cells need solid boundary conditions here");
  const bool partner = vc->partner_is_self == 0 && vc->other_pos_dev != nullptr;
  if (partner && vc->n_other != 1 && vc->n_other != n_rows)
    return fail(RIAB_ERR_INVALID, "agent vector cells: %lld partner rows for %lld rows (pair row by row, or one partner)",
                (long long)vc->n_other, n_rows);
  memset(&c, 0, sizeof(c));
  c.n_cells = vc->n_cells; c.n_pad = vc->n_pad;
  c.ego = vc->egocentric ? 1 : 0; c.occlude = vc->walls_occlude ? 1 : 0; c.self = vc->partner_is_self ? 1 : 0;
  c.wall0 = env.W < 4 ? env.W : 4;                       // Environment.py:715-717: walls[4:]
  c.n_inner = env.W - c.wall0;
  const bool none = !c.self && vc->other_pos_dev == nullptr;
  c.min_fr = none ? 0.f : vc->min_fr; c.span = none ? 0.f : vc->max_fr - vc->min_fr;   // no partner: zeros (Neurons.py:2231)
  c.packed = vc->packed_dev; c.head_dir = head_dir;
  c.other = c.self ? nullptr : vc->other_pos_dev;
  c.other_ld = (vc->n_other == 1) ? 0 : 2;
  return 0;
}

// PhasePrecessingPlaceCells at the clock pc->t: the place constants in their direct form, and the launch's theta phase
// and von Mises constants in float64, in the reference's operation order (PhasePrecessingPlaceCells.py:100-117,
// utils.py:452-456).  vel: the rows' velocities.
int make_pppc(const riab_pppc_cells* pc, const EnvK& env, const double* vel, PppcConst& c) {
  if (pc == nullptr) return fail(RIAB_ERR_INVALID, "phase precessing place cells NULL");
  memset(&c, 0, sizeof(c));
  int rc;
  if ((rc = make_place(&pc->place, env, c))) return rc;
  if (pc->place.description == RIAB_PC_ONE_HOT)
    return fail(RIAB_ERR_INVALID, "phase precessing place cells need a description with widths (not one_hot)");
  if (!(std::isfinite(pc->theta_freq) && pc->theta_freq != 0.0) || !(std::isfinite(pc->sigma) && pc->sigma > 0.0) ||
      !std::isfinite(pc->precess_fraction) || !std::isfinite(pc->t))
    return fail(RIAB_ERR_INVALID, "phase precessing place cells: theta_freq %g, sigma %g, precess_fraction %g, t %g",
                pc->theta_freq, pc->sigma, pc->precess_fraction, pc->t);
  c.expanded = 0; c.fold = 0; c.lspan = 0.f;                          // the direct form of the DESC = -1 kernels
  c.comp = 1;                                                          // compensated (make_place)
  const double period = 1.0 / pc->theta_freq;
  double r = fmod(pc->t, period);                                      // Python's t % period: the sign of the divisor
  if (r != 0.0 && ((r < 0.0) != (period < 0.0))) r += period;
  const double phi = pc->theta_freq * r * 2.0 * M_PI;
  c.u = (float)((M_PI - phi) / (2.0 * M_PI));
  const double kappa = 1.0 / (pc->sigma * pc->sigma);
  double norm = exp(kappa) / (2.0 * M_PI * std::cyl_bessel_i(0.0, kappa));
  norm = norm / exp(kappa);
  c.k2 = (float)(kappa * 1.4426950408889634);
  c.lnorm = (float)log2(norm * 2.0 * M_PI);
  const double m = (pc->place.description == RIAB_PC_GAUSSIAN) ? 2.0 : 1.0;   // gaussian fields end at 2 sigma (:104-105)
  c.gs = pc->precess_fraction / (2.0 * m) * sqrt(2.0 / 1.4426950408889634);
  c.vel = vel;
  return 0;
}

// PlaneWaveNeurons: rate = 0.5 (cos phi + 1) span + min_fr = As cos phi + Bs (PlaneWaveNeurons.py:85-89)
int make_pwn(const riab_pwn_cells* pw, PwnConst& c) {
  if (pw == nullptr || pw->packed_dev == nullptr) return fail(RIAB_ERR_INVALID, "plane wave neurons / packed_dev NULL");
  if (pw->n_cells <= 0 || pw->n_pad != (pw->n_cells + CELL_PAD - 1) / CELL_PAD * CELL_PAD)
    return fail(RIAB_ERR_INVALID, "plane wave neurons: n_cells %d / n_pad %d (pack with riab_pwn_pack)", pw->n_cells, pw->n_pad);
  if (((uintptr_t)pw->packed_dev) % 16 != 0) return fail(RIAB_ERR_INVALID, "plane wave neurons: packed_dev must be 16-byte aligned");
  memset(&c, 0, sizeof(c));
  c.n_cells = pw->n_cells; c.n_pad = pw->n_pad;
  const double half = 0.5 * ((double)pw->max_fr - (double)pw->min_fr);
  c.As = (float)half; c.Bs = (float)(half + (double)pw->min_fr);
  c.packed = pw->packed_dev;
  c.turns = pw->phase_turns ? 1 : 0;
  return 0;
}

// The current device's SM count, cached per device ordinal (a process may drive several GPUs)
int num_sms(int& sms) {
  static int sms_of[64] = {0};
  int dev = 0;
  RIAB_CUDA_OK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return fail(RIAB_ERR_UNSUPPORTED, "device ordinal %d", dev);
  if (sms_of[dev] == 0) RIAB_CUDA_OK(cudaDeviceGetAttribute(&sms_of[dev], cudaDevAttrMultiProcessorCount, dev));
  sms = sms_of[dev];
  return 0;
}

// The noise / spike post-pass (k_finish_rows) over n_rows rows, when out has either
int finish_rows(const OutK& out, int n_cells, long long n_rows, cudaStream_t s) {
  if (out.noise == nullptr && out.spikes == nullptr) return 0;
  const int np128 = (n_cells + CELL_PAD - 1) / CELL_PAD * CELL_PAD;
  k_finish_rows<<<dim3((unsigned)n_rows, (unsigned)((np128 / 4 + NT - 1) / NT)), NT, 0, s>>>(out, n_cells, np128, n_rows);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// MODE 0: rates for given positions; 1: motion -> rates (one step); 2: skewed (rates of the current
// positions, then motion for the NEXT step -- used inside riab_run); 3: the whole run (RunK); 4: the whole run following
// the motion source run->src.
template <class P, int MODE>
int launch_tile(const EnvK& env, const riab_agents& ag, const riab_motion_params& mp, const riab_step_io& io,
                const typename P::Const& pc, const OutK& out_in, const double* pos_in, long long n_rows, cudaStream_t s,
                const RunK* run_in = nullptr) {
  if (n_rows == 0) return 0;
  int sms, rc;
  if ((rc = num_sms(sms))) return rc;
  const bool spikes = out_in.spikes != nullptr, noise = out_in.noise != nullptr;
  // thinned stream: bounded rates AND a policy for which it measured faster (P::THIN); see the policies
  const bool thin = spikes && !noise && out_in.thin && P::THIN;
  // warp-role configuration (see StepCfg)
  const int cfg = (noise || thin || (spikes && !P::LIGHT)) ? 4 : (spikes ? 12 : ((P::LIGHT && MODE != 0) ? 8 : 12));
  // agents per ring slot: 32 for large batches; small ones get equal shares per (CTA, consumer group)
  OutK outk = out_in;
  {
    const int ct = pc.n_pad / 4;                                      // cell-threads of one consumer group
    const int ring = (cfg == 4) ? ring_slots<P, StepCfg<4>>() : (cfg == 8) ? ring_slots<P, StepCfg<8>>() : ring_slots<P, StepCfg<12>>();
    const long long groups = (ct > 0 && ct <= RW * 32) ? (long long)sms * lean_groups(ct, ring) : (long long)sms;
    int ta = TA;
    if (n_rows < 4ll * TA * groups) {
      const long long per = (n_rows + groups - 1) / groups;          // agents per group if every group gets one slot
      const long long rounds = (per + TA - 1) / TA;                   // slots per group
      ta = (int)((n_rows + groups * rounds - 1) / (groups * rounds));
      ta = (ta + 1) & ~1;
      if (ta < 2) ta = 2;
      if (ta > TA) ta = TA;
    }
    outk.tile_agents = ta;
  }
  const OutK& out = outk;
  RunK run;
  memset(&run, 0, sizeof(run));
  if (run_in != nullptr) run = *run_in;
  const long long n_tiles = (n_rows + out.tile_agents - 1) / out.tile_agents;
  const unsigned grid = (unsigned)(n_tiles < sms ? n_tiles : sms);
  MotionDerived md;
  memset(&md, 0, sizeof(md));
  if (MODE != 0) derive_motion(mp, md);
  if (noise) k_step<P, MODE, 1, true, StepCfg<4>><<<grid, StepCfg<4>::THREADS, 0, s>>>(env, ag, mp, md, io, pc, out, pos_in, n_rows, run);
  else if (thin) {
    if constexpr (P::THIN) k_step<P, MODE, 2, false, StepCfg<4>><<<grid, StepCfg<4>::THREADS, 0, s>>>(env, ag, mp, md, io, pc, out, pos_in, n_rows, run);
  }
  else if (spikes) {
    // dense stream: light consumers (Euclidean Gaussian place cells) are producer-bound next to 4 producer warps and get 8;
    // the heavier loops keep the 104-register consumers
    using C = std::conditional_t<P::LIGHT, StepCfg<12>, StepCfg<4>>;
    auto* kern = k_step<P, MODE, 1, false, C>;
    size_t stage = 0;
    if (MODE >= 3) {
      // the whole run assembles the spike rows in shared memory (k_step): the opt-in covers the largest population the
      // lean loop takes (RW * 32 * 4 cells); the attribute belongs to the current device's function image, so it is set
      // per launch (a single process may drive several GPUs)
      RIAB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)spike_stage_bytes(ring_slots<P, C>(), RW * 32 * 4 / 32)));
      stage = (size_t)spike_stage_bytes(ring_slots<P, C>(), out.spike_ld);
    }
    kern<<<grid, C::THREADS, stage, s>>>(env, ag, mp, md, io, pc, out, pos_in, n_rows, run);
  }
  else {
    // light consumers without spikes run at the HBM write rate: fat producers (only instantiated for them)
    if constexpr (P::LIGHT && MODE != 0) k_step<P, MODE, 0, false, StepCfg<8>><<<grid, StepCfg<8>::THREADS, 0, s>>>(env, ag, mp, md, io, pc, out, pos_in, n_rows, run);
    else k_step<P, MODE, 0, false, StepCfg<12>><<<grid, StepCfg<12>::THREADS, 0, s>>>(env, ag, mp, md, io, pc, out, pos_in, n_rows, run);
  }
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// A Place-like policy (PlacePolicy, PppcPolicy) for pc's geometry, compensated-sum switch and inner walls (compile-time
// bound 0, 1, 2, 4 or 8); called with COMP = false, it first picks COMP from pc.comp.  Geodesic has one inner wall
// (make_place) and the run-time profile switch; its kernel and every other DESC = -1 kernel take the compensated form.
template <template <int, int, bool, bool> class Pol, int MODE, int DESC, bool COMP = false, class C>
int launch_walls(const EnvK& env, const riab_agents& ag, const riab_motion_params& mp, const riab_step_io& io, const C& pc,
                 const OutK& out, const double* pos_in, long long n_rows, cudaStream_t s, const RunK* run) {
  if constexpr (DESC < 0 && !COMP) {
    if (pc.geometry == RIAB_GEOM_GEODESIC)
      return launch_tile<Pol<1, DESC, true, true>, MODE>(env, ag, mp, io, pc, out, pos_in, n_rows, s, run);
    return launch_walls<Pol, MODE, DESC, true>(env, ag, mp, io, pc, out, pos_in, n_rows, s, run);
  } else {
    if constexpr (!COMP) {
      if (pc.comp) return launch_walls<Pol, MODE, DESC, true>(env, ag, mp, io, pc, out, pos_in, n_rows, s, run);
    }
    const int wi = pc.n_inner;
    if (wi == 0) return launch_tile<Pol<0, DESC, COMP, false>, MODE>(env, ag, mp, io, pc, out, pos_in, n_rows, s, run);
    if (wi == 1) return launch_tile<Pol<1, DESC, COMP, false>, MODE>(env, ag, mp, io, pc, out, pos_in, n_rows, s, run);
    if (wi == 2) return launch_tile<Pol<2, DESC, COMP, false>, MODE>(env, ag, mp, io, pc, out, pos_in, n_rows, s, run);
    if (wi <= 4) return launch_tile<Pol<4, DESC, COMP, false>, MODE>(env, ag, mp, io, pc, out, pos_in, n_rows, s, run);
    return launch_tile<Pol<8, DESC, COMP, false>, MODE>(env, ag, mp, io, pc, out, pos_in, n_rows, s, run);
  }
}

int launch_onehot(const EnvK& env, const PlaceConst& pc, const OutK& out, const double* pos, long long n_rows,
                  cudaStream_t s) {
  if (n_rows == 0) return 0;
  k_place_onehot<<<(unsigned)((n_rows + NT / 32 - 1) / (NT / 32)), NT, 0, s>>>(env, pc, pos, n_rows, out);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return finish_rows(out, pc.n_cells, n_rows, s);
}

// PlaceCells other than one_hot (launch_onehot)
template <int MODE>
int launch_place(const EnvK& env, const riab_agents& ag, const riab_motion_params& mp, const riab_step_io& io,
                 const PlaceConst& pc, const OutK& out, const double* pos_in, long long n_rows, cudaStream_t s,
                 const RunK* run) {
  // the common Gaussian profile without geodesic detours gets a compile-time specialisation
  if (pc.desc == RIAB_PC_GAUSSIAN && pc.geometry != RIAB_GEOM_GEODESIC)
    return launch_walls<PlacePolicy, MODE, RIAB_PC_GAUSSIAN>(env, ag, mp, io, pc, out, pos_in, n_rows, s, run);
  return launch_walls<PlacePolicy, MODE, -1>(env, ag, mp, io, pc, out, pos_in, n_rows, s, run);
}

// PhasePrecessingPlaceCells: the run-time description profile only, MODE 0 / 1 / 2 (no whole run)
template <int MODE>
int launch_pppc(const EnvK& env, const riab_agents& ag, const riab_motion_params& mp, const riab_step_io& io,
                const PppcConst& pc, const OutK& out, const double* pos_in, long long n_rows, cudaStream_t s) {
  static_assert(MODE <= 2, "phase precessing place cells have no whole-run launch");
  return launch_walls<PppcPolicy, MODE, -1>(env, ag, mp, io, pc, out, pos_in, n_rows, s, nullptr);
}

// riab_run pipelines BoundaryVectorCells across steps: the float64 ray kernel of step s+1 (latency-bound, FP64 pipe) runs
// on the caller's stream while the angular integral of step s (MUFU-bound) still runs on a side stream -- different pipes,
// so the two overlap almost completely.  Needs a second ray-distance buffer (steps alternate) and, per buffer, an event
// that the integral which read it has finished.  Allocentric cells only (egocentric ones read the head directions the next
// motion step overwrites).
constexpr int PIPE_POPS = 8;
struct BvcPipe {
  cudaStream_t side = nullptr;
  cudaEvent_t rays_done = nullptr, int_done[2][PIPE_POPS] = {};
  bool used[2][PIPE_POPS] = {};
  float* scratch2[PIPE_POPS] = {};
  long long step = 0;
};

int check_bvc(const EnvK& env, const riab_bvc_cells* bvc, const float* scratch, long long n_rows) {
  if (bvc == nullptr || bvc->packed_dev == nullptr || bvc->test_dirs_dev == nullptr)
    return fail(RIAB_ERR_INVALID, "bvc cells / packed_dev / test_dirs_dev NULL");
  if (scratch == nullptr) return fail(RIAB_ERR_INVALID, "bvc scratch NULL");
  if (env.periodic) return fail(RIAB_ERR_INVALID, "boundary cells only possible with solid boundary conditions (Neurons.py:1580-1582)");
  if (n_rows == 0) return 0;
  const int T = bvc->n_test_angles;
  if ((size_t)T * (BVC_CT + 2 * BVC_AT) * sizeof(float) > 220 * 1024)
    return fail(RIAB_ERR_UNSUPPORTED, "n_test_angles=%d too large for shared memory", T);
  if ((T * BVC_AT * 4) % 16 != 0 || ((uintptr_t)scratch) % 16 != 0 || ((uintptr_t)bvc->packed_dev) % 16 != 0)
    return fail(RIAB_ERR_INVALID, "bvc buffers must be 16-byte aligned");
  return 0;
}

// One BVC evaluation over n_rows rows, checked by check_bvc.  pipe: riab_run's pipeline, or NULL.
int launch_bvc(const EnvK& env, const riab_bvc_cells* bvc, const OutK& out, const double* pos_in, long long n_rows,
               float* scratch, int32_t* first_wall, const double* head_dir, cudaStream_t s, BvcPipe* pipe = nullptr) {
  if (n_rows == 0) return 0;
  BvcConst bc;
  bc.n_cells = bvc->n_cells; bc.n_pad = bvc->n_pad; bc.T = bvc->n_test_angles;
  bc.min_fr = bvc->min_fr; bc.span = bvc->max_fr - bvc->min_fr;
  bc.packed = bvc->packed_dev; bc.test_dirs = bvc->test_dirs_dev;
  bc.ego = bvc->egocentric; bc.head_dir = head_dir;
  const long long n_tiles = (n_rows + BVC_AT - 1) / BVC_AT;
  const size_t smemA = (size_t)bc.T * 2 * sizeof(double);
  const size_t smemB = (size_t)bc.T * (BVC_CT + 2 * BVC_AT) * sizeof(float);
  // spikes without OU noise are drawn in the integration kernel's epilogue (the ray kernel clears the rows first);
  // OU noise (a read-modify-write of the noise state per rate) and odd shard offsets keep the k_finish_rows post-pass
  const int fold = (out.spikes != nullptr && out.noise == nullptr && (out.id_offset & 1ll) == 0) ? 1 : 0;
  uint32_t* const zsp = fold ? out.spikes : nullptr;
  if (pipe != nullptr && (out.pop < 0 || out.pop >= PIPE_POPS || pipe->scratch2[out.pop] == nullptr)) pipe = nullptr;
  const int pb = pipe ? (int)(pipe->step & 1) : 0;
  if (pipe) {
    if (pb) scratch = pipe->scratch2[out.pop];
    // the integral of two steps ago read this buffer (and wrote the ring slot a short ring re-uses now)
    if (pipe->used[pb][out.pop]) RIAB_CUDA_OK(cudaStreamWaitEvent(s, pipe->int_done[pb][out.pop], 0));
  }
  // (angle, wall) table of the float32 screen in shared memory: up to BVC_NW walls and 40 KB (one ray CTA still fits next to
  // two integration CTAs of the previous step, 2 x 92 KB at T = 180)
  const size_t smemT = smemA + (size_t)bc.T * (sizeof(float2) + (size_t)env.W * sizeof(BvcTab));
  const bool table = env.W <= BVC_NW && smemT <= 40 * 1024;
  if (table) k_bvc_rays<true><<<(unsigned)n_tiles, NT, smemT, s>>>(env, bc, pos_in, n_rows, scratch, first_wall, zsp, out.spike_ld);
  else {
    // the walls in float64 and float32 beside the directions: past 48 KB from about 950 walls at T = 180
    const size_t smemW = smemA + (size_t)env.W * (4 * sizeof(double) + sizeof(float4));
    if (smemW > 48 * 1024) RIAB_CUDA_OK(cudaFuncSetAttribute(k_bvc_rays<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemW));
    k_bvc_rays<false><<<(unsigned)n_tiles, NT, smemW, s>>>(env, bc, pos_in, n_rows, scratch, first_wall, zsp, out.spike_ld);
  }
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  if (pipe) {                                         // the integral (and its post-pass) go to the side stream
    RIAB_CUDA_OK(cudaEventRecord(pipe->rays_done, s));
    RIAB_CUDA_OK(cudaStreamWaitEvent(pipe->side, pipe->rays_done, 0));
    s = pipe->side;
  }
  // (the attribute belongs to the current device's function image: set per call, a single process may drive several GPUs)
  RIAB_CUDA_OK(cudaFuncSetAttribute(k_bvc_integrate, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  int sms, rc;
  if ((rc = num_sms(sms))) return rc;
  const unsigned cts = (unsigned)(bc.n_pad / BVC_CT);
  unsigned gy = (unsigned)((2 * sms + cts - 1) / cts);           // ~2 CTAs per SM in total
  if (gy > n_tiles) gy = (unsigned)n_tiles;
  if (gy < 1) gy = 1;
  if (bc.ego) {
    RIAB_CUDA_OK(cudaFuncSetAttribute(k_bvc_integrate_ego, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    const size_t smemE = ((size_t)((bc.T + 1) / 2 * 2) * 2 + (size_t)bc.T * 2 * BVC_AT) * sizeof(float);
    k_bvc_integrate_ego<<<dim3(cts, gy), NT, smemE, s>>>(bc, scratch, n_rows, n_tiles, out, fold);
  } else {
    k_bvc_integrate<<<dim3(cts, gy), NT, smemB, s>>>(bc, scratch, n_rows, n_tiles, out, fold);
  }
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  if (!fold && (rc = finish_rows(out, bc.n_cells, n_rows, s))) return rc;
  if (pipe) {
    RIAB_CUDA_OK(cudaEventRecord(pipe->int_done[pb][out.pop], s));
    pipe->used[pb][out.pop] = true;
  }
  return 0;
}

// ---------------------------------------------------------------------------
// FeedForwardLayer (riab_ffl.cuh).  cuTensorMapEncodeTiled comes from the driver through the runtime's entry-point query,
// so the library links against the runtime only.
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
int ffl_tmap(CUtensorMap* map, const float* base, long long inner, long long outer, long long ld, int box_outer) {
  static EncodeTiledFn encode = nullptr;
  if (encode == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    RIAB_CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    if (q != cudaDriverEntryPointSuccess || fn == nullptr) return fail(RIAB_ERR_CUDA, "cuTensorMapEncodeTiled not found");
    encode = (EncodeTiledFn)fn;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {(cuuint32_t)FFL_BK, (cuuint32_t)box_outer};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(RIAB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}

template <int BN>
int launch_ffl_bn(FflK& k, cudaStream_t s) {
  constexpr int smem = ffl_smem_bytes<BN>();
  RIAB_CUDA_OK(cudaFuncSetAttribute(k_ffl<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k.n_tiles = (k.n_cells + BN - 1) / BN;
  const long long m_tiles = (k.n_rows + FFL_BM - 1) / FFL_BM;
  k_ffl<BN><<<(unsigned)(m_tiles * k.n_tiles), FFL_THREADS, smem, s>>>(k);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// packed: the layer's contraction reads W_hi | W_lo blocks (every FeedForwardLayer but a per-agent TD layer)
int check_ffl(const riab_ffl_cells* f, const OutK& out, long long n_rows, bool packed = true) {
  if (f == nullptr || f->bias_dev == nullptr) return fail(RIAB_ERR_INVALID, "ffl / bias_dev NULL");
  if (f->n_cells <= 0) return fail(RIAB_ERR_INVALID, "ffl: n_cells must be > 0");
  if (f->n_inputs < 0 || f->n_inputs > RIAB_FFL_MAX_INPUTS)
    return fail(RIAB_ERR_UNSUPPORTED, "ffl: %d inputs (at most %d)", f->n_inputs, RIAB_FFL_MAX_INPUTS);
  if (f->activation < RIAB_ACT_LINEAR || f->activation > RIAB_ACT_SOFTPLUS) return fail(RIAB_ERR_INVALID, "ffl: bad activation %d", f->activation);
  if (f->prime_dev != nullptr && out.ld % 4 != 0) return fail(RIAB_ERR_INVALID, "ffl: ld must be a multiple of 4");
  if (n_rows == 0) return 0;
  for (int i = 0; i < f->n_inputs; ++i) {
    const riab_ffl_input& in = f->inputs[i];
    if (in.rows_dev == nullptr) continue;                        // an input that was never updated contributes zeros
    if ((packed && in.w_dev == nullptr) || in.n_in <= 0 || in.k_pad != (in.n_in + FFL_BK - 1) / FFL_BK * FFL_BK || in.ld < in.n_in)
      return fail(RIAB_ERR_INVALID, "ffl input %d: bad weights / sizes (pack with riab_ffl_pack)", i);
    if (((uintptr_t)in.rows_dev) % 16 != 0 || (in.ld * 4) % 16 != 0 || ((uintptr_t)in.w_dev) % 16 != 0)
      return fail(RIAB_ERR_INVALID, "FFL operands need 16-byte aligned rows");
  }
  return 0;
}

// One FeedForwardLayer evaluation over n_rows rows (+ noise / spikes through the k_finish_rows post-pass), checked by
// check_ffl.
int launch_ffl(const riab_ffl_cells* f, long long n_rows, const double* pos, const OutK& out, cudaStream_t s) {
  if (n_rows == 0) return 0;
  // N tile: the wgmma N of 8, 32 or 64 that wastes least (64: accumulator + per-stage partial = 64 registers)
  const int bn = f->n_cells <= 8 ? 8 : (f->n_cells <= 32 ? 32 : 64);
  FflK k;
  memset(&k, 0, sizeof(k));
  int rc;
  const int n_pad = (f->n_cells + 7) / 8 * 8;
  for (int i = 0; i < f->n_inputs; ++i) {
    const riab_ffl_input& in = f->inputs[i];
    if (in.rows_dev == nullptr) continue;
    const int l = k.n_inputs++;
    if ((rc = ffl_tmap(&k.in[l], in.rows_dev, in.n_in, n_rows, in.ld, FFL_BM)) ||
        (rc = ffl_tmap(&k.whi[l], in.w_dev, in.k_pad, n_pad, in.k_pad, bn)) ||
        (rc = ffl_tmap(&k.wlo[l], in.w_dev + (size_t)n_pad * in.k_pad, in.k_pad, n_pad, in.k_pad, bn))) return rc;
    k.ktiles[l] = in.k_pad / FFL_BK;
  }
  k.n_cells = f->n_cells; k.act = f->activation;
  k.p0 = f->act[0]; k.p1 = f->act[1]; k.p2 = f->act[2]; k.p3 = f->act[3];
  k.n_rows = n_rows; k.ld = out.ld;
  k.rates = out.rates; k.prime = f->prime_dev; k.bias = f->bias_dev; k.pos = pos;
  if (bn == 8) rc = launch_ffl_bn<8>(k, s);
  else if (bn == 32) rc = launch_ffl_bn<32>(k, s);
  else rc = launch_ffl_bn<64>(k, s);
  return rc ? rc : finish_rows(out, f->n_cells, n_rows, s);
}

// ---------------------------------------------------------------------------
// NeuralNetworkNeurons (riab_nnn.cuh).  Layer 1's W_hi | W_lo block of input i starts after those of inputs 0..i-1.
long long nnn_w1_offset(const riab_nnn_cells* c, int i) {
  long long off = 0;
  for (int j = 0; j < i; ++j) off += 2LL * ((c->widths[1] + 7) / 8 * 8) * ((c->inputs[j].n_in + FFL_BK - 1) / FFL_BK * FFL_BK);
  return off;
}

// The layer widths and activations of a module with n_layers >= 1 and inputs of n_in > 0 rates each, as riab_nnn_pack
// packs them and the kernels run them; who: the messages' prefix.
int check_nnn_layers(const riab_nnn_cells* c, const char* who) {
  int n_in = 0;
  for (int i = 0; i < c->n_inputs; ++i) n_in += c->inputs[i].n_in;
  if (n_in != c->widths[0]) return fail(RIAB_ERR_INVALID, "%s: inputs give %d rates, widths[0] is %d", who, n_in, c->widths[0]);
  for (int l = 1; l <= c->n_layers; ++l) {
    if (c->widths[l] <= 0) return fail(RIAB_ERR_INVALID, "%s: width %d of layer %d", who, c->widths[l], l);
    if (l < c->n_layers && c->widths[l] > RIAB_NNN_MAX_HIDDEN)
      return fail(RIAB_ERR_UNSUPPORTED, "%s: hidden width %d (at most %d)", who, c->widths[l], RIAB_NNN_MAX_HIDDEN);
    if (c->act[l - 1] < RIAB_NNN_IDENTITY || c->act[l - 1] > RIAB_NNN_TANH)
      return fail(RIAB_ERR_INVALID, "%s: bad activation %d", who, c->act[l - 1]);
  }
  return 0;
}

int check_nnn(const riab_nnn_cells* c, long long n_rows) {
  if (c == nullptr) return fail(RIAB_ERR_INVALID, "nnn cells NULL");
  if (c->n_cells <= 0) return fail(RIAB_ERR_INVALID, "nnn: n_cells must be > 0");
  if (c->n_layers < 0 || c->n_layers > RIAB_NNN_MAX_LAYERS)
    return fail(RIAB_ERR_UNSUPPORTED, "nnn: %d Linear layers (at most %d)", c->n_layers, RIAB_NNN_MAX_LAYERS);
  if (c->n_inputs < (c->n_layers == 0 ? 1 : 0) || c->n_inputs > RIAB_FFL_MAX_INPUTS)
    return fail(RIAB_ERR_UNSUPPORTED, "nnn: %d inputs (at most %d)", c->n_inputs, RIAB_FFL_MAX_INPUTS);
  if (c->n_layers == 0) {
    const riab_ffl_input& in = c->inputs[0];
    if (n_rows > 0 && (in.rows_dev == nullptr || in.ld < c->n_cells)) return fail(RIAB_ERR_INVALID, "nnn: bad precomputed rows");
    return 0;
  }
  if (c->packed_dev == nullptr || ((uintptr_t)c->packed_dev) % 16 != 0) return fail(RIAB_ERR_INVALID, "nnn: packed_dev NULL or misaligned");
  for (int i = 0; i < c->n_inputs; ++i) {
    const riab_ffl_input& in = c->inputs[i];
    if (in.n_in <= 0 || in.k_pad != (in.n_in + FFL_BK - 1) / FFL_BK * FFL_BK || (in.rows_dev != nullptr && in.ld < in.n_in))
      return fail(RIAB_ERR_INVALID, "nnn input %d: bad sizes (pack with riab_nnn_pack)", i);
    if (((uintptr_t)in.rows_dev) % 16 != 0 || (in.ld * 4) % 16 != 0) return fail(RIAB_ERR_INVALID, "NNN inputs need 16-byte aligned rows");
  }
  int rc;
  if ((rc = check_nnn_layers(c, "nnn"))) return rc;
  if (c->widths[c->n_layers] != c->n_cells) return fail(RIAB_ERR_INVALID, "nnn: n_cells != the last layer's width");
  return 0;
}

// One NeuralNetworkNeurons evaluation over n_rows rows (+ noise / spikes through the k_finish_rows post-pass), checked by
// check_nnn.  Inputs that were never updated contribute zeros, as for a FeedForwardLayer.
int launch_nnn(const riab_nnn_cells* c, long long n_rows, const double* pos, const OutK& out, cudaStream_t s) {
  if (n_rows == 0) return 0;
  if (c->n_layers == 0) {
    RIAB_CUDA_OK(nnn_rows_launch(c->inputs[0].rows_dev, c->inputs[0].ld, out.rates, out.ld, c->n_cells, n_rows, pos, s));
    g_launches++;
  } else {
    NnnK k;
    memset(&k, 0, sizeof(k));
    int rc;
    const int h1 = c->widths[1], n_pad = (h1 + 7) / 8 * 8;
    // N tile of layer 1: 32 columns cover the default MLP's 20 in one chunk; wider first layers take chunks of 64
    const int bn = h1 <= 32 ? 32 : 64;
    for (int i = 0; i < c->n_inputs; ++i) {
      const riab_ffl_input& in = c->inputs[i];
      const float* w = c->packed_dev + nnn_w1_offset(c, i);
      if (in.rows_dev == nullptr) continue;
      const int l = k.n_inputs++;
      if ((rc = ffl_tmap(&k.in[l], in.rows_dev, in.n_in, n_rows, in.ld, NNN_BM)) ||
          (rc = ffl_tmap(&k.whi[l], w, in.k_pad, n_pad, in.k_pad, bn)) ||
          (rc = ffl_tmap(&k.wlo[l], w + (size_t)n_pad * in.k_pad, in.k_pad, n_pad, in.k_pad, bn))) return rc;
      k.ktiles[l] = in.k_pad / FFL_BK;
    }
    k.n_layers = c->n_layers;
    int hmax = 1;
    for (int l = 0; l <= c->n_layers; ++l) k.widths[l] = c->widths[l];
    for (int l = 0; l < c->n_layers; ++l) k.act[l] = c->act[l];
    for (int l = 1; l < c->n_layers; ++l) hmax = std::max(hmax, c->widths[l]);
    k.h_ld = hmax | 1;
    k.bias1 = c->packed_dev + nnn_w1_offset(c, c->n_inputs);
    k.n_rows = n_rows; k.ld = out.ld; k.rates = out.rates; k.pos = pos;
    RIAB_CUDA_OK(nnn_launch(k, bn, s));
    g_launches++;
  }
  return finish_rows(out, c->n_cells, n_rows, s);
}

// ---------------------------------------------------------------------------
// TD learning (riab_td.cuh).  check_td: the TD state of a layer whose riab_ffl_cells part check_ffl already accepted.
int check_td(const riab_td_cells* t, long long out_ld) {
  if (t == nullptr) return fail(RIAB_ERR_INVALID, "td cells NULL");
  const riab_ffl_cells& f = t->ffl;
  if (t->fr_prev_dev == nullptr || t->deriv_dev == nullptr || t->td_error_dev == nullptr)
    return fail(RIAB_ERR_INVALID, "td: fr_prev / deriv / td_error NULL");
  if (t->ld != out_ld || t->ld % 4 != 0 || t->ld < f.n_cells)
    return fail(RIAB_ERR_INVALID, "td: ld %lld must equal the rates' ld (%lld), a multiple of 4", (long long)t->ld, out_ld);
  if (!(t->dt > 0.0) || !(t->tau_e > 0.0) || !std::isfinite(t->tau_e) || !std::isfinite(t->dt))
    return fail(RIAB_ERR_INVALID, "td: dt and tau_e must be finite and > 0");
  if (t->self_input < -1 || t->self_input >= f.n_inputs) return fail(RIAB_ERR_INVALID, "td: bad self_input %d", t->self_input);
  if (t->per_agent_weights != 0 && t->per_agent_weights != 1)
    return fail(RIAB_ERR_INVALID, "td: per_agent_weights must be 0 or 1, not %d", t->per_agent_weights);
  if (f.n_inputs < 0 || f.n_inputs > RIAB_FFL_MAX_INPUTS) return fail(RIAB_ERR_UNSUPPORTED, "td: %d inputs", f.n_inputs);
  for (int l = 0; l < f.n_inputs; ++l) {
    const riab_ffl_input& in = f.inputs[l];
    if (t->trace_dev[l] == nullptr || t->w_master_dev[l] == nullptr || (!t->per_agent_weights && in.w_dev == nullptr) ||
        in.n_in <= 0 ||
        in.k_pad != (in.n_in + FFL_BK - 1) / FFL_BK * FFL_BK)
      return fail(RIAB_ERR_INVALID, "td input %d: trace / master / packed weights missing or mis-sized", l);
    if (t->trace_ld[l] < in.n_in || t->trace_ld[l] % 4 != 0 || ((uintptr_t)t->trace_dev[l]) % 16 != 0)
      return fail(RIAB_ERR_INVALID, "td input %d: trace rows must be 16-byte aligned with ld >= n_in, a multiple of 4", l);
  }
  return 0;
}

// k_td_trace over n_rows rows after the layer's rates (checked by check_ffl / check_td)
int launch_td_trace(const riab_td_cells* t, long long n_rows, const float* rates, cudaStream_t s) {
  if (n_rows == 0) return 0;
  TdTraceK k;
  memset(&k, 0, sizeof(k));
  k.rates = rates; k.fr_prev = t->fr_prev_dev; k.deriv = t->deriv_dev;
  k.ld = t->ld; k.n_rows = n_rows; k.n_cells = t->ffl.n_cells; k.n_inputs = t->ffl.n_inputs;
  for (int l = 0; l < k.n_inputs; ++l) {
    const riab_ffl_input& in = t->ffl.inputs[l];
    const bool self = l == t->self_input;              // ValueNeuron.update reads the layer's NEW firingrate
    k.in[l] = self ? rates : in.rows_dev;
    k.in_ld[l] = self ? t->ld : in.ld;
    k.trace[l] = t->trace_dev[l]; k.trace_ld[l] = t->trace_ld[l]; k.n_in[l] = in.n_in;
  }
  k.dt = (float)t->dt;
  k.decay = (float)(1.0 - t->dt / t->tau_e);
  k_td_trace<<<(unsigned)n_rows, TD_TRACE_THREADS, 0, s>>>(k);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// The per-agent layer's contraction over n_rows rows (k_td_forward_pa): row r reads the masters of agent w_row[r] and the
// input rows in_row[r] (NULL: r).  Up to 8 rows per CTA so that small layers still give every warp a (row, cell) pair;
// the rows are staged in shared memory when they fit in 48 KB.  Checked by check_ffl / check_td.
int launch_td_forward_pa(const riab_td_cells* t, long long n_rows, const long long* w_row, const long long* in_row,
                         const double* pos, float* rates, long long ld, float* prime, cudaStream_t s) {
  if (n_rows == 0) return 0;
  const riab_ffl_cells& f = t->ffl;
  TdFwdPaK k;
  memset(&k, 0, sizeof(k));
  int stage_ld = 0;
  for (int l = 0; l < f.n_inputs; ++l) {
    const riab_ffl_input& in = f.inputs[l];
    k.in[l] = in.rows_dev; k.in_ld[l] = in.ld; k.w[l] = t->w_master_dev[l]; k.n_in[l] = in.n_in;
    k.soff[l] = stage_ld;
    stage_ld += (in.n_in + 3) / 4 * 4;
  }
  k.n_inputs = f.n_inputs; k.n_cells = f.n_cells; k.stage_ld = stage_ld;
  k.act = ActK{f.activation, f.act[0], f.act[1], f.act[2], f.act[3]};
  k.bias = f.bias_dev; k.w_row = w_row; k.in_row = in_row; k.pos = pos;
  k.rates = rates; k.prime = prime; k.ld = ld; k.n_rows = n_rows;
  constexpr int kStageBytes = 48 * 1024, kWarps = TD_FWD_THREADS / 32;
  const int rows = std::max(1, kWarps / std::min(f.n_cells, kWarps));
  const int fit = stage_ld > 0 ? kStageBytes / (stage_ld * 4) : rows;
  k.rows_per_cta = fit > 0 ? std::min(rows, fit) : rows;
  const unsigned grid = (unsigned)((n_rows + k.rows_per_cta - 1) / k.rows_per_cta);
  if (fit > 0) {
    const size_t smem = (size_t)k.rows_per_cta * stage_ld * 4;
    k_td_forward_pa<true><<<grid, TD_FWD_THREADS, smem, s>>>(k);
  } else {
    k_td_forward_pa<false><<<grid, TD_FWD_THREADS, 0, s>>>(k);
  }
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// The split of the agent axis of one learning contraction: from the shapes alone (so the same shapes always sum in the
// same order), about TD_TARGET_CTAS CTAs (16 per SM for the bandwidth-bound 8-row tiles, whose loads need the CTAs in
// flight; 4 per SM for the 64 x 64 tiles), chunks a multiple of TD_KC agents.
constexpr int TD_TARGET_CTAS = 4 * 132, TD_TARGET_CTAS_SMALL = 16 * 132;
struct TdSplit {
  bool small = false;            // n <= 8: one 8-row CUDA-core tile (8 x 256), else 64 x 64 wgmma tiles
  int tiles = 0;
  long long chunk = 0, splits = 0;
};
TdSplit td_split(int n, int n_in, long long A) {
  TdSplit t;
  t.small = n <= 8;
  const int bm = t.small ? 8 : 64, bn = t.small ? 256 : 64;
  t.tiles = ((n + bm - 1) / bm) * ((n_in + bn - 1) / bn);
  const long long rounds = (A + TD_KC - 1) / TD_KC;
  const int target = t.small ? TD_TARGET_CTAS_SMALL : TD_TARGET_CTAS;
  const long long want = std::max(1LL, std::min(rounds, (long long)((target + t.tiles - 1) / t.tiles)));
  t.chunk = (rounds + want - 1) / want * TD_KC;
  t.splits = (A + t.chunk - 1) / t.chunk;
  return t;
}
long long td_g_ld(int n) { return (n + 7) / 8 * 8; }
size_t td_g_bytes(int n, long long A) { return ((size_t)A * td_g_ld(n) * 4 + 255) / 256 * 256; }

// ---------------------------------------------------------------------------
// RandomSpatialNeurons (riab_rsn.cuh).  The sample points are a place-cell population: make_place validates them and
// sets up their constants, in the direct (not expanded) Gaussian form with the [0, 1] scale.
int make_rsn(const riab_rsn_cells* r, const EnvK& env, PlaceConst& c) {
  if (r == nullptr || r->targets_dev == nullptr) return fail(RIAB_ERR_INVALID, "rsn / targets_dev NULL");
  if (r->n_cells <= 0 || r->n_points <= 0 || r->k_pad != (r->n_points + FFL_BK - 1) / FFL_BK * FFL_BK ||
      r->points.n_cells != r->k_pad || r->points.description != RIAB_PC_GAUSSIAN || r->points.min_fr != 0.f ||
      r->points.max_fr != 1.f)
    return fail(RIAB_ERR_INVALID, "rsn: bad sizes / sample points (pack with riab_rsn_pack)");
  if (!(r->min_fr <= r->max_fr)) return fail(RIAB_ERR_INVALID, "rsn: min_fr > max_fr");
  if (((uintptr_t)r->targets_dev) % 16 != 0) return fail(RIAB_ERR_INVALID, "rsn: targets_dev must be 16-byte aligned");
  int rc;
  if ((rc = make_place(&r->points, env, c))) return rc;
  if (r->points.wall_geometry != RIAB_GEOM_EUCLIDEAN && r->points.centres_dev == nullptr)
    return fail(RIAB_ERR_INVALID, "rsn: centres_dev NULL");
  c.expanded = 0; c.fold = 0; c.lspan = 0.f; c.kx = 0.f;
  c.comp = 0;                          // k_rsn evaluates the plain direct form
  return 0;
}

template <int WI, int DESC, int BN>
int launch_rsn_k(RsnK& k, cudaStream_t s) {
  constexpr int smem = rsn_smem_bytes<BN>(), CWG = WI >= 4 ? 1 : 2;     // consumer warpgroups (see riab_rsn.cuh)
  RIAB_CUDA_OK(cudaFuncSetAttribute(k_rsn<WI, DESC, BN, CWG>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const long long m_tiles = (k.n_rows + 64 * CWG - 1) / (64 * CWG);
  k.n_tiles = (k.n_cells + BN - 1) / BN;
  k_rsn<WI, DESC, BN, CWG><<<(unsigned)(m_tiles * k.n_tiles), rsn_threads<CWG>(), smem, s>>>(k);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// the N tile of k_ffl (8, 32 or 64 from n); 8 inner walls stop at 32, whose accumulators fit next to their point registers
template <int WI, int DESC>
int launch_rsn_bn(RsnK& k, cudaStream_t s) {
  if (k.n_cells <= 8) return launch_rsn_k<WI, DESC, 8>(k, s);
  if (k.n_cells <= 32 || WI >= 8) return launch_rsn_k<WI, DESC, 32>(k, s);
  if constexpr (WI < 8) return launch_rsn_k<WI, DESC, 64>(k, s);
  return 0;
}

// One RandomSpatialNeurons evaluation at n_rows positions (+ noise / spikes through the k_finish_rows post-pass, as for
// FeedForwardLayers); r and pc checked by make_rsn.
int launch_rsn(const riab_rsn_cells* r, const PlaceConst& pc, const EnvK& env, const double* pos, long long n_rows,
               const OutK& out, cudaStream_t s) {
  if (n_rows == 0) return 0;
  const int wi = pc.n_inner;
  const int bn = r->n_cells <= 8 ? 8 : ((r->n_cells <= 32 || wi > 4) ? 32 : 64);    // as launch_rsn_bn
  const int n_pad = (r->n_cells + 7) / 8 * 8;
  RsnK k;
  memset(&k, 0, sizeof(k));
  int rc;
  if ((rc = ffl_tmap(&k.thi, r->targets_dev, r->k_pad, n_pad, r->k_pad, bn)) ||
      (rc = ffl_tmap(&k.tlo, r->targets_dev + (size_t)n_pad * r->k_pad, r->k_pad, n_pad, r->k_pad, bn))) return rc;
  k.pc = pc;
  k.walls = env.walls;
  k.n_cells = r->n_cells; k.ktiles = r->k_pad / FFL_BK; k.n_points = r->n_points;
  k.n_rows = n_rows; k.ld = out.ld; k.rates = out.rates; k.pos = pos;
  // the geodesic detour needs the run-time profile switch of place_rates4 (as launch_place), and then has one inner wall
  if (pc.geometry == RIAB_GEOM_GEODESIC && wi == 1) rc = launch_rsn_bn<1, -1>(k, s);
  else if (wi == 0) rc = launch_rsn_bn<0, RIAB_PC_GAUSSIAN>(k, s);
  else if (wi == 1) rc = launch_rsn_bn<1, RIAB_PC_GAUSSIAN>(k, s);
  else if (wi == 2) rc = launch_rsn_bn<2, RIAB_PC_GAUSSIAN>(k, s);
  else if (wi <= 4) rc = launch_rsn_bn<4, RIAB_PC_GAUSSIAN>(k, s);
  else rc = launch_rsn_bn<8, RIAB_PC_GAUSSIAN>(k, s);
  return rc ? rc : finish_rows(out, r->n_cells, n_rows, s);
}

int make_src(const riab_motion_source* src, long long n_agents, SrcK& k) {
  memset(&k, 0, sizeof(k));
  k.kind = src->kind;
  k.t = src->t;
  if (src->kind == RIAB_MOTION_IMPORTED) {
    const riab_trajectory& tr = src->traj;
    if (tr.times_dev == nullptr || tr.y_dev == nullptr || tr.M_dev == nullptr || tr.T < 4 || !(tr.t_max > 0.0))
      return fail(RIAB_ERR_INVALID, "motion source: bad trajectory");
    if (tr.n_traj != 1 && tr.n_traj != n_agents)
      return fail(RIAB_ERR_INVALID, "motion source: %lld trajectories for %lld agents", (long long)tr.n_traj, n_agents);
    k.times = tr.times_dev; k.y = tr.y_dev; k.M = tr.M_dev; k.T = tr.T; k.n_traj = tr.n_traj; k.t_max = tr.t_max;
    return 0;
  }
  if (src->kind == RIAB_MOTION_FORCED) {
    if (src->forced_dev == nullptr) return fail(RIAB_ERR_INVALID, "motion source: forced positions NULL");
    k.forced = src->forced_dev; k.bcast = src->forced_broadcast != 0;
    return 0;
  }
  return fail(RIAB_ERR_INVALID, "motion source: kind %d", src->kind);
}

// ---------------------------------------------------------------------------
// (the motion and step arguments of MODE-0 launches, which read neither)
const riab_motion_params kNoMotion = {};
const riab_step_io kNoStep = {};

// One population of one step, checked: its kind's constants and its output.
struct Pop {
  int kind = -1, n_cells = 0;
  int n_pad = 0;                        // the k_step kinds' packed cell count (a multiple of CELL_PAD), else 0
  bool step_policy = false;             // has_step_policy
  bool walls = false;                   // its rate kernels read the walls (pop_reads_walls)
  double bound = -1.0;                  // an upper bound of the rates for thinned spikes (make_out), negative for none
  OutK out;
  PlaceConst place; GridConst grid; OvcConst ovc; KinConst kin; AvcConst avc; PppcConst pppc; PwnConst pwn;
  const riab_bvc_cells* bvc = nullptr; float* bvc_scratch = nullptr; int32_t* first_wall = nullptr;
  const riab_ffl_cells* ffl = nullptr;
  const riab_td_cells* td = nullptr;    // RIAB_CELLS_TD: its layer is `ffl`
  const riab_rsn_cells* rsn = nullptr;  // its sample points: `place`
  const riab_nnn_cells* nnn = nullptr;
};

// Whether a population's rates come from a k_step policy, so that a motion step can be fused into its rate kernel.  The
// others: one_hot PlaceCells (an arg-min across cells), BVC (the latency-bound ray kernel wants all its CTAs in ONE wave:
// the 128-register motion code would halve its occupancy), FeedForwardLayers and NeuralNetworkNeurons (they read other
// populations' rows, not the positions) and RandomSpatialNeurons (a GEMM kernel without motion warps).
bool has_step_policy(int kind, const void* cells) {
  if (kind == RIAB_CELLS_PLACE) return cells != nullptr && ((const riab_place_cells*)cells)->description != RIAB_PC_ONE_HOT;
  return kind == RIAB_CELLS_GRID || kind == RIAB_CELLS_OVC || kind == RIAB_CELLS_KIN || kind == RIAB_CELLS_AVC ||
         kind == RIAB_CELLS_PPPC || kind == RIAB_CELLS_PWN;
}

// Whether a population's rate kernels read the walls: BVC rays (any wall count up to RIAB_MAX_WALLS), and the line of
// sight / geodesic distances and occlusion tests, which k_step, k_place_onehot and k_rsn run over at most MAXW staged walls.
bool pop_reads_walls(int kind, const void* cells) {
  if (kind == RIAB_CELLS_BVC) return true;
  if (kind == RIAB_CELLS_PLACE) return ((const riab_place_cells*)cells)->wall_geometry != RIAB_GEOM_EUCLIDEAN;
  if (kind == RIAB_CELLS_PPPC) return ((const riab_pppc_cells*)cells)->place.wall_geometry != RIAB_GEOM_EUCLIDEAN;
  if (kind == RIAB_CELLS_RSN) return ((const riab_rsn_cells*)cells)->points.wall_geometry != RIAB_GEOM_EUCLIDEAN;
  if (kind == RIAB_CELLS_OVC) return ((const riab_ovc_cells*)cells)->walls_occlude != 0;
  if (kind == RIAB_CELLS_AVC) return ((const riab_avc_cells*)cells)->walls_occlude != 0;
  return false;
}

int make_pop(const EnvK& ek, int kind, const void* cells, const riab_rates_out* out, const riab_neuron_noise* noise,
             double dt, const riab_agents& ag, Pop& d) {
  if (cells == nullptr) return fail(RIAB_ERR_INVALID, "cells NULL");
  int rc = 0;
  d.kind = kind;
  d.step_policy = has_step_policy(kind, cells);
  d.walls = pop_reads_walls(kind, cells);
  if (d.walls && kind != RIAB_CELLS_BVC && ek.W > MAXW)
    return fail(RIAB_ERR_UNSUPPORTED, "n_walls=%d: line_of_sight / geodesic distances and walls_occlude read at most %d walls "
                "(wall_geometry=\"euclidean\" or walls_occlude=False read none and take up to %d)", ek.W, MAXW, RIAB_MAX_WALLS);
  if (kind == RIAB_CELLS_PLACE) {
    const riab_place_cells* pc = (const riab_place_cells*)cells;
    rc = make_place(pc, ek, d.place);
    d.n_cells = pc->n_cells; d.n_pad = d.place.n_pad;
    if (pc->description != RIAB_PC_ONE_HOT) d.bound = fmaxf(pc->min_fr, pc->max_fr);   // one_hot: post-pass spikes, dense
  } else if (kind == RIAB_CELLS_GRID) {
    const riab_grid_cells* gc = (const riab_grid_cells*)cells;
    rc = make_grid(gc, ek, d.grid);
    d.n_cells = gc->n_cells; d.n_pad = d.grid.n_pad;
    d.bound = fmaxf(gc->min_fr, gc->max_fr);
  } else if (kind == RIAB_CELLS_OVC) {
    rc = make_ovc((const riab_ovc_cells*)cells, ek, ag.head_direction, d.ovc);
    d.n_cells = d.ovc.n_cells; d.n_pad = d.ovc.n_pad;
  } else if (kind == RIAB_CELLS_BVC) {
    d.bvc = (const riab_bvc_cells*)cells;
    d.n_cells = d.bvc->n_cells;
  } else if (kind == RIAB_CELLS_FFL) {
    d.ffl = (const riab_ffl_cells*)cells;
    d.n_cells = d.ffl->n_cells;
  } else if (kind == RIAB_CELLS_TD) {
    d.td = (const riab_td_cells*)cells;
    d.ffl = &d.td->ffl;
    d.n_cells = d.ffl->n_cells;
  } else if (kind == RIAB_CELLS_RSN) {
    d.rsn = (const riab_rsn_cells*)cells;
    rc = make_rsn(d.rsn, ek, d.place);
    d.n_cells = d.rsn->n_cells;
  } else if (kind == RIAB_CELLS_KIN) {
    rc = make_kin((const riab_kin_cells*)cells, ag, d.kin);
    d.n_cells = d.kin.n_cells; d.n_pad = d.kin.n_pad;
  } else if (kind == RIAB_CELLS_AVC) {
    rc = make_avc((const riab_avc_cells*)cells, ek, ag.head_direction, ag.n_agents, d.avc);
    d.n_cells = d.avc.n_cells; d.n_pad = d.avc.n_pad;
  } else if (kind == RIAB_CELLS_PPPC) {
    rc = make_pppc((const riab_pppc_cells*)cells, ek, ag.velocity, d.pppc);
    d.n_cells = ((const riab_pppc_cells*)cells)->place.n_cells; d.n_pad = d.pppc.n_pad;
  } else if (kind == RIAB_CELLS_PWN) {
    const riab_pwn_cells* pw = (const riab_pwn_cells*)cells;
    rc = make_pwn(pw, d.pwn);
    d.n_cells = pw->n_cells; d.n_pad = d.pwn.n_pad;
    d.bound = fmaxf(pw->min_fr, pw->max_fr);
  } else if (kind == RIAB_CELLS_NNN) {
    d.nnn = (const riab_nnn_cells*)cells;
    d.n_cells = d.nnn->n_cells;
  } else {
    return fail(RIAB_ERR_INVALID, "bad cells_kind %d", kind);
  }
  if (rc || (rc = make_out(out, noise, d.n_cells, dt, ag.id_offset, d.out, d.bound))) return rc;
  if (kind == RIAB_CELLS_BVC) return check_bvc(ek, d.bvc, d.bvc_scratch = out->bvc_scratch, ag.n_agents);
  if (kind == RIAB_CELLS_TD)
    return (rc = check_ffl(d.ffl, d.out, ag.n_agents, d.td->per_agent_weights == 0)) ? rc : check_td(d.td, d.out.ld);
  if (kind == RIAB_CELLS_NNN) return check_nnn(d.nnn, ag.n_agents);
  return kind == RIAB_CELLS_FFL ? check_ffl(d.ffl, d.out, ag.n_agents) : 0;
}

// FeedForwardLayer-like kinds: they read other populations' rows and run after them (plan_run)
bool ffl_like(int kind) { return kind == RIAB_CELLS_FFL || kind == RIAB_CELLS_TD || kind == RIAB_CELLS_NNN; }

// One population's kernels for one step.  MODE 0: rates at the agents' positions; 1: the motion step fused in; 2: skewed
// (rates at the current positions while the motion of the next step runs, riab_run); 3 / 4: riab_run's whole run (run),
// for the kinds whole_run_applies admits.  Kinds without a k_step policy run MODE 0 only.
template <int MODE>
int launch_pop(const EnvK& env, const riab_agents& ag, const riab_motion_params& mp, const riab_step_io& io, const Pop& d,
               cudaStream_t s, BvcPipe* pipe = nullptr, const RunK* run = nullptr) {
  // rates alone, of a population that reads no walls: stage none (MODE 1 - 4 also run the motion: step_kernel_walls)
  const EnvK ek = (MODE == 0 && !d.walls) ? without_walls(env) : env;
  const double* pos_in = (MODE == 0 || MODE == 2) ? ag.pos : nullptr;
  const long long n = ag.n_agents;
  if (!d.step_policy) {
    if constexpr (MODE == 0) {
      if (d.kind == RIAB_CELLS_PLACE) return launch_onehot(ek, d.place, d.out, ag.pos, n, s);
      if (d.kind == RIAB_CELLS_BVC)
        return launch_bvc(ek, d.bvc, d.out, ag.pos, n, d.bvc_scratch, d.first_wall, ag.head_direction, s, pipe);
      if (d.kind == RIAB_CELLS_RSN) return launch_rsn(d.rsn, d.place, ek, ag.pos, n, d.out, s);
      if (d.kind == RIAB_CELLS_NNN) return launch_nnn(d.nnn, n, ag.pos, d.out, s);
      int rc;
      if (d.td != nullptr && d.td->per_agent_weights) {
        rc = launch_td_forward_pa(d.td, n, nullptr, nullptr, ag.pos, d.out.rates, d.out.ld, d.ffl->prime_dev, s);
        if (!rc) rc = finish_rows(d.out, d.n_cells, n, s);
      } else {
        rc = launch_ffl(d.ffl, n, ag.pos, d.out, s);
      }
      return (rc || d.kind != RIAB_CELLS_TD) ? rc : launch_td_trace(d.td, n, d.out.rates, s);
    }
    return fail(RIAB_ERR_INVALID, "cells kind %d is launched unfused", d.kind);
  }
  if (d.kind == RIAB_CELLS_PLACE) return launch_place<MODE>(ek, ag, mp, io, d.place, d.out, pos_in, n, s, run);
  if (d.kind == RIAB_CELLS_GRID)
    return d.grid.turns ? launch_tile<GridPolicy<1>, MODE>(ek, ag, mp, io, d.grid, d.out, pos_in, n, s, run)
                        : launch_tile<GridPolicy<0>, MODE>(ek, ag, mp, io, d.grid, d.out, pos_in, n, s, run);
  if constexpr (MODE <= 2) {
    if (d.kind == RIAB_CELLS_OVC) return launch_tile<OvcPolicy, MODE>(ek, ag, mp, io, d.ovc, d.out, pos_in, n, s);
    if (d.kind == RIAB_CELLS_KIN) return launch_tile<KinPolicy, MODE>(ek, ag, mp, io, d.kin, d.out, pos_in, n, s);
    if (d.kind == RIAB_CELLS_AVC) return launch_tile<AvcPolicy, MODE>(ek, ag, mp, io, d.avc, d.out, pos_in, n, s);
    if (d.kind == RIAB_CELLS_PPPC) return launch_pppc<MODE>(ek, ag, mp, io, d.pppc, d.out, pos_in, n, s);
  }
  if (d.kind == RIAB_CELLS_PWN) return launch_tile<PwnPolicy, MODE>(ek, ag, mp, io, d.pwn, d.out, pos_in, n, s, run);
  return fail(RIAB_ERR_INVALID, "cells kind %d has no whole-run launch", d.kind);
}

// The motion steps a rate kernel cannot take: parity taps (only the stand-alone motion kernel records them), and those of
// populations without a k_step policy.
bool needs_motion_kernel(const EnvK& ek, const riab_step_io& io, const Pop& d) {
  return io.collision_mask || io.first_hit || io.n_iters || !d.step_policy || !step_kernel_walls(ek);
}

// One motion step, then population d's rates at the new positions; everything is checked before.
int step_fused(const riab_agents* agents, const riab_env* env, const EnvK& ek, const riab_motion_params* prm,
               const riab_step_io* io, const Pop& d, cudaStream_t s, BvcPipe* pipe = nullptr) {
  if (!needs_motion_kernel(ek, *io, d)) return launch_pop<1>(ek, *agents, *prm, *io, d, s);
  const int rc = riab_agent_update(agents, env, prm, io, s);
  return rc ? rc : launch_pop<0>(ek, *agents, kNoMotion, kNoStep, d, s, pipe);
}

// riab_step_fused (fused: the motion step, then the rates) and riab_neurons_update (the rates at agents->pos)
int neurons_update_impl(bool fused, const riab_agents* agents, const riab_env* env, const riab_motion_params* prm,
                        const riab_step_io* io, int32_t cells_kind, const void* cells, const riab_neuron_noise* noise,
                        const riab_rates_out* out, void* stream) {
  EnvK ek;
  Pop d;
  int rc;
  if ((rc = check_agents(agents)) || (rc = make_env(env, ek)) || (fused && (rc = check_motion(prm)))) return rc;
  if (fused && io == nullptr) return fail(RIAB_ERR_INVALID, "io NULL");
  if ((rc = make_pop(ek, cells_kind, cells, out, noise, fused ? prm->dt : (noise ? noise->dt : 1.0), *agents, d))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  return fused ? step_fused(agents, env, ek, prm, io, d, s) : launch_pop<0>(ek, *agents, kNoMotion, kNoStep, d, s);
}

// get_state: the rates at n_pos given positions (and head directions, egocentric cells), without noise or spikes
int rates_at(int kind, const void* cells, const double* pos_dev, int64_t n_pos, const riab_env* env, const double* head_dir,
             float* scratch, int32_t* first_wall, float* out_dev, int64_t ld_out, void* stream,
             const double* velocity = nullptr) {
  if (n_pos == 0) return 0;
  EnvK ek;
  Pop d;
  int rc;
  if ((rc = make_env(env, ek))) return rc;
  if (n_pos > 0 && pos_dev == nullptr) return fail(RIAB_ERR_INVALID, "pos_dev NULL");
  riab_rates_out ro = {};
  ro.rates_row = out_dev; ro.ld = ld_out; ro.bvc_scratch = scratch;
  riab_agents at = {};
  at.n_agents = n_pos; at.pos = (double*)pos_dev; at.head_direction = (double*)head_dir; at.velocity = (double*)velocity;
  if ((rc = make_pop(ek, kind, cells, &ro, nullptr, 1.0, at, d))) return rc;
  d.first_wall = first_wall;
  return launch_pop<0>(ek, at, kNoMotion, kNoStep, d, (cudaStream_t)stream);
}

// riab_ffl_rates / riab_nnn_rates: a layer over n_rows rows of its inputs; pos_dev masks the rows whose x is NaN
int layer_rates(int kind, const void* cells, int64_t n_rows, const double* pos_dev, const riab_neuron_noise* noise,
                const riab_rates_out* out, void* stream) {
  EnvK ek;
  memset(&ek, 0, sizeof(ek));                       // no walls: a layer reads its inputs' rows
  riab_agents at = {};
  at.n_agents = n_rows; at.pos = (double*)pos_dev; at.id_offset = noise ? noise->id_offset : 0;
  Pop d;
  int rc;
  if ((rc = make_pop(ek, kind, cells, out, noise, noise ? noise->dt : 1.0, at, d))) return rc;
  return launch_pop<0>(ek, at, kNoMotion, kNoStep, d, (cudaStream_t)stream);
}

// Row (next + k) mod rows of a ring of rows of row_len elements (next + k >= 0)
template <class T>
T* ring_row(T* ring, long long next_k, int rows, long long row_len) { return ring + (size_t)(next_k % rows) * row_len; }

// riab_run's use of the BVC pipeline (BvcPipe).  begin() pipelines the run when every population is an allocentric BVC
// one with a ring of >= 2 rows and the run has >= 2 steps: next to Place / Grid rate kernels (HBM- and dispatch-bound) the
// overlapped integral just competes for the same SMs (measured slower on configs[4]).  Leaving the run joins the side
// stream and frees the second ray buffers.
struct PipeScope {
  BvcPipe* pipe = nullptr;
  cudaStream_t s = nullptr;
  int begin(const riab_population* pops, int n_pops, long long n_agents, long long n_steps, cudaStream_t stream) {
    if (n_pops < 1 || n_pops > PIPE_POPS || n_steps < 2) return 0;
    for (int q = 0; q < n_pops; ++q)
      if (pops[q].kind != RIAB_CELLS_BVC || pops[q].cells == nullptr || ((const riab_bvc_cells*)pops[q].cells)->egocentric ||
          pops[q].ring_rows < 2 || pops[q].out.bvc_scratch == nullptr)
        return 0;
    static thread_local BvcPipe pipes[16];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return 0;
    BvcPipe* p = &pipes[dev];
    if (p->side == nullptr) {
      // keep the stream-ordered pool's memory across runs (by default it goes back to the driver at every synchronisation
      // and each run would pay a ~1 ms cudaMalloc for its second ray buffer again)
      cudaMemPool_t pool;
      if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        unsigned long long keep = ~0ull;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
      }
      RIAB_CUDA_OK(cudaStreamCreateWithFlags(&p->side, cudaStreamNonBlocking));
      RIAB_CUDA_OK(cudaEventCreateWithFlags(&p->rays_done, cudaEventDisableTiming));
      for (int b = 0; b < 2; ++b)
        for (int q = 0; q < PIPE_POPS; ++q) RIAB_CUDA_OK(cudaEventCreateWithFlags(&p->int_done[b][q], cudaEventDisableTiming));
    }
    memset(p->used, 0, sizeof(p->used));
    memset(p->scratch2, 0, sizeof(p->scratch2));
    pipe = p;
    s = stream;
    for (int q = 0; q < n_pops; ++q) {
      const int pid = pops[q].noise.population_id, T = ((const riab_bvc_cells*)pops[q].cells)->n_test_angles;
      if (pid >= 0 && pid < PIPE_POPS)
        RIAB_CUDA_OK(cudaMallocAsync((void**)&p->scratch2[pid], (size_t)riab_bvc_scratch_floats(n_agents, T) * sizeof(float), s));
    }
    return 0;
  }
  ~PipeScope() {
    if (pipe == nullptr) return;
    for (int b = 0; b < 2; ++b)
      for (int q = 0; q < PIPE_POPS; ++q)
        if (pipe->used[b][q]) cudaStreamWaitEvent(s, pipe->int_done[b][q], 0);
    for (int q = 0; q < PIPE_POPS; ++q)
      if (pipe->scratch2[q] != nullptr) { cudaFreeAsync(pipe->scratch2[q], s); pipe->scratch2[q] = nullptr; }
  }
};

// Whether riab_run takes the whole run as ONE launch (k_step MODE 3, or 4 with a motion source; see RunK) under the
// conditions DESIGN.md §4 lists; a motion source's whole run does not look at xi or the parity taps.  d: population 0 on
// its ring bases (make_out's alignment checks then hold for every row).
int whole_run_applies(const EnvK& ek, const riab_agents& ag, const riab_motion_params& prm, const riab_step_io& io,
                      const riab_motion_source* src, const riab_population* pops, int n_pops,
                      const riab_agent_history* hist, Pop& d, bool& yes) {
  yes = false;
  if (n_pops != 1 || !step_kernel_walls(ek) || getenv("RIAB_NO_WHOLE_RUN") != nullptr || io.drift_velocity != nullptr || io.pos_mirror != nullptr ||
      (src == nullptr && (io.xi != nullptr || io.collision_mask || io.first_hit || io.n_iters)))
    return 0;
  const riab_population& pp = pops[0];
  if ((pp.kind != RIAB_CELLS_PLACE && pp.kind != RIAB_CELLS_GRID && pp.kind != RIAB_CELLS_PWN) || pp.rates_ring == nullptr ||
      pp.ring_rows <= 0 || pp.noise.noise_std != 0.f)
    return 0;
  riab_rates_out ro = pp.out;
  ro.rates_row = pp.rates_ring; ro.spikes_row = pp.spikes_ring;
  riab_neuron_noise nz = pp.noise;
  nz.dt = prm.dt;
  int rc;
  if ((rc = make_pop(ek, pp.kind, pp.cells, &ro, &nz, prm.dt, ag, d))) return rc;
  const OutK& ok = d.out;
  const long long A = ag.n_agents;
  const int ct = d.n_pad / 4;
  const bool rows_ok = ((A * ok.ld) % 4 == 0) && ((A * ok.spike_ld) % 4 == 0);        // every ring row stays 16-byte aligned
  const bool lean = ok.vec_ok && rows_ok && (d.n_cells % 4 == 0) && ct <= RW * 32 &&
                    (ok.spikes == nullptr || (ag.id_offset & 1) == 0) &&
                    (4 % lean_groups(ct, 8) == 0) && (4 % lean_groups(ct, 4) == 0);      // groups divide the 4 producers
  // with a spike ring of one row a producer's clear of step s+1's rows could land before the consumers' RED.OR of step s
  yes = d.step_policy && lean && (hist == nullptr || hist->ring == nullptr || hist->ring_rows > 0) &&
        (pp.spikes_ring == nullptr || pp.ring_rows >= 2);
  return 0;
}

// The schedule of a riab_run: WHOLE (one launch), SKEWED or PLAIN, and the order of a step's populations.
struct RunPlan {
  enum { PLAIN, SKEWED, WHOLE } sched = PLAIN;
  bool motion_alone = false;      // PLAIN: the motion kernel runs on its own first, else population 0's launch takes the step
  std::vector<int> order;
  Pop whole;                      // WHOLE: the population
};

int plan_run(const EnvK& ek, const riab_agents& ag, const riab_motion_params& prm, const riab_step_io& io,
             const riab_motion_source* src, const riab_population* pops, int n_pops, const riab_agent_history* hist,
             RunPlan& plan) {
  bool whole;
  int rc;
  if ((rc = whole_run_applies(ek, ag, prm, io, src, pops, n_pops, hist, plan.whole, whole))) return rc;
  if (whole) {
    plan.sched = RunPlan::WHOLE;
    return 0;
  }
  // A FeedForwardLayer reads other populations' rows of the same step and masks the agents whose position of that step is
  // NaN, so an Agent with one keeps the plain schedule: the positions advance before any population of the step.
  bool any_ffl = false;
  for (int p = 0; p < n_pops; ++p) any_ffl = any_ffl || ffl_like(pops[p].kind);
  // Skewed schedule (population 0 has a k_step policy): motion(0) alone, then per step one kernel that evaluates rates(s)
  // of the current positions while its producer warps already run motion(s+1); the last step is rates only.  Same results
  // as the plain sequence, but the float64 motion chain never gates the rate warps.  A motion source keeps the plain
  // schedule (its motion kernel is cheap next to the rates).
  const bool skew = n_pops >= 1 && has_step_policy(pops[0].kind, pops[0].cells) && !any_ffl && io.xi == nullptr &&
                    !io.collision_mask && !io.first_hit && !io.n_iters && src == nullptr && step_kernel_walls(ek);
  plan.sched = skew ? RunPlan::SKEWED : RunPlan::PLAIN;
  plan.motion_alone = !skew && (src != nullptr || n_pops == 0 || ffl_like(pops[0].kind) || !step_kernel_walls(ek));
  // populations 1.. first (they read the positions of step st), population 0 last (it may advance them); then the
  // FeedForwardLayers in registration order, after every row they read of this step exists
  for (int p = skew ? 1 : 0; p < n_pops; ++p)
    if (!ffl_like(pops[p].kind)) plan.order.push_back(p);
  if (skew) plan.order.push_back(0);
  for (int p = 0; p < n_pops; ++p)
    if (ffl_like(pops[p].kind)) plan.order.push_back(p);
  return 0;
}

// riab_run / riab_run_src.  src: NULL for the random motion, else an imported trajectory (already checked).
int run_impl(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm, const riab_step_io* io,
             const riab_motion_source* src, const riab_population* pops, int32_t n_pops,
             const riab_agent_history* hist, int64_t n_steps, void* stream) {
  if (agents == nullptr || io == nullptr || n_pops < 0 || (n_pops > 0 && pops == nullptr))
    return fail(RIAB_ERR_INVALID, "riab_run: bad argument");
  if (n_steps <= 0) return 0;
  EnvK ek;
  RunPlan plan;
  int rc;
  if ((rc = check_agents(agents)) || (rc = make_env(env, ek)) || (rc = check_motion(prm)) ||
      (rc = plan_run(ek, *agents, *prm, *io, src, pops, n_pops, hist, plan)))
    return rc;
  const int64_t A = agents->n_agents;
  const bool agent_ring = hist != nullptr && hist->ring != nullptr && hist->ring_rows > 0;
  cudaStream_t s = (cudaStream_t)stream;
  if (plan.sched == RunPlan::WHOLE) {
    const riab_population& pp = pops[0];
    RunK run;
    memset(&run, 0, sizeof(run));
    run.n_steps = n_steps;
    run.rates_ring = pp.rates_ring; run.spikes_ring = pp.spikes_ring;
    run.ring_rows = pp.ring_rows; run.ring_next = pp.ring_next;
    if (agent_ring) {
      run.hist_ring = hist->ring; run.hist_rows = hist->ring_rows; run.hist_next = hist->ring_next;
    }
    riab_step_io io0 = *io;
    io0.history_row = nullptr;
    if (src != nullptr && (rc = make_src(src, A, run.src))) return rc;
    return src ? launch_pop<4>(ek, *agents, *prm, io0, plan.whole, s, nullptr, &run)
               : launch_pop<3>(ek, *agents, *prm, io0, plan.whole, s, nullptr, &run);
  }

  riab_motion_source src_st;                          // step st's clock: t_st = t_{st-1} + dt
  if (src != nullptr) src_st = *src;
  auto step_io = [&](int64_t st) {
    riab_step_io sio = *io;
    sio.step = io->step + (uint64_t)st;
    sio.history_row = agent_ring ? ring_row(hist->ring, hist->ring_next + st, hist->ring_rows, A * 8) : nullptr;
    return sio;
  };
  if (plan.sched == RunPlan::SKEWED) {
    const riab_step_io s0 = step_io(0);
    if ((rc = riab_agent_update(agents, env, prm, &s0, stream))) return rc;
  }
  PipeScope pipe;
  if ((rc = pipe.begin(pops, n_pops, A, n_steps, s))) return rc;
  // PhasePrecessingPlaceCells: each population's clock of step st, t_st = t_{st-1} + dt like Agent.update's
  std::vector<double> t_pop((size_t)n_pops, 0.0);
  for (int p = 0; p < n_pops; ++p)
    if (pops[p].kind == RIAB_CELLS_PPPC && pops[p].cells != nullptr) t_pop[p] = ((const riab_pppc_cells*)pops[p].cells)->t;
  for (int64_t st = 0; st < n_steps; ++st) {
    if (pipe.pipe) pipe.pipe->step = st;
    const riab_step_io sio = step_io(st);
    if (plan.motion_alone) {
      if (src == nullptr) {
        rc = riab_agent_update(agents, env, prm, &sio, stream);
      } else {
        rc = riab_agent_update_src(agents, env, prm, &sio, &src_st, stream);
        src_st.t = src_st.t + prm->dt;
      }
      if (rc) return rc;
    }
    for (const int p : plan.order) {
      const riab_population& pp = pops[p];
      if (pp.rates_ring == nullptr || pp.ring_rows <= 0) return fail(RIAB_ERR_INVALID, "population %d: no rates ring", p);
      riab_rates_out ro = pp.out;                   // on the ring bases: make_out's alignment checks hold for every row
      ro.rates_row = pp.rates_ring; ro.spikes_row = pp.spikes_ring;
      riab_neuron_noise nz = pp.noise;
      nz.step = pp.noise.step + (uint64_t)st; nz.dt = prm->dt;
      riab_td_cells tc;                             // an FFL population uses tc.ffl only
      riab_ffl_cells& fc = tc.ffl;
      riab_nnn_cells nc;
      riab_pppc_cells ppc;
      const void* cells = pp.cells;
      if (pp.kind == RIAB_CELLS_PPPC && pp.cells != nullptr) {
        ppc = *(const riab_pppc_cells*)pp.cells;
        ppc.t = t_pop[p];                           // the skewed launch evaluating step st's rates uses step st's phase
        cells = &ppc;
      }
      if (ffl_like(pp.kind)) {
        // inputs registered before the layer give this step's ring row, the others (the layer itself included) the
        // previous step's: before the first step, the row the caller passed
        int n_inputs;
        riab_ffl_input* inputs;
        if (pp.cells == nullptr) return fail(RIAB_ERR_INVALID, "population %d: cells NULL", p);
        if (pp.kind == RIAB_CELLS_NNN) {
          nc = *(const riab_nnn_cells*)pp.cells;
          if (nc.n_layers == 0)
            return fail(RIAB_ERR_UNSUPPORTED, "population %d: a NeuralNetworkNeurons module the kernel does not run", p);
          cells = &nc;
          n_inputs = nc.n_inputs; inputs = nc.inputs;
        } else {
          if (pp.kind == RIAB_CELLS_TD) {
            tc = *(const riab_td_cells*)pp.cells;
            cells = &tc;
          } else {
            fc = *(const riab_ffl_cells*)pp.cells;
            cells = &fc;
          }
          n_inputs = fc.n_inputs; inputs = fc.inputs;
        }
        for (int i = 0; i < n_inputs && i < RIAB_FFL_MAX_INPUTS; ++i) {
          riab_ffl_input& in = inputs[i];
          if (in.population < 0 || in.population >= n_pops || (in.lag == 0) != (in.population < p) || in.lag < 0 || in.lag > 1)
            return fail(RIAB_ERR_INVALID, "population %d: FeedForwardLayer input %d (population %d, lag %d) out of order", p, i,
                        in.population, in.lag);
          const riab_population& ip = pops[in.population];
          if (in.lag == 1 && st == 0) continue;
          if (in.lag == 1 && ip.ring_rows < 2)
            return fail(RIAB_ERR_INVALID, "population %d feeds a FeedForwardLayer with one step of lag: it needs 2 ring rows", in.population);
          in.rows_dev = ring_row(ip.rates_ring, ip.ring_next + st - in.lag, ip.ring_rows, A * ip.out.ld);
          in.ld = ip.out.ld;
        }
        if (pp.kind == RIAB_CELLS_TD && tc.self_input >= 0 && tc.self_input < fc.n_inputs) {
          fc.inputs[tc.self_input].rows_dev = tc.fr_prev_dev;       // firingrate_last, as in the stepped update
          fc.inputs[tc.self_input].ld = tc.ld;
        }
      }
      Pop d;
      if ((rc = make_pop(ek, pp.kind, cells, &ro, &nz, prm->dt, *agents, d))) return rc;
      d.out.rates = ring_row(pp.rates_ring, pp.ring_next + st, pp.ring_rows, A * pp.out.ld);
      if (d.out.spikes != nullptr) d.out.spikes = ring_row(pp.spikes_ring, pp.ring_next + st, pp.ring_rows, A * d.out.spike_ld);
      if (p != 0 || plan.motion_alone) rc = launch_pop<0>(ek, *agents, kNoMotion, kNoStep, d, s, pipe.pipe);
      else if (plan.sched == RunPlan::PLAIN) rc = step_fused(agents, env, ek, prm, &sio, d, s, pipe.pipe);
      else if (st + 1 < n_steps) rc = launch_pop<2>(ek, *agents, *prm, step_io(st + 1), d, s);   // its motion: step st+1's
      else rc = launch_pop<0>(ek, *agents, kNoMotion, kNoStep, d, s);
      if (rc) return rc;
    }
    for (int p = 0; p < n_pops; ++p) t_pop[p] = t_pop[p] + prm->dt;
  }
  return 0;
}

// ---- host-buffer motion step on two streams (see include/riab_b200.h)
struct HostIo {
  cudaStream_t side = nullptr;
  cudaEvent_t up_done = nullptr, motion_done = nullptr, pos_done = nullptr;
  bool pos_inflight = false;
};
thread_local HostIo g_hostio[16];
int hostio(HostIo*& h) {
  int dev = 0;
  RIAB_CUDA_OK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 16) return fail(RIAB_ERR_UNSUPPORTED, "device ordinal %d", dev);
  h = &g_hostio[dev];
  if (h->side == nullptr) {
    RIAB_CUDA_OK(cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking));
    RIAB_CUDA_OK(cudaEventCreateWithFlags(&h->up_done, cudaEventDisableTiming));
    RIAB_CUDA_OK(cudaEventCreateWithFlags(&h->motion_done, cudaEventDisableTiming));
    RIAB_CUDA_OK(cudaEventCreateWithFlags(&h->pos_done, cudaEventDisableTiming));
  }
  return 0;
}
}  // namespace

// ------------------------------------------------- DumbAgent, ShiftAgent, ReplayAgent
// One agent per thread: the position of this lead step (riab_subagent.cuh).  A replaying ReplayAgent advances its sham
// agent's rollout with motion_step in place.
template <int KIND>
__global__ void __launch_bounds__(128) k_subagent(const riab_subagent sa, const riab_motion_params mp, const MotionDerived md,
                                                  const EnvK env) {
  extern __shared__ __align__(128) unsigned char dyn_sub[];           // env.W * 32 bytes of walls (none for a ShiftAgent)
  double* s_walls = reinterpret_cast<double*>(dyn_sub);
  __shared__ uint64_t s_bar;
  if (KIND != RIAB_SUBAGENT_SHIFT) stage_walls(s_walls, &s_bar, env);
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= sa.n_agents) return;
  const double2 lp = reinterpret_cast<const double2*>(sa.lead_pos)[i];
  const unsigned long long gid = (unsigned long long)(sa.id_offset + i);
  double px = lp.x, py = lp.y;
  if (KIND == RIAB_SUBAGENT_SHIFT) {                                  // SubAgent.py:476
    const double2 hd = reinterpret_cast<const double2*>(sa.lead_head_direction)[i];
    px = (D(lp.x) + D(hd.x) * D(sa.shift_m)).v;
    py = (D(lp.y) + D(hd.y) * D(sa.shift_m)).v;
  } else if (KIND == RIAB_SUBAGENT_DUMB) {                            // SubAgent.py:151-179
    double2 d = reinterpret_cast<const double2*>(sa.displacement)[i];
    double2 v = reinterpret_cast<const double2*>(sa.displacement_velocity)[i];
    double n1, n2;
    if (sa.xi_displacement != nullptr) {
      n1 = sa.xi_displacement[2 * i]; n2 = sa.xi_displacement[2 * i + 1];
    } else {
      uint32_t c[4];
      philox_ctr(c, gid, 0u, sa.step, RIAB_STREAM_DUMB, 0u);
      philox_normals(c, sa.seed, n1, n2);
    }
    const D dt(sa.dt), theta(sa.ou_theta), sigma(sa.ou_sigma), a(sa.acceleration_scale);
    dumb_spring(d.x, v.x, dt, theta, sigma, a, D(n1));
    dumb_spring(d.y, v.y, dt, theta, sigma, a, D(n2));
    dumb_wall_cut(lp.x, lp.y, d.x, d.y, s_walls, env.W);
    D qx = D(lp.x) + D(d.x), qy = D(lp.y) + D(d.y);
    if (sa.resample_pos != nullptr && env.polygon && !env_contains(qx.v, qy.v, s_walls, env.nb, env.h0, env.nh)) {
      qx = D(sa.resample_pos[2 * i]); qy = D(sa.resample_pos[2 * i + 1]);
    } else {
      apply_boundary(qx, qy, env.ext, s_walls, env.periodic != 0, env.polygon != 0, env.nb, env.h0, env.nh,
                     [&](uint32_t t, double& u1, double& u2) {
                       subagent_uniforms(sa.seed, gid, 1u + t, sa.step, RIAB_STREAM_DUMB, u1, u2);
                     });
    }
    D wx, wy;                                                         // :178, through the boundary when periodic
    step_displacement(qx, qy, D(lp.x), D(lp.y), env.periodic != 0, env.scale, wx, wy);
    reinterpret_cast<double2*>(sa.displacement)[i] = make_double2(wx.v, wy.v);
    reinterpret_cast<double2*>(sa.displacement_velocity)[i] = v;
    px = qx.v; py = qy.v;
  } else {                                                            // SubAgent.py:391-423
    uint8_t rep = sa.replaying[i];
    double* st = sa.replay_state + (size_t)RIAB_REPLAY_FIELDS * i;
    const double* tap = sa.replay_draws != nullptr ? sa.replay_draws + 6 * i : nullptr;
    if (!rep) {
      double u, u_speed;
      if (tap != nullptr) { u = tap[0]; u_speed = 0.0; }
      else subagent_uniforms(sa.seed, gid, 0u, sa.step, RIAB_STREAM_REPLAY, u, u_speed);
      if (!(u > sa.p_start)) {                                       // :395-407: a replay starts
        double u_dur, u_dir;
        if (tap == nullptr) subagent_uniforms(sa.seed, gid, 1u, sa.step, RIAB_STREAM_REPLAY, u_dur, u_dir);
        const double speed = tap ? tap[1] : rayleigh_of(sa.mean_speed, u_speed);
        const double raw = tap ? tap[2] : rayleigh_of(sa.mean_duration, u_dur);
        const double half = (D(sa.mean_duration) / D(2.0)).v;
        const double duration = half > raw ? half : raw;              // max(rayleigh, mean / 2)
        const double dir = tap ? tap[5] : (D(2.0 * M_PI) * D(u_dir)).v;   // np.random.uniform(0, 2 pi)
        double x0, y0;
        if (tap != nullptr) {
          x0 = tap[3]; y0 = tap[4];
        } else {
          // sample_positions(n=1, "random") (Environment.py:561-600): uniform in the extent, re-drawn until inside
          for (uint32_t k = 0; k < 1024u; ++k) {
            double ux, uy;
            subagent_uniforms(sa.seed, gid, 2u + k, sa.step, RIAB_STREAM_REPLAY, ux, uy);
            x0 = (D(env.ext[0]) + D(env.ext[1] - env.ext[0]) * D(ux)).v;
            y0 = (D(env.ext[2]) + D(env.ext[3] - env.ext[2]) * D(uy)).v;
            if (!env.polygon || env_contains(x0, y0, s_walls, env.nb, env.h0, env.nh)) break;
          }
        }
        // initialise_position_and_velocity (Agent.py:523-535); the sham's measured velocity, head direction and
        // distance carry over from its previous replay
        AgentState s;
        load_agent(sa.sham, i, s);
        s.px = x0; s.py = y0;
        s.vx = (D(mp.speed_mean) * D(cos(dir))).v;
        s.vy = (D(mp.speed_mean) * D(sin(dir))).v;
        s.rot = 0.0;
        store_agent(sa.sham, i, s);
        st[0] = speed; st[1] = duration;
        st[2] = sa.t; st[3] = (D(sa.t) + D(duration)).v;
        st[4] = (D(s.dist) + D(1.1) * D(speed) * D(duration)).v;     // :408's stop distance
        st[5] = s.dist;
        st[6] = s.dist; st[7] = x0; st[8] = y0;
        sa.replay_count[2 * i] += 1;
        sa.replay_count[2 * i + 1] = 0;
        rep = 1;
        px = x0; py = y0;
      }
    } else {
      // :416-418 while t < end: the query distance; on the step the replay ends (:420-423) the rollout is finished to
      // its stop distance instead, as the reference's eager one was: the sham's state carries over into the next replay
      const bool live = sa.t < st[3];
      const double q = live ? (D(st[0]) * (D(sa.t) - D(st[2]))).v : INFINITY;
      AgentState s;
      load_agent(sa.sham, i, s);
      long long k = sa.replay_count[2 * i + 1];
      const unsigned long long r = (unsigned long long)(sa.replay_count[2 * i] - 1);
      const double start = st[5], stop = st[4];
      double d_prev = st[6], x_prev = st[7], y_prev = st[8];
      const double f1 = __longlong_as_double((long long)sa.seed);
      while ((live && k == 0) || ((D(s.dist) - D(start)).v < q && s.dist < stop)) {
        d_prev = s.dist; x_prev = s.px; y_prev = s.py;
        double n1, n2;
        if (sa.xi_replay != nullptr && k < sa.xi_steps) {
          n1 = sa.xi_replay[2 * (i * sa.xi_steps + k)];
          n2 = sa.xi_replay[2 * (i * sa.xi_steps + k) + 1];
        } else {
          uint32_t c[4];
          philox_ctr(c, gid, (uint32_t)r, (uint64_t)k, RIAB_STREAM_REPLAY_FWD, 0u);
          philox_normals(c, sa.seed, n1, n2);
        }
        // exactly-zero displacement / polygon re-draw fall-backs: keyed by replay, step and agent
        const double f2 = __longlong_as_double((long long)(((unsigned long long)k | (r << 32)) ^ (gid << 20) ^
                                                           0x5245504c41590000ull));
        motion_step<false>(s, s_walls, env.W, mp, md, env.ext, env.periodic != 0, env.scale, env.polygon != 0, env.nb, env.h0,
                           env.nh, n1, n2, false, 0.0, 0.0, f1, f2, nullptr, nullptr, nullptr);
        ++k;
      }
      store_agent(sa.sham, i, s);
      sa.replay_count[2 * i + 1] = k;
      st[6] = d_prev; st[7] = x_prev; st[8] = y_prev;
      if (live) {
        // interp1d over the distances relative to the start (:411-418) between the kept pair
        const double lo = (D(d_prev) - D(start)).v, hi = (D(s.dist) - D(start)).v;
        if (hi >= q && q >= lo) {
          px = interp_linear(q, lo, hi, x_prev, s.px);
          py = interp_linear(q, lo, hi, y_prev, s.py);
        } else {
          px = py = theta_nan();
        }
      } else {
        rep = 0;                                                      // back to the lead
      }
    }
    sa.replaying[i] = rep;
  }
  reinterpret_cast<double2*>(sa.out_pos)[i] = make_double2(px, py);
}

// ===========================================================================
extern "C" {


int riab_abi_version(void) { return RIAB_ABI_VERSION; }
const char* riab_last_error(void) { return g_err; }
int riab_history_rate_maps(const riab_history_view* h, const double* edges_x_dev, int32_t n_edges_x,
                           const double* edges_y_dev, int32_t n_edges_y, double* sum_dev, uint64_t* count_dev, void* stream) {
  if (h == nullptr || h->agent_ring == nullptr || edges_x_dev == nullptr || edges_y_dev == nullptr || count_dev == nullptr)
    return fail(RIAB_ERR_INVALID, "riab_history_rate_maps: NULL argument");
  if (n_edges_x < 2 || n_edges_y < 2 || h->agent_ring_rows <= 0 || h->n_steps < 0 || h->n_agents <= 0)
    return fail(RIAB_ERR_INVALID, "riab_history_rate_maps: bad sizes");
  if (h->rates_ring != nullptr && (sum_dev == nullptr || h->rates_ring_rows <= 0 || h->ld < h->n_cells))
    return fail(RIAB_ERR_INVALID, "riab_history_rate_maps: rates ring without sum_dev / ld < n_cells");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t bins = (size_t)(n_edges_x - 1) * (size_t)(n_edges_y - 1);
  RIAB_CUDA_OK(cudaMemsetAsync(count_dev, 0, bins * sizeof(uint64_t), s));
  if (h->rates_ring != nullptr) RIAB_CUDA_OK(cudaMemsetAsync(sum_dev, 0, bins * (size_t)h->ld * sizeof(double), s));
  const long long n_samples = h->n_steps * h->n_agents;
  if (n_samples == 0) return 0;
  int sms, rc;
  if ((rc = num_sms(sms))) return rc;
  long long blocks = (n_samples + NT / 32 - 1) / (NT / 32);
  if (blocks > sms * 8ll) blocks = sms * 8ll;
  k_history_maps<<<(unsigned)blocks, NT, 0, s>>>(*h, edges_x_dev, n_edges_x, edges_y_dev, n_edges_y, sum_dev,
                                                 (unsigned long long*)count_dev);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

int64_t riab_launch_count(void) { return (int64_t)g_launches.load(); }
int riab_stream_synchronize(void* stream) {
  RIAB_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

int riab_agent_update(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm,
                      const riab_step_io* io, void* stream) {
  EnvK ek;
  int rc;
  if ((rc = check_agents(agents)) || (rc = make_env(env, ek)) || (rc = check_motion(prm))) return rc;
  if (io == nullptr) return fail(RIAB_ERR_INVALID, "io is NULL");
  if (agents->n_agents == 0) return 0;
  const unsigned grid = (unsigned)((agents->n_agents + 127) / 128);
  const bool rec = io->collision_mask || io->first_hit || io->n_iters;
  MotionDerived md;
  derive_motion(*prm, md);
  const size_t smem = motion_walls_bytes(ek);
  if (rec) k_agent_update<true><<<grid, 128, smem, (cudaStream_t)stream>>>(*agents, *prm, md, *io, ek);
  else k_agent_update<false><<<grid, 128, smem, (cudaStream_t)stream>>>(*agents, *prm, md, *io, ek);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------- imported / forced motion
int riab_trajectory_build(const riab_trajectory* tr, const double* times_host, void* stream) {
  if (tr == nullptr || times_host == nullptr || tr->times_dev == nullptr || tr->y_dev == nullptr || tr->M_dev == nullptr)
    return fail(RIAB_ERR_INVALID, "riab_trajectory_build: NULL argument");
  const long long T = tr->T, ncol = 2 * tr->n_traj;
  if (T < 4 || tr->n_traj <= 0) return fail(RIAB_ERR_INVALID, "riab_trajectory_build: T = %lld (>= 4 samples), n_traj = %lld", T, (long long)tr->n_traj);
  for (long long i = 0; i + 1 < T; ++i)
    if (!(times_host[i + 1] > times_host[i])) return fail(RIAB_ERR_INVALID, "riab_trajectory_build: times not strictly increasing at %lld", i);
  std::vector<double> fac((size_t)(4 * (T - 2) + T - 1));
  traj_factors(times_host, T, fac.data());
  cudaStream_t s = (cudaStream_t)stream;
  double* fac_dev = nullptr;
  RIAB_CUDA_OK(cudaMallocAsync((void**)&fac_dev, fac.size() * sizeof(double), s));
  RIAB_CUDA_OK(cudaMemcpyAsync(fac_dev, fac.data(), fac.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  k_traj_build<<<(unsigned)((ncol + 127) / 128), 128, 0, s>>>(tr->y_dev, tr->M_dev, fac_dev, T, ncol);
  g_launches++;
  const cudaError_t e = cudaGetLastError();
  RIAB_CUDA_OK(cudaFreeAsync(fac_dev, s));
  // the pageable source of the copy must outlive it
  RIAB_CUDA_OK(cudaStreamSynchronize(s));
  if (e != cudaSuccess) return fail(RIAB_ERR_CUDA, "k_traj_build: %s", cudaGetErrorString(e));
  return 0;
}


int riab_agent_update_src(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm,
                          const riab_step_io* io, const riab_motion_source* src, void* stream) {
  if (src == nullptr || src->kind == RIAB_MOTION_RANDOM) return riab_agent_update(agents, env, prm, io, stream);
  EnvK ek;
  SrcK sk;
  int rc;
  if ((rc = check_agents(agents)) || (rc = make_env(env, ek)) || (rc = check_motion(prm))) return rc;
  if (io == nullptr) return fail(RIAB_ERR_INVALID, "io is NULL");
  if ((rc = make_src(src, agents->n_agents, sk))) return rc;
  if (agents->n_agents == 0) return 0;
  MotionDerived md;
  derive_motion(*prm, md);
  k_agent_update_src<<<(unsigned)((agents->n_agents + 127) / 128), 128, 0, (cudaStream_t)stream>>>(*agents, *prm, md, *io, sk, ek);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------- ThetaSequenceAgent
// One agent per thread: append the lead's row to the look-behind ring, then the sweep position of this step
// (riab_theta.cuh).  Look-ahead steps advance the agent's forward rollout with motion_step in place.
__global__ void __launch_bounds__(128) k_theta_seq(const riab_theta_seq ts, const riab_motion_params mp,
                                                   const MotionDerived md, const EnvK env) {
  extern __shared__ __align__(128) unsigned char dyn_theta[];         // env.W * 32 bytes of walls
  double* s_walls = reinterpret_cast<double*>(dyn_theta);
  __shared__ uint64_t s_bar;
  stage_walls(s_walls, &s_bar, env);
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ts.n_agents) return;
  const long long A = ts.n_agents, R = ts.ring_rows;
  const double2 lp = reinterpret_cast<const double2*>(ts.lead_pos)[i];
  const double ld = ts.lead_distance[i];
  const long long row = ts.ring_head * A + i;
  ts.ring[row] = lp.x;
  ts.ring[R * A + row] = lp.y;
  ts.ring[2 * R * A + row] = ld;

  double px = theta_nan(), py = theta_nan();
  const double target = __dadd_rn(ld, ts.offset);
  if (ts.phase == RIAB_THETA_BEHIND) {
    if (ld < ts.d_half) {
      px = lp.x; py = lp.y;
    } else {
      ThetaWindow W;
      W.ring = ts.ring; W.A = A; W.R = R; W.w = ts.window; W.i = i;
      W.first = ts.ring_head - (ts.window - 1);
      if (W.first < 0) W.first += R;
      theta_look_behind(W, target, px, py);
    }
  } else if (ts.phase == RIAB_THETA_AHEAD_FIRST || ts.phase == RIAB_THETA_AHEAD) {
    AgentState s;
    load_agent(ts.fwd, i, s);
    double2 prev;
    double d_prev;
    long long k;
    double stop;
    if (ts.phase == RIAB_THETA_AHEAD_FIRST) {
      const double2 lv = reinterpret_cast<const double2*>(ts.lead_velocity)[i];
      s.px = lp.x; s.py = lp.y; s.vx = lv.x; s.vy = lv.y;
      s.rot = ts.lead_rotational_velocity[i];
      s.dist = ld;
      k = 0;
      stop = __dadd_rn(ld, ts.forward_distance);
      ts.fwd_stop[i] = stop;
      d_prev = s.dist; prev = make_double2(s.px, s.py);
    } else {
      k = ts.fwd_steps[i];
      stop = ts.fwd_stop[i];
      d_prev = ts.fwd_pair[3 * i]; prev = make_double2(ts.fwd_pair[3 * i + 1], ts.fwd_pair[3 * i + 2]);
    }
    const unsigned long long gid = (unsigned long long)(ts.id_offset + i);
    const double f1 = __longlong_as_double((long long)ts.seed);
    while (k == 0 || (s.dist < target && s.dist < stop)) {
      d_prev = s.dist; prev = make_double2(s.px, s.py);
      double n1, n2;
      if (ts.xi_forward != nullptr && k < ts.xi_steps) {
        n1 = ts.xi_forward[2 * (i * ts.xi_steps + k)];
        n2 = ts.xi_forward[2 * (i * ts.xi_steps + k) + 1];
      } else {
        theta_fwd_normals(ts.seed, ts.rollout, (unsigned long long)k, gid, n1, n2);
      }
      // exactly-zero displacement / polygon re-draw fall-backs: keyed by rollout, step and agent
      const double f2 = __longlong_as_double((long long)(((unsigned long long)k | (ts.rollout << 32)) ^ (gid << 20) ^
                                                         0x5448455441000000ull));
      motion_step<false>(s, s_walls, env.W, mp, md, env.ext, env.periodic != 0, env.scale, env.polygon != 0, env.nb, env.h0,
                         env.nh, n1, n2, false, 0.0, 0.0, f1, f2, nullptr, nullptr, nullptr);
      ++k;
    }
    store_agent(ts.fwd, i, s);
    ts.fwd_steps[i] = k;
    ts.fwd_pair[3 * i] = d_prev; ts.fwd_pair[3 * i + 1] = prev.x; ts.fwd_pair[3 * i + 2] = prev.y;
    if (s.dist >= target && target >= d_prev) {
      px = interp_linear(target, d_prev, s.dist, prev.x, s.px);
      py = interp_linear(target, d_prev, s.dist, prev.y, s.py);
    }
  }
  // SubAgent.py:341-343: farther than d_half from the lead (a sweep interpolated across a periodic boundary) -> NaN
  if (px == px && py == py) {
    D vx, vy;
    step_displacement(D(px), D(py), D(lp.x), D(lp.y), env.periodic != 0, env.scale, vx, vy);
    if (dsqrt(vx * vx + vy * vy).v > ts.d_half) px = py = theta_nan();
  }
  reinterpret_cast<double2*>(ts.out_pos)[i] = make_double2(px, py);
}

int riab_theta_seq_step(const riab_theta_seq* ts, const riab_env* env, const riab_motion_params* fwd_prm, void* stream) {
  EnvK ek;
  int rc;
  if (ts == nullptr) return fail(RIAB_ERR_INVALID, "riab_theta_seq_step: ts is NULL");
  if ((rc = make_env(env, ek)) || (rc = check_motion(fwd_prm))) return rc;
  if (ts->phase < RIAB_THETA_NONE || ts->phase > RIAB_THETA_AHEAD) return fail(RIAB_ERR_INVALID, "bad theta phase %d", ts->phase);
  if (ts->n_agents < 0) return fail(RIAB_ERR_INVALID, "n_agents < 0");
  if (ts->n_agents == 0) return 0;
  if (!ts->lead_pos || !ts->lead_velocity || !ts->lead_rotational_velocity || !ts->lead_distance || !ts->ring ||
      !ts->fwd_pair || !ts->fwd_stop || !ts->fwd_steps || !ts->out_pos)
    return fail(RIAB_ERR_INVALID, "riab_theta_seq_step: NULL array");
  riab_agents fwd = ts->fwd;
  fwd.n_agents = ts->n_agents;
  if ((rc = check_agents(&fwd))) return rc;
  if (ts->ring_rows < 1 || ts->ring_head < 0 || ts->ring_head >= ts->ring_rows)
    return fail(RIAB_ERR_INVALID, "ring_head %lld outside a ring of %lld rows", (long long)ts->ring_head, (long long)ts->ring_rows);
  if (ts->phase == RIAB_THETA_BEHIND && (ts->window < 1 || ts->window > ts->ring_rows))
    return fail(RIAB_ERR_INVALID, "window %lld outside [1, ring_rows = %lld]", (long long)ts->window, (long long)ts->ring_rows);
  if (ts->xi_forward != nullptr && ts->xi_steps < 0) return fail(RIAB_ERR_INVALID, "xi_steps < 0");
  MotionDerived md;
  derive_motion(*fwd_prm, md);
  k_theta_seq<<<(unsigned)((ts->n_agents + 127) / 128), 128, motion_walls_bytes(ek), (cudaStream_t)stream>>>(*ts, *fwd_prm, md, ek);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------- DumbAgent, ShiftAgent, ReplayAgent (k_subagent: before extern "C")
int riab_subagent_step(const riab_subagent* sa, const riab_env* env, const riab_motion_params* sham_prm, void* stream) {
  EnvK ek;
  int rc;
  if (sa == nullptr) return fail(RIAB_ERR_INVALID, "riab_subagent_step: sa is NULL");
  if ((rc = make_env(env, ek))) return rc;
  if (sa->kind < RIAB_SUBAGENT_SHIFT || sa->kind > RIAB_SUBAGENT_REPLAY) return fail(RIAB_ERR_INVALID, "bad SubAgent kind %d", sa->kind);
  if (sa->n_agents < 0) return fail(RIAB_ERR_INVALID, "n_agents < 0");
  if (sa->n_agents == 0) return 0;
  if (!sa->lead_pos || !sa->out_pos) return fail(RIAB_ERR_INVALID, "riab_subagent_step: NULL array");
  const unsigned grid = (unsigned)((sa->n_agents + 127) / 128);
  MotionDerived md{};
  riab_motion_params mp{};
  if (sa->kind == RIAB_SUBAGENT_SHIFT) {
    if (!sa->lead_head_direction) return fail(RIAB_ERR_INVALID, "riab_subagent_step: NULL lead_head_direction");
    k_subagent<RIAB_SUBAGENT_SHIFT><<<grid, 128, 0, (cudaStream_t)stream>>>(*sa, mp, md, ek);     // stages no walls
  } else if (sa->kind == RIAB_SUBAGENT_DUMB) {
    if (!sa->displacement || !sa->displacement_velocity) return fail(RIAB_ERR_INVALID, "riab_subagent_step: NULL displacement");
    k_subagent<RIAB_SUBAGENT_DUMB><<<grid, 128, motion_walls_bytes(ek), (cudaStream_t)stream>>>(*sa, mp, md, ek);
  } else {
    if (sham_prm == nullptr) return fail(RIAB_ERR_INVALID, "riab_subagent_step: a ReplayAgent needs sham_prm");
    if ((rc = check_motion(sham_prm))) return rc;
    if (!sa->replaying || !sa->replay_state || !sa->replay_count) return fail(RIAB_ERR_INVALID, "riab_subagent_step: NULL replay state");
    riab_agents sham = sa->sham;
    sham.n_agents = sa->n_agents;
    if ((rc = check_agents(&sham))) return rc;
    if (sa->xi_replay != nullptr && sa->xi_steps < 0) return fail(RIAB_ERR_INVALID, "xi_steps < 0");
    derive_motion(*sham_prm, md);
    k_subagent<RIAB_SUBAGENT_REPLAY><<<grid, 128, motion_walls_bytes(ek), (cudaStream_t)stream>>>(*sa, *sham_prm, md, ek);
  }
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// ----------------------------------------------------------------- PlaceCells
static int place_n_pad(int n) { return (n + CELL_PAD - 1) / CELL_PAD * CELL_PAD; }

int64_t riab_place_pack_floats(int32_t n_cells, int32_t n_inner_walls) {
  return (int64_t)place_n_pad(n_cells) * (4 + 2 * (n_inner_walls > 0 ? n_inner_walls : 0) + 4);
}

int riab_place_pack(const double* centres, const double* widths, int32_t n, const double* walls, int32_t n_walls,
                    int32_t n_boundary, const double* extent, int32_t geometry, riab_place_cells* meta, float* out) {
  if (!centres || !widths || !extent || !meta || !out || n <= 0) return fail(RIAB_ERR_INVALID, "riab_place_pack: bad argument");
  const int np = place_n_pad(n);
  const int n_inner = (geometry == RIAB_GEOM_EUCLIDEAN) ? 0 : (n_walls - n_boundary);
  if (n_inner < 0) return fail(RIAB_ERR_INVALID, "n_walls < n_boundary_walls");
  if (n_inner > 0 && !walls) return fail(RIAB_ERR_INVALID, "walls NULL");
  const double cxm = 0.5 * (extent[0] + extent[1]), cym = 0.5 * (extent[2] + extent[3]);
  const int64_t total = riab_place_pack_floats(n, n_inner);
  for (int64_t i = 0; i < total; ++i) out[i] = 0.f;
  float *cx = out, *cy = out + np, *kk = out + 2 * np;
  for (int i = 0; i < np; ++i) {
    if (i < n) {
      cx[i] = (float)(centres[2 * i] - cxm);
      cy[i] = (float)(centres[2 * i + 1] - cym);
      kk[i] = (float)(1.4426950408889634 / (2.0 * widths[i] * widths[i]));   // log2(e) / (2 w^2)
    } else { cx[i] = 1.0e3f; cy[i] = 1.0e3f; kk[i] = 0.f; }
  }
  {
    bool uniform = true;
    for (int i = 1; i < n; ++i) uniform = uniform && (widths[i] == widths[0]);
    const double hx = 0.5 * (extent[1] - extent[0]), hy = 0.5 * (extent[3] - extent[2]);
    double r2 = hx * hx + hy * hy;
    for (int i = 0; i < n; ++i) {
      const double c2 = (double)cx[i] * cx[i] + (double)cy[i] * cy[i];
      if (c2 > r2) r2 = c2;
    }
    meta->k_uniform = uniform ? kk[0] : 0.f;
    meta->r2_max = (float)r2;
    float* aa = out + 3 * (size_t)np;                     // -k |c|^2 of the float32-rounded centre
    for (int i = 0; i < np; ++i) aa[i] = (i < n && uniform) ? (float)(-(double)kk[0] * ((double)cx[i] * cx[i] + (double)cy[i] * cy[i])) : -1.0e5f;
  }
  meta->n_pad = np;
  meta->n_inner_walls = n_inner;
  meta->ep_valid = 0;
  for (int j = 0; j < 8; ++j) meta->eps[j] = 0.f;
  for (int j = 0; j < n_inner; ++j) {
    const double* w = walls + 4 * (n_boundary + j);
    float* fc = out + (size_t)(4 + 2 * j) * np;
    float* tc = out + (size_t)(5 + 2 * j) * np;
    double tmax = 1.0, dmax = 0.0;
    for (int cxi = 0; cxi < 2; ++cxi)
      for (int cyi = 0; cyi < 2; ++cyi) {            // agents live inside the box: bound |f|, |t| over its corners
        double f, t;
        wall_coords(extent[cxi], extent[2 + cyi], w[0], w[1], w[2], w[3], f, t);
        if (fabs(t) + 1.0 > tmax) tmax = fabs(t) + 1.0;
        if (fabs(f) > dmax) dmax = fabs(f);
      }
    double fcmax = 0.0;
    for (int i = 0; i < n; ++i) {
      double f, t;
      wall_coords(centres[2 * i], centres[2 * i + 1], w[0], w[1], w[2], w[3], f, t);
      if (fabs(t) + 1.0 > tmax) tmax = fabs(t) + 1.0;
      if (fabs(f) > fcmax) fcmax = fabs(f);
    }
    const double band = 2.0e-6 * (dmax + fcmax) * tmax;   // ~10x the float32 rounding error of M' and |D|
    for (int i = 0; i < np; ++i) {
      if (i < n) {
        double f, t;
        wall_coords(centres[2 * i], centres[2 * i + 1], w[0], w[1], w[2], w[3], f, t);
        fc[i] = (float)f; tc[i] = (float)t;
        // a centre (numerically) on the wall's line: (0,0) makes M' = 0, inside the band -> exact float64 path
        if (fabs(f) < 1.0e-6 * (dmax + fcmax)) { fc[i] = 0.f; tc[i] = 0.f; }
      } else { fc[i] = 1.f; tc[i] = -1.f; }
    }
    if (j < 8) meta->eps[j] = (float)band;
  }
  {                                                       // residuals of the centred centres (compensated direct form)
    float* cxl = out + (size_t)(6 + 2 * n_inner) * np;
    float* cyl = out + (size_t)(7 + 2 * n_inner) * np;
    for (int i = 0; i < n; ++i) {
      cxl[i] = (float)((centres[2 * i] - cxm) - (double)cx[i]);
      cyl[i] = (float)((centres[2 * i + 1] - cym) - (double)cy[i]);
    }
  }
  if (geometry == RIAB_GEOM_GEODESIC && n_inner >= 1) {
    const double* w = walls + 4 * n_boundary;
    float* ce0 = out + (size_t)(4 + 2 * n_inner) * np;
    float* ce1 = out + (size_t)(5 + 2 * n_inner) * np;
    for (int e = 0; e < 2; ++e) {
      const double ex = w[2 * e], ey = w[2 * e + 1];
      if (ex > extent[0] && ex < extent[1] && ey > extent[2] && ey < extent[3]) meta->ep_valid |= (1 << e);
    }
    for (int i = 0; i < n; ++i) {
      const double a = centres[2 * i] - w[0], b = centres[2 * i + 1] - w[1];
      const double c = centres[2 * i] - w[2], d = centres[2 * i + 1] - w[3];
      ce0[i] = (float)sqrt(a * a + b * b);
      ce1[i] = (float)sqrt(c * c + d * d);
    }
  }
  return 0;
}

int riab_place_rates(const double* pos_dev, int64_t n_pos, const riab_env* env, const riab_place_cells* pc,
                     float* out_dev, int64_t ld_out, void* stream) {
  return rates_at(RIAB_CELLS_PLACE, pc, pos_dev, n_pos, env, nullptr, nullptr, nullptr, out_dev, ld_out, stream);
}

// ------------------------------------------------------------------ GridCells
int64_t riab_grid_pack_floats(int32_t n_cells) { return (int64_t)place_n_pad(n_cells) * 9; }

int riab_grid_pack(const double* gridscales, const double* phase_offsets, const double* w, int32_t n,
                   const double* extent, riab_grid_cells* meta, float* out) {
  if (!gridscales || !phase_offsets || !w || !extent || !meta || !out || n <= 0)
    return fail(RIAB_ERR_INVALID, "riab_grid_pack: bad argument");
  const int np = place_n_pad(n);
  const double cxm = 0.5 * (extent[0] + extent[1]), cym = 0.5 * (extent[2] + extent[3]);
  for (int64_t i = 0; i < (int64_t)np * 9; ++i) out[i] = 0.f;
  // The radian form rounds phases of up to |k| r_max (r_max: half-diagonal of the box) to float32 and hands them to
  // __cosf: its rate error grows like 1.1e-7 |k| r_max of the rate scale (1.7e-6 with the default grid scales in the unit
  // box, 1.6e-5 at scale 10).  Above |k| r_max = 40 (4.3e-6) the block holds turns for the compensated phase instead.
  double kr = 0.0;
  const double rmax = 0.5 * hypot(extent[1] - extent[0], extent[3] - extent[2]);
  for (int i = 0; i < n; ++i) kr = fmax(kr, (2.0 * M_PI) / fabs(gridscales[i]) * rmax);
  const int turns = kr > 40.0 ? 1 : 0;
  const double unit = turns ? 1.0 / (2.0 * M_PI) : 1.0;
  for (int i = 0; i < n; ++i) {
    const double kappa = (2.0 * M_PI) / gridscales[i];
    // origin = gridscale * phase_offset / (2 pi)   (Neurons.py:1191)
    const double ox = gridscales[i] * phase_offsets[2 * i] / (2.0 * M_PI) - cxm;
    const double oy = gridscales[i] * phase_offsets[2 * i + 1] / (2.0 * M_PI) - cym;
    for (int k = 0; k < 3; ++k) {
      const double wx = w[6 * i + 2 * k], wy = w[6 * i + 2 * k + 1];
      double ph = kappa * (ox * wx + oy * wy);
      ph = remainder(ph, 2.0 * M_PI);
      out[(size_t)(3 * k + 0) * np + i] = (float)(kappa * wx * unit);
      out[(size_t)(3 * k + 1) * np + i] = (float)(kappa * wy * unit);
      out[(size_t)(3 * k + 2) * np + i] = (float)(ph * unit);
    }
  }
  meta->n_pad = np;
  meta->phase_turns = turns;
  return 0;
}

int riab_grid_rates(const double* pos_dev, int64_t n_pos, const riab_env* env, const riab_grid_cells* gc,
                    float* out_dev, int64_t ld_out, void* stream) {
  return rates_at(RIAB_CELLS_GRID, gc, pos_dev, n_pos, env, nullptr, nullptr, nullptr, out_dev, ld_out, stream);
}

// ----------------------------------------------------------- PlaneWaveNeurons
int64_t riab_pwn_pack_floats(int32_t n_cells) { return (int64_t)place_n_pad(n_cells) * 5; }

int riab_pwn_pack(const double* phase_offsets, const double* w, const double* wavescales, int32_t n, const double* extent,
                  int32_t phase_form, riab_pwn_cells* meta, float* out) {
  if (!phase_offsets || !w || !wavescales || !extent || !meta || !out || n <= 0 || phase_form < -1 || phase_form > 1)
    return fail(RIAB_ERR_INVALID, "riab_pwn_pack: bad argument");
  const int np = place_n_pad(n);
  const double cxm = 0.5 * (extent[0] + extent[1]), cym = 0.5 * (extent[2] + extent[3]);
  const double rmax = 0.5 * hypot(extent[1] - extent[0], extent[3] - extent[2]);
  for (int64_t i = 0; i < (int64_t)np * 5; ++i) out[i] = 0.f;
  // The radian form's rate error grows like 1.2e-7 |2 pi k| r_max of the span (r_max: the box's half-diagonal), as for
  // GridCells: past |2 pi k| r_max = 40 (4.8e-6) the block holds turns for the compensated phase (riab_pwn.cuh).
  double kr = 0.0;
  for (int i = 0; i < n; ++i) {
    const double kx = w[2 * i] / wavescales[i], ky = w[2 * i + 1] / wavescales[i];
    if (!(std::isfinite(kx) && std::isfinite(ky) && std::isfinite(phase_offsets[2 * i]) && std::isfinite(phase_offsets[2 * i + 1])))
      return fail(RIAB_ERR_INVALID, "riab_pwn_pack: cell %d: w / wavescale or phase offset not finite", i);
    kr = fmax(kr, 2.0 * M_PI * hypot(kx, ky) * rmax);
  }
  const int turns = phase_form >= 0 ? phase_form : (kr > 40.0 ? 1 : 0);
  for (int i = 0; i < n; ++i) {
    const double kx = w[2 * i] / wavescales[i], ky = w[2 * i + 1] / wavescales[i];
    const double ph = remainder(kx * (phase_offsets[2 * i] - cxm) + ky * (phase_offsets[2 * i + 1] - cym), 1.0);   // turns
    if (turns) {
      const float hx = (float)kx, hy = (float)ky;
      out[(size_t)0 * np + i] = hx;
      out[(size_t)1 * np + i] = hy;
      out[(size_t)2 * np + i] = (float)(kx - (double)hx);
      out[(size_t)3 * np + i] = (float)(ky - (double)hy);
      out[(size_t)4 * np + i] = (float)ph;
    } else {
      out[(size_t)0 * np + i] = (float)(2.0 * M_PI * kx);
      out[(size_t)1 * np + i] = (float)(2.0 * M_PI * ky);
      out[(size_t)4 * np + i] = (float)(2.0 * M_PI * ph);
    }
  }
  meta->n_pad = np;
  meta->phase_turns = turns;
  return 0;
}

int riab_pwn_rates(const double* pos_dev, int64_t n_pos, const riab_env* env, const riab_pwn_cells* cells, float* out_dev,
                   int64_t ld_out, void* stream) {
  return rates_at(RIAB_CELLS_PWN, cells, pos_dev, n_pos, env, nullptr, nullptr, nullptr, out_dev, ld_out, stream);
}

// ------------------------------------------------------------------------ BVC
static int bvc_n_pad(int n) { return (n + BVC_CT - 1) / BVC_CT * BVC_CT; }

int64_t riab_bvc_pack_floats(int32_t n_cells, int32_t T) {
  const int64_t np = bvc_n_pad(n_cells);
  return 3 * np + np * (int64_t)T + 3 * np + 2 * (int64_t)T + np + 2 * (np / 32);
}
// Cut-off of the angular windows: a von Mises weight (peak 1) below 2^-30 is dropped.  The dropped part of a rate is at
// most T 2^-30 / norm of the population's peak rate (norm = sum of the peak-1 weights >= 1), below float32 resolution of the sum.
static const double BVC_VM_CUT = 9.313225746154785e-10;
int64_t riab_bvc_scratch_floats(int64_t n_pos, int32_t T) {
  return ((n_pos + BVC_AT - 1) / BVC_AT) * (int64_t)T * BVC_AT;
}

int riab_bvc_pack(const double* mu_d, const double* mu_t, const double* sg_d, const double* sg_t, int32_t n,
                  const double* test_angles, int32_t T, riab_bvc_cells* meta, float* out) {
  if (!mu_d || !mu_t || !sg_d || !sg_t || !test_angles || !meta || !out || n <= 0 || T <= 0)
    return fail(RIAB_ERR_INVALID, "riab_bvc_pack: bad argument");
  const int np = bvc_n_pad(n);
  const int64_t total = riab_bvc_pack_floats(n, T);
  for (int64_t i = 0; i < total; ++i) out[i] = 0.f;
  float* s = out; float* m = out + np; float* sc = out + 2 * np; float* vm = out + 3 * (size_t)np;
  // Slots: the cells sorted by preferred angle, so that the 32 cells of a warp of k_bvc_integrate share a narrow angular
  // window outside which every von Mises weight is < BVC_VM_CUT and the terms are skipped.  s | m | sc stay in cell order;
  // the von Mises table is in slot order; perm[slot] = cell (padding slots map to themselves).
  std::vector<int> order(n);
  std::vector<double> key(n);
  const double two_pi = 6.283185307179586;
  for (int i = 0; i < n; ++i) { order[i] = i; double a = fmod(mu_t[i], two_pi); key[i] = a < 0 ? a + two_pi : a; }
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return key[a] < key[b]; });
  for (int i = 0; i < n; ++i) {
    const double sv = sqrt(1.4426950408889634 / 2.0) / sg_d[i];       // exp(-(d-mu)^2/(2 sg^2)) = 2^-((d-mu) s)^2
    s[i] = (float)sv; m[i] = (float)(mu_d[i] * sv);
    const double kappa = 1.0 / (sg_t[i] * sg_t[i]);                   // utils.von_mises (utils.py:441-457), norm=1
    double norm = 0.0;
    for (int t = 0; t < T; ++t) norm += exp(kappa * cos(test_angles[t] - 0.0)) * (1.0 / exp(kappa));   // Neurons.py:1599-1604
    sc[i] = (float)(1.0 / norm);
  }
  int32_t* perm = reinterpret_cast<int32_t*>(out + 3 * (size_t)np + (size_t)np * T + 3 * (size_t)np + 2 * (size_t)T);
  int32_t* win = perm + np;
  std::vector<char> keep(T);
  for (int slot = 0; slot < np; ++slot) {
    const int i = slot < n ? order[slot] : slot;
    perm[slot] = i;
    if (slot < n) {
      const double kappa = 1.0 / (sg_t[i] * sg_t[i]);
      const int tile = slot / BVC_CT, cl = slot % BVC_CT;
      for (int t = 0; t < T; ++t)
        vm[((size_t)tile * T + t) * BVC_CT + cl] = (float)(exp(kappa * cos(test_angles[t] - mu_t[i])) * (1.0 / exp(kappa)));
    }
    if (slot % 32 == 31) {                                            // window of this warp's 32 slots: [th0, th0 + len) mod T
      const int s0 = slot - 31, tile = s0 / BVC_CT;
      for (int t = 0; t < T; ++t) {
        keep[t] = 0;
        for (int q = s0; q <= slot; ++q)
          if (!(vm[((size_t)tile * T + t) * BVC_CT + q % BVC_CT] < (float)BVC_VM_CUT)) { keep[t] = 1; break; }   // NaN keeps
      }
      int best_len = 0, best_end = 0;                                 // longest circular run of skippable angles
      for (int t0 = 0; t0 < T; ++t0) {
        if (keep[t0] || !keep[(t0 + T - 1) % T]) continue;            // runs start after a kept angle
        int len = 0;
        while (len < T && !keep[(t0 + len) % T]) ++len;
        if (len > best_len) { best_len = len; best_end = (t0 + len) % T; }
      }
      bool any = false;
      for (int t = 0; t < T; ++t) any = any || keep[t];
      win[2 * (s0 / 32)] = any ? (best_len ? best_end : 0) : 0;
      win[2 * (s0 / 32) + 1] = any ? T - best_len : 0;
    }
  }
  float* ext = vm + (size_t)np * T;                                  // egocentric: kap | cmu | smu | cth | sth
  for (int i = 0; i < n; ++i) {
    ext[i] = (float)(1.4426950408889634 / (sg_t[i] * sg_t[i]));
    ext[np + i] = (float)cos(mu_t[i]);
    ext[2 * np + i] = (float)sin(mu_t[i]);
  }
  for (int t = 0; t < T; ++t) {
    ext[3 * (size_t)np + t] = (float)cos(test_angles[t]);
    ext[3 * (size_t)np + T + t] = (float)sin(test_angles[t]);
  }
  meta->n_pad = np;
  return 0;
}

int riab_bvc_rates(const double* pos_dev, int64_t n_pos, const riab_env* env, const riab_bvc_cells* bvc,
                   float* scratch_dev, int32_t* first_wall_dev, const double* head_direction_dev, float* out_dev,
                   int64_t ld_out, void* stream) {
  return rates_at(RIAB_CELLS_BVC, bvc, pos_dev, n_pos, env, head_direction_dev, scratch_dev, first_wall_dev, out_dev, ld_out,
                  stream);
}

// ------------------------------------------------------------ kinematic cells
int64_t riab_kin_pack_floats(int32_t n_cells) { return (int64_t)place_n_pad(n_cells) * 3; }

int riab_kin_pack(const double* preferred_angles, const double* angular_tunings, int32_t n, int32_t variant,
                  int32_t use_velocity, float min_fr, float max_fr, double one_sigma_speed, riab_kin_cells* meta, float* out) {
  if (!meta || !out || n <= 0 || variant < RIAB_KIN_HEAD_DIRECTION || variant > RIAB_KIN_SPEED ||
      (variant != RIAB_KIN_SPEED && (!preferred_angles || !angular_tunings)))
    return fail(RIAB_ERR_INVALID, "riab_kin_pack: bad argument");
  const int np = place_n_pad(n);
  const double log2e = 1.4426950408889634;
  for (int i = 0; i < np; ++i) {
    const bool in = i < n && variant != RIAB_KIN_SPEED;
    const double kappa = in ? 1.0 / (angular_tunings[i] * angular_tunings[i]) : 0.0;   // utils.von_mises (utils.py:452)
    out[i] = in ? (float)cos(0.5 * preferred_angles[i]) : 1.f;
    out[(size_t)np + i] = in ? (float)sin(0.5 * preferred_angles[i]) : 0.f;
    out[(size_t)2 * np + i] = (float)sqrt(2.0 * kappa * log2e);
  }
  meta->n_cells = n; meta->variant = variant; meta->use_velocity = (variant == RIAB_KIN_VELOCITY) ? 1 : (use_velocity ? 1 : 0);
  meta->reserved0 = 0; meta->reserved1 = 0;
  meta->min_fr = min_fr; meta->max_fr = max_fr;
  meta->inv_one_sigma_speed = 1.0 / one_sigma_speed;
  meta->n_pad = np;
  return 0;
}

int riab_kin_rates(const double* vec_dev, int32_t vec_per_position, int64_t n_pos, double speed_scale,
                   const riab_kin_cells* cells, float* out_dev, int64_t ld_out, void* stream) {
  if (n_pos < 0 || (n_pos > 0 && vec_dev == nullptr)) return fail(RIAB_ERR_INVALID, "riab_kin_rates: bad argument");
  if (n_pos == 0) return 0;
  EnvK ek;
  memset(&ek, 0, sizeof(ek));                       // no walls: the rates do not depend on a position
  riab_rates_out ro = {};
  ro.rates_row = out_dev; ro.ld = ld_out;
  riab_agents at = {};
  at.n_agents = n_pos;
  at.head_direction = at.velocity = at.measured_velocity = (double*)vec_dev;
  Pop d;
  int rc;
  if ((rc = make_pop(ek, RIAB_CELLS_KIN, cells, &ro, nullptr, 1.0, at, d))) return rc;
  d.kin.vec_ld = vec_per_position ? 2 : 0;
  d.kin.fixed_scale = speed_scale;
  return launch_pop<0>(ek, at, kNoMotion, kNoStep, d, (cudaStream_t)stream);
}

// ------------------------------------------------------------ AgentVectorCells
int64_t riab_avc_pack_floats(int32_t n_cells) { return (int64_t)place_n_pad(n_cells) * 5; }

int riab_avc_pack(const double* tuning_distances, const double* tuning_angles, const double* sigma_distances,
                  const double* sigma_angles, int32_t n, riab_avc_cells* meta, float* out) {
  if (!tuning_distances || !tuning_angles || !sigma_distances || !sigma_angles || !meta || !out || n <= 0)
    return fail(RIAB_ERR_INVALID, "riab_avc_pack: bad argument");
  const int np = place_n_pad(n);
  const double log2e = 1.4426950408889634;
  for (int i = 0; i < np; ++i) {                       // riab_ovc_pack's first five columns; pads (0, 0, 1, 0, 0)
    const bool in = i < n;
    const double kappa = in ? 1.0 / (sigma_angles[i] * sigma_angles[i]) : 0.0;       // utils.von_mises (utils.py:441-457)
    out[i] = in ? (float)tuning_distances[i] : 0.f;
    out[(size_t)np + i] = in ? (float)(sqrt(0.5 * log2e) / sigma_distances[i]) : 0.f;  // utils.gaussian (utils.py:424-438)
    out[(size_t)2 * np + i] = in ? (float)cos(0.5 * tuning_angles[i]) : 1.f;
    out[(size_t)3 * np + i] = in ? (float)sin(0.5 * tuning_angles[i]) : 0.f;
    out[(size_t)4 * np + i] = (float)sqrt(2.0 * kappa * log2e);
  }
  meta->n_cells = n;
  meta->n_pad = np;
  return 0;
}

int riab_avc_rates(const double* pos_dev, int64_t n_pos, const double* other_pos_dev, int32_t other_per_position,
                   const riab_env* env, const riab_avc_cells* cells, const double* head_direction_dev, float* out_dev,
                   int64_t ld_out, void* stream) {
  if (cells == nullptr || other_pos_dev == nullptr) return fail(RIAB_ERR_INVALID, "riab_avc_rates: bad argument");
  riab_avc_cells c = *cells;
  c.other_pos_dev = other_pos_dev;
  c.n_other = other_per_position ? n_pos : 1;
  c.partner_is_self = 0;
  return rates_at(RIAB_CELLS_AVC, &c, pos_dev, n_pos, env, head_direction_dev, nullptr, nullptr, out_dev, ld_out, stream);
}

// ------------------------------------------------------ PhasePrecessingPlaceCells
int riab_pppc_rates(const double* pos_dev, const double* velocity_dev, int64_t n_pos, const riab_env* env,
                    const riab_pppc_cells* cells, float* out_dev, int64_t ld_out, void* stream) {
  if (n_pos > 0 && velocity_dev == nullptr) return fail(RIAB_ERR_INVALID, "riab_pppc_rates: velocity_dev NULL");
  return rates_at(RIAB_CELLS_PPPC, cells, pos_dev, n_pos, env, nullptr, nullptr, nullptr, out_dev, ld_out, stream, velocity_dev);
}

// ------------------------------------------------------------ ObjectVectorCells
int64_t riab_ovc_pack_floats(int32_t n_cells) { return (int64_t)place_n_pad(n_cells) * 6; }

int riab_ovc_pack(const double* tuning_distances, const double* tuning_angles, const double* sigma_distances,
                  const double* sigma_angles, const int32_t* tuning_types, int32_t n, riab_ovc_cells* meta, float* out) {
  if (!tuning_distances || !tuning_angles || !sigma_distances || !sigma_angles || !tuning_types || !meta || !out || n <= 0)
    return fail(RIAB_ERR_INVALID, "riab_ovc_pack: bad argument");
  const int np = place_n_pad(n);
  const double log2e = 1.4426950408889634;
  for (int i = 0; i < np; ++i) {
    const bool in = i < n;
    const double kappa = in ? 1.0 / (sigma_angles[i] * sigma_angles[i]) : 0.0;       // utils.von_mises (utils.py:441-457)
    out[i] = in ? (float)tuning_distances[i] : 0.f;
    out[(size_t)np + i] = in ? (float)(sqrt(0.5 * log2e) / sigma_distances[i]) : 0.f;  // utils.gaussian (utils.py:424-438)
    out[(size_t)2 * np + i] = in ? (float)cos(0.5 * tuning_angles[i]) : 1.f;
    out[(size_t)3 * np + i] = in ? (float)sin(0.5 * tuning_angles[i]) : 0.f;
    out[(size_t)4 * np + i] = (float)sqrt(2.0 * kappa * log2e);
    out[(size_t)5 * np + i] = in ? (float)tuning_types[i] : -2.f;                     // padding cells match no object
  }
  meta->n_pad = np;
  return 0;
}

int riab_ovc_rates(const double* pos_dev, int64_t n_pos, const riab_env* env, const riab_ovc_cells* ovc,
                   const double* head_direction_dev, float* out_dev, int64_t ld_out, void* stream) {
  return rates_at(RIAB_CELLS_OVC, ovc, pos_dev, n_pos, env, head_direction_dev, nullptr, nullptr, out_dev, ld_out, stream);
}

// ------------------------------------------------------------ FeedForwardLayer
static int ffl_n_pad(int n) { return (n + 7) / 8 * 8; }
static int ffl_k_pad(int n_in) { return (n_in + FFL_BK - 1) / FFL_BK * FFL_BK; }
// cvt.rna.tf32.f32 on the host: round to nearest (ties away from zero) to 10 mantissa bits, the low 13 bits cleared
static float tf32_rna(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  if ((u & 0x7f800000u) != 0x7f800000u) u = (u + 0x1000u) & ~0x1fffu;
  float r;
  memcpy(&r, &u, 4);
  return r;
}

int64_t riab_ffl_pack_floats(int32_t n_cells, int32_t n_in) {
  return 2 * (int64_t)ffl_n_pad(n_cells) * ffl_k_pad(n_in);
}

int riab_ffl_pack(const double* w, int32_t n, int32_t n_in, riab_ffl_input* meta, float* out) {
  if (w == nullptr || meta == nullptr || out == nullptr || n <= 0 || n_in <= 0) return fail(RIAB_ERR_INVALID, "riab_ffl_pack: bad argument");
  const int np = ffl_n_pad(n), kp = ffl_k_pad(n_in);
  float* hi = out;
  float* lo = out + (size_t)np * kp;
  for (int i = 0; i < np; ++i)
    for (int j = 0; j < kp; ++j) {
      const size_t o = (size_t)i * kp + j;
      const float x = (i < n && j < n_in) ? (float)w[(size_t)i * n_in + j] : 0.f;
      hi[o] = tf32_rna(x);
      lo[o] = tf32_rna(x - hi[o]);
    }
  meta->w_dev = nullptr;
  meta->n_in = n_in;
  meta->k_pad = kp;
  return 0;
}

int riab_ffl_rates(const riab_ffl_cells* ffl, int64_t n_rows, const double* pos_dev, const riab_neuron_noise* noise,
                   const riab_rates_out* out, void* stream) {
  if (ffl == nullptr || n_rows < 0) return fail(RIAB_ERR_INVALID, "riab_ffl_rates: bad argument");
  return layer_rates(RIAB_CELLS_FFL, ffl, n_rows, pos_dev, noise, out, stream);
}

// ------------------------------------------------------------ NeuralNetworkNeurons
int64_t riab_nnn_pack_floats(const riab_nnn_cells* meta) {
  if (meta == nullptr || meta->n_layers < 1 || meta->n_layers > RIAB_NNN_MAX_LAYERS || meta->n_inputs < 1 ||
      meta->n_inputs > RIAB_FFL_MAX_INPUTS)
    return -1;
  int64_t n = 0;
  for (int i = 0; i < meta->n_inputs; ++i) n += riab_ffl_pack_floats(meta->widths[1], meta->inputs[i].n_in);
  n += ffl_n_pad(meta->widths[1]);
  for (int l = 2; l <= meta->n_layers; ++l) n += (int64_t)(meta->widths[l - 1] + 1) * ffl_n_pad(meta->widths[l]);
  return n;
}

int riab_nnn_pack(const double* params, riab_nnn_cells* meta, float* out) {
  if (params == nullptr || meta == nullptr || out == nullptr) return fail(RIAB_ERR_INVALID, "riab_nnn_pack: bad argument");
  const int L = meta->n_layers;
  if (L < 1 || L > RIAB_NNN_MAX_LAYERS)
    return fail(RIAB_ERR_UNSUPPORTED, "riab_nnn_pack: %d Linear layers (1 to %d)", L, RIAB_NNN_MAX_LAYERS);
  if (meta->n_inputs < 1 || meta->n_inputs > RIAB_FFL_MAX_INPUTS)
    return fail(RIAB_ERR_UNSUPPORTED, "riab_nnn_pack: %d inputs (1 to %d)", meta->n_inputs, RIAB_FFL_MAX_INPUTS);
  for (int i = 0; i < meta->n_inputs; ++i)
    if (meta->inputs[i].n_in <= 0) return fail(RIAB_ERR_INVALID, "riab_nnn_pack: input %d has %d rates", i, meta->inputs[i].n_in);
  int rc;
  if ((rc = check_nnn_layers(meta, "riab_nnn_pack"))) return rc;
  const int n_in = meta->widths[0];
  // layer 1: W_1's column block of each input through riab_ffl_pack
  const int h1 = meta->widths[1];
  const double* p = params;
  float* o = out;
  std::vector<double> block;
  int col0 = 0;
  for (int i = 0; i < meta->n_inputs; ++i) {
    const int ni = meta->inputs[i].n_in;
    block.assign((size_t)h1 * ni, 0.0);
    for (int r = 0; r < h1; ++r)
      for (int j = 0; j < ni; ++j) block[(size_t)r * ni + j] = p[(size_t)r * n_in + col0 + j];
    riab_ffl_input tmp = meta->inputs[i];
    if ((rc = riab_ffl_pack(block.data(), h1, ni, &tmp, o))) return rc;
    meta->inputs[i].k_pad = tmp.k_pad;
    o += riab_ffl_pack_floats(h1, ni);
    col0 += ni;
  }
  p += (size_t)h1 * n_in;
  for (int c = 0; c < ffl_n_pad(h1); ++c) o[c] = c < h1 ? (float)p[c] : 0.f;
  o += ffl_n_pad(h1);
  p += h1;
  // layers 2..L: W_l^T (h_in, pad8(h_out)) then b_l
  for (int l = 2; l <= L; ++l) {
    const int ni = meta->widths[l - 1], no = meta->widths[l], no8 = ffl_n_pad(no);
    for (int i = 0; i < ni; ++i)
      for (int c = 0; c < no8; ++c) o[(size_t)i * no8 + c] = c < no ? (float)p[(size_t)c * ni + i] : 0.f;
    o += (size_t)ni * no8;
    p += (size_t)no * ni;
    for (int c = 0; c < no8; ++c) o[c] = c < no ? (float)p[c] : 0.f;
    o += no8;
    p += no;
  }
  meta->n_cells = meta->widths[L];
  return 0;
}

int riab_nnn_rates(const riab_nnn_cells* cells, int64_t n_rows, const double* pos_dev, const riab_neuron_noise* noise,
                   const riab_rates_out* out, void* stream) {
  if (cells == nullptr || n_rows < 0) return fail(RIAB_ERR_INVALID, "riab_nnn_rates: bad argument");
  return layer_rates(RIAB_CELLS_NNN, cells, n_rows, pos_dev, noise, out, stream);
}

// ------------------------------------------------------------------ TD learning
int64_t riab_td_splits(int32_t n_cells, int32_t n_in, int64_t n_rows) {
  if (n_cells <= 0 || n_in <= 0 || n_rows < 0) {
    fail(RIAB_ERR_INVALID, "riab_td_splits: bad argument");
    return -1;
  }
  return td_split(n_cells, n_in, n_rows).splits;
}

int64_t riab_td_scratch_bytes(const riab_td_cells* t, int64_t n_rows) {
  if (t == nullptr || n_rows < 0 || t->ffl.n_cells <= 0 || t->ffl.n_inputs < 0 || t->ffl.n_inputs > RIAB_FFL_MAX_INPUTS) {
    fail(RIAB_ERR_INVALID, "riab_td_scratch_bytes: bad argument");
    return -1;
  }
  if (t->per_agent_weights) return 0;              // k_td_learn_pa updates the masters in place
  size_t part = 0;
  for (int l = 0; l < t->ffl.n_inputs; ++l) {
    const int n_in = t->ffl.inputs[l].n_in;
    if (n_in <= 0) { fail(RIAB_ERR_INVALID, "riab_td_scratch_bytes: input %d has n_in %d", l, n_in); return -1; }
    const TdSplit sp = td_split(t->ffl.n_cells, n_in, n_rows);
    part = std::max(part, (size_t)sp.splits * t->ffl.n_cells * n_in * sizeof(double));
  }
  return (int64_t)(td_g_bytes(t->ffl.n_cells, n_rows) + part);
}

int riab_td_learn(const riab_td_cells* t, int64_t n_rows, const void* reward, int32_t reward_mode, float* td_error_out,
                  void* scratch, void* stream) {
  if (t == nullptr || n_rows < 0 || reward == nullptr || td_error_out == nullptr ||
      (scratch == nullptr && !t->per_agent_weights) ||
      (reward_mode != RIAB_TD_REWARD_SHARED && reward_mode != RIAB_TD_REWARD_ROWS))
    return fail(RIAB_ERR_INVALID, "riab_td_learn: bad argument");
  if (((uintptr_t)scratch) % 16 != 0) return fail(RIAB_ERR_INVALID, "riab_td_learn: scratch must be 16-byte aligned");
  int rc;
  if ((rc = check_td(t, t->ld))) return rc;
  const riab_ffl_cells& f = t->ffl;
  if (f.prime_dev == nullptr) return fail(RIAB_ERR_INVALID, "riab_td_learn: prime_dev NULL");
  if (n_rows == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int n = f.n_cells;
  TdGK g;
  g.fr = t->fr_prev_dev; g.deriv = t->deriv_dev; g.prime = f.prime_dev;
  g.reward_shared = reward_mode == RIAB_TD_REWARD_SHARED ? (const double*)reward : nullptr;
  g.reward_rows = reward_mode == RIAB_TD_REWARD_ROWS ? (const float*)reward : nullptr;
  g.td = td_error_out;
  g.g = t->per_agent_weights ? nullptr : (float*)scratch;     // the per-agent update forms g from td itself
  g.ld = t->ld; g.ldg = td_g_ld(n); g.n_rows = n_rows; g.n_cells = n;
  g.inv_tau = 1.0 / t->tau;
  const long long ng = n_rows * g.ldg;
  k_td_g<<<(unsigned)((ng + 255) / 256), 256, 0, s>>>(g);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  if (t->per_agent_weights) {
    for (int l = 0; l < f.n_inputs; ++l) {
      TdLearnPaK k;
      k.td = td_error_out; k.prime = f.prime_dev; k.e = t->trace_dev[l]; k.w = t->w_master_dev[l];
      k.ld = t->ld; k.lde = t->trace_ld[l]; k.n_cells = n; k.n_in = f.inputs[l].n_in;
      k.c_grad = t->dt * t->eta;                      // self.Agent.dt * self.eta
      k.c_decay = t->eta * t->dt * t->L2;             // self.eta * self.Agent.dt * self.L2
      k_td_learn_pa<<<(unsigned)n_rows, TD_LEARN_PA_THREADS, 0, s>>>(k);
      g_launches++;
      RIAB_CUDA_OK(cudaGetLastError());
    }
    return 0;
  }
  double* part = (double*)((char*)scratch + td_g_bytes(n, n_rows));
  for (int l = 0; l < f.n_inputs; ++l) {
    const riab_ffl_input& in = f.inputs[l];
    const TdSplit sp = td_split(n, in.n_in, n_rows);
    TdLearnK lk;
    lk.g = g.g; lk.e = t->trace_dev[l]; lk.part = part;
    lk.ldg = g.ldg; lk.lde = t->trace_ld[l]; lk.n_rows = n_rows; lk.chunk = sp.chunk;
    lk.n_cells = n; lk.n_in = in.n_in;
    const dim3 grid((unsigned)sp.tiles, (unsigned)sp.splits);
    if (sp.small) k_td_learn<8, 256, 8, 1><<<grid, TD_THREADS, 0, s>>>(lk);
    else k_td_learn_tc<<<grid, TD_TC_THREADS, 0, s>>>(lk);
    g_launches++;
    RIAB_CUDA_OK(cudaGetLastError());
    TdApplyK ak;
    ak.part = part; ak.w = t->w_master_dev[l];
    ak.whi = const_cast<float*>(in.w_dev);
    ak.wlo = ak.whi + (size_t)((n + 7) / 8 * 8) * in.k_pad;
    ak.n_cells = n; ak.n_in = in.n_in; ak.k_pad = in.k_pad; ak.splits = (int)sp.splits;
    ak.n_rows = (double)n_rows;
    ak.c_grad = t->dt * t->eta;                       // self.Agent.dt * self.eta
    ak.c_decay = t->eta * t->dt * t->L2;              // self.eta * self.Agent.dt * self.L2
    const long long nw = (long long)n * in.n_in;
    if (sp.splits >= 32) k_td_apply<true><<<(unsigned)((32 * nw + 255) / 256), 256, 0, s>>>(ak);
    else k_td_apply<false><<<(unsigned)((nw + 255) / 256), 256, 0, s>>>(ak);
    g_launches++;
    RIAB_CUDA_OK(cudaGetLastError());
  }
  return 0;
}

int riab_td_rates_pa(const riab_td_cells* t, int64_t n_rows, const int64_t* weight_agent_of_row_dev,
                     const int64_t* input_row_of_row_dev, float* out_dev, int64_t ld_out, void* stream) {
  if (t == nullptr || n_rows < 0 || (n_rows > 0 && out_dev == nullptr) || ld_out < t->ffl.n_cells)
    return fail(RIAB_ERR_INVALID, "riab_td_rates_pa: bad argument");
  if (!t->per_agent_weights) return fail(RIAB_ERR_INVALID, "riab_td_rates_pa: the layer's weights are shared");
  int rc;
  OutK out;
  memset(&out, 0, sizeof(out));
  out.ld = ld_out;
  if ((rc = check_ffl(&t->ffl, out, n_rows, false))) return rc;
  for (int l = 0; l < t->ffl.n_inputs; ++l)
    if (t->w_master_dev[l] == nullptr || t->ffl.inputs[l].n_in <= 0)
      return fail(RIAB_ERR_INVALID, "riab_td_rates_pa: input %d has no masters", l);
  static_assert(sizeof(long long) == sizeof(int64_t), "row maps");
  return launch_td_forward_pa(t, n_rows, (const long long*)weight_agent_of_row_dev, (const long long*)input_row_of_row_dev,
                              nullptr, out_dev, ld_out, nullptr, (cudaStream_t)stream);
}

int riab_td_reset(const riab_td_cells* t, int64_t n_rows, const uint8_t* mask, void* stream) {
  if (t == nullptr || n_rows < 0) return fail(RIAB_ERR_INVALID, "riab_td_reset: bad argument");
  int rc;
  if ((rc = check_td(t, t->ld))) return rc;
  if (n_rows == 0) return 0;
  TdResetK k;
  memset(&k, 0, sizeof(k));
  k.rows[0] = t->fr_prev_dev; k.rows[1] = t->deriv_dev; k.rows[2] = t->td_error_dev;
  k.ld = t->ld; k.n_rows = n_rows; k.n_inputs = t->ffl.n_inputs; k.mask = mask;
  for (int l = 0; l < k.n_inputs; ++l) { k.trace[l] = t->trace_dev[l]; k.trace_ld[l] = t->trace_ld[l]; }
  k_td_reset<<<(unsigned)n_rows, 128, 0, (cudaStream_t)stream>>>(k);
  g_launches++;
  RIAB_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------- RandomSpatialNeurons
int64_t riab_rsn_pack_floats(int32_t n_cells, int32_t n_points, int32_t n_inner_walls) {
  if (n_cells <= 0 || n_points <= 0) return 0;
  return riab_place_pack_floats(ffl_k_pad(n_points), n_inner_walls) + riab_ffl_pack_floats(n_cells, n_points);
}

int riab_rsn_pack(const double* X, int32_t n_points, const double* targets, int32_t n_cells, double lengthscale,
                  const double* walls, int32_t n_walls, int32_t n_boundary, const double* extent, int32_t geometry,
                  riab_rsn_cells* meta, float* out, double* centres_out) {
  if (!X || !targets || !extent || !meta || !out || !centres_out || n_points <= 0 || n_cells <= 0 || !(lengthscale > 0.0))
    return fail(RIAB_ERR_INVALID, "riab_rsn_pack: bad argument");
  const int kp = ffl_k_pad(n_points);
  // the sample points in the packed K order (pads repeat point 0: inside the box, they leave the screen's bounds as they are)
  std::vector<double> widths((size_t)kp, lengthscale);
  for (int p = 0; p < kp; ++p) {
    const int j = (p / FFL_BK) * FFL_BK + rsn_k_of_packed(p % FFL_BK);
    const int src = j < n_points ? j : 0;
    centres_out[2 * p] = X[2 * src];
    centres_out[2 * p + 1] = X[2 * src + 1];
  }
  memset(&meta->points, 0, sizeof(meta->points));
  int rc;
  if ((rc = riab_place_pack(centres_out, widths.data(), kp, walls, n_walls, n_boundary, extent, geometry, &meta->points, out)))
    return rc;
  meta->points.n_cells = kp;
  meta->points.description = RIAB_PC_GAUSSIAN;
  meta->points.wall_geometry = geometry;
  meta->points.min_fr = 0.f;
  meta->points.max_fr = 1.f;
  meta->points.top_hat_width = lengthscale;
  // the targets along K in sample-point order: W = targets.T (n_cells, n_points)
  std::vector<double> wt((size_t)n_cells * n_points);
  for (int j = 0; j < n_points; ++j)
    for (int i = 0; i < n_cells; ++i) wt[(size_t)i * n_points + j] = targets[(size_t)j * n_cells + i];
  riab_ffl_input tm;
  if ((rc = riab_ffl_pack(wt.data(), n_cells, n_points, &tm, out + riab_place_pack_floats(kp, meta->points.n_inner_walls))))
    return rc;
  meta->targets_dev = nullptr;
  meta->n_cells = n_cells;
  meta->n_points = n_points;
  meta->k_pad = tm.k_pad;
  return 0;
}

int riab_rsn_rates(const double* pos_dev, int64_t n_pos, const riab_env* env, const riab_rsn_cells* rsn, float* out_dev,
                   int64_t ld_out, void* stream) {
  return rates_at(RIAB_CELLS_RSN, rsn, pos_dev, n_pos, env, nullptr, nullptr, nullptr, out_dev, ld_out, stream);
}

// ----------------------------------------------------------------- fused step

int riab_step_fused(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm,
                    const riab_step_io* io, int32_t cells_kind, const void* cells, const riab_neuron_noise* noise,
                    const riab_rates_out* out, void* stream) {
  return neurons_update_impl(true, agents, env, prm, io, cells_kind, cells, noise, out, stream);
}

int riab_neurons_update(const riab_agents* agents, const riab_env* env, int32_t cells_kind, const void* cells,
                        const riab_neuron_noise* noise, const riab_rates_out* out, void* stream) {
  return neurons_update_impl(false, agents, env, nullptr, nullptr, cells_kind, cells, noise, out, stream);
}



int riab_run(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm, const riab_step_io* io,
             const riab_population* pops, int32_t n_pops, const riab_agent_history* hist, int64_t n_steps,
             void* stream) {
  return run_impl(agents, env, prm, io, nullptr, pops, n_pops, hist, n_steps, stream);
}

int riab_run_src(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm, const riab_step_io* io,
                 const riab_motion_source* src, const riab_population* pops, int32_t n_pops,
                 const riab_agent_history* hist, int64_t n_steps, void* stream) {
  if (src == nullptr || src->kind == RIAB_MOTION_RANDOM) return riab_run(agents, env, prm, io, pops, n_pops, hist, n_steps, stream);
  if (src->kind != RIAB_MOTION_IMPORTED) return fail(RIAB_ERR_UNSUPPORTED, "riab_run_src: a forced position belongs to one step");
  if (agents == nullptr) return fail(RIAB_ERR_INVALID, "riab_run: bad argument");
  SrcK sk;
  int rc;
  if ((rc = make_src(src, agents->n_agents, sk))) return rc;
  return run_impl(agents, env, prm, io, src, pops, n_pops, hist, n_steps, stream);
}

int riab_step_fused_host(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm,
                         riab_step_io* io, int32_t cells_kind, const void* cells, const riab_neuron_noise* noise,
                         const riab_rates_out* out, const double* drift_host, double* drift_staging_dev,
                         double* pos_out_host, void* stream) {
  if (agents == nullptr || io == nullptr) return fail(RIAB_ERR_INVALID, "agents / io NULL");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t bytes = (size_t)agents->n_agents * 2 * sizeof(double);
  if (drift_host != nullptr) {
    if (drift_staging_dev == nullptr) return fail(RIAB_ERR_INVALID, "drift_staging_dev NULL");
    RIAB_CUDA_OK(cudaMemcpyAsync(drift_staging_dev, drift_host, bytes, cudaMemcpyHostToDevice, s));
    io->drift_velocity = drift_staging_dev;
  }
  const int rc = riab_step_fused(agents, env, prm, io, cells_kind, cells, noise, out, stream);
  if (rc) return rc;
  if (pos_out_host != nullptr) RIAB_CUDA_OK(cudaMemcpyAsync(pos_out_host, agents->pos, bytes, cudaMemcpyDeviceToHost, s));
  return 0;
}

int riab_positions_fence(void* stream) {
  HostIo* h = nullptr;
  int rc;
  if ((rc = hostio(h))) return rc;
  if (h->pos_inflight) RIAB_CUDA_OK(cudaStreamWaitEvent((cudaStream_t)stream, h->pos_done, 0));
  return 0;
}

int riab_positions_wait(void) {
  HostIo* h = nullptr;
  int rc;
  if ((rc = hostio(h))) return rc;
  if (h->pos_inflight) RIAB_CUDA_OK(cudaEventSynchronize(h->pos_done));
  return 0;
}

int riab_agent_update_host(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm,
                           riab_step_io* io, const double* drift_host, double* drift_staging_dev,
                           double* pos_out_host, void* stream) {
  if (agents == nullptr || io == nullptr) return fail(RIAB_ERR_INVALID, "agents / io NULL");
  HostIo* h = nullptr;
  int rc;
  if ((rc = hostio(h))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t bytes = (size_t)agents->n_agents * 2 * sizeof(double);
  if (drift_host != nullptr) {
    if (drift_staging_dev == nullptr) return fail(RIAB_ERR_INVALID, "drift_staging_dev NULL");
    // the previous motion kernel (the last reader of the staging buffer) finished before the side stream's last copy
    // started (that copy waited for motion_done), so the upload may start at once
    RIAB_CUDA_OK(cudaMemcpyAsync(drift_staging_dev, drift_host, bytes, cudaMemcpyHostToDevice, h->side));
    RIAB_CUDA_OK(cudaEventRecord(h->up_done, h->side));
    RIAB_CUDA_OK(cudaStreamWaitEvent(s, h->up_done, 0));
    io->drift_velocity = drift_staging_dev;
  }
  if (h->pos_inflight) RIAB_CUDA_OK(cudaStreamWaitEvent(s, h->pos_done, 0));   // the copy that still reads agents->pos
  if ((rc = riab_agent_update(agents, env, prm, io, stream))) return rc;
  RIAB_CUDA_OK(cudaEventRecord(h->motion_done, s));
  RIAB_CUDA_OK(cudaStreamWaitEvent(h->side, h->motion_done, 0));
  if (pos_out_host != nullptr) {
    RIAB_CUDA_OK(cudaMemcpyAsync(pos_out_host, agents->pos, bytes, cudaMemcpyDeviceToHost, h->side));
    RIAB_CUDA_OK(cudaEventRecord(h->pos_done, h->side));
    h->pos_inflight = true;
  }
  return 0;
}

}  // extern "C"

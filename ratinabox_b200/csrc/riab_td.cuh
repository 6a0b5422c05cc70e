// TD learning for ValueNeuron / SuccessorFeatures (riab_td_cells, include/riab_b200.h) on sm_90a.
//
//   k_td_trace   after the layer's k_ffl (+ k_finish_rows): per agent row deriv = (fr - fr_prev) / dt, fr_prev <- fr and
//                e_l <- dt I_l + (1 - dt / tau_e) e_l for every input; one CTA per row, float4 streams.
//   k_td_g       update_weights, pass 1: td = reward + deriv - fr_prev / tau -> td_error, g = td phi' -> (A, ldg) scratch.
//   pass 2, the contraction over the AGENT axis, P_s[i, j] = sum_{a in chunk s} g[a, i] e[a, j]: each CTA owns a tile
//                of (cells x inputs) and one chunk of agents, staged 32 agents at a time in shared memory from the
//                agent-major rows; every 32 agents the float32 partial sums are added into float64 accumulators, then the
//                tile is written to its chunk's slot of the float64 partial buffer.
//     k_td_learn_tc   n > 8: 64 x 64 tiles on the tensor cores, 3xTF32 wgmma (hi.hi + hi.lo + lo.hi, as k_ffl).  wgmma's
//                     tf32 B operand must be K-major in shared memory and K is the agent axis, so the trace tile is
//                     TRANSPOSED while it is staged (and split into hi / lo there); the g tile is the A operand, read
//                     from shared memory in the row layout it arrives in and split in registers.
//     k_td_learn      n <= 8: 8 x 256 tiles on the CUDA cores (bandwidth-bound: one trace read, 8 FMAs per element).
//   k_td_apply   pass 3: per weight, the chunk partials summed in a fixed order (float64: serially in chunk order, or
//                with many chunks by a warp, each lane over a fixed stride of chunks then a fixed shuffle tree), the reference's update
//                dW = dt eta (S / A) - eta dt L2 W applied to the float64 master, and W_hi | W_lo re-split exactly as
//                riab_ffl_pack does (cvt.rna.tf32 of float32(W), then of the remainder).
//   k_td_reset   zero fr_prev / deriv / td_error / traces of the masked rows.
// Per-agent weights (riab_td_cells.per_agent_weights), the masters (A, n, n_in) float64:
//   k_td_forward_pa  the layer's contraction in place of k_ffl: one warp per (row, cell), the row's inputs staged in
//                    shared memory, W rows read coalesced in float64, a float64 lane sum then a fixed xor shuffle tree;
//                    the bias and k_ffl's activation epilogue (layer_activate).  k_finish_rows and k_td_trace follow.
//   k_td_learn_pa    after k_td_g (td only): W[a] += (dt eta) (td phi')[a, j] e[a, i] - (eta dt L2) W[a], elementwise.
//   Both stream W once (forward 8 A n n_in bytes, learning 16 A n n_in): bandwidth-bound, no atomics.
// Every reduction has a fixed order that depends on the shapes only: the stepped API and Agent.run give the same bits,
// and two identical runs give identical weights.
#pragma once
#include "riab_common.cuh"
#include "riab_ffl.cuh"

namespace riab {

struct TdTraceK {
  const float* rates;                         // (A, ld) this update's rates (after noise)
  float* fr_prev;
  float* deriv;
  long long ld, n_rows;
  int n_cells, n_inputs;
  const float* in[RIAB_FFL_MAX_INPUTS];       // (A, in_ld) rows the contraction read; NULL = zeros
  long long in_ld[RIAB_FFL_MAX_INPUTS];
  float* trace[RIAB_FFL_MAX_INPUTS];
  long long trace_ld[RIAB_FFL_MAX_INPUTS];
  int n_in[RIAB_FFL_MAX_INPUTS];
  float dt, decay;                            // float32(dt), float32(1 - dt / tau_e)
};

constexpr int TD_TRACE_THREADS = 128;

__global__ void __launch_bounds__(TD_TRACE_THREADS) k_td_trace(const __grid_constant__ TdTraceK k) {
  const long long row = blockIdx.x;
  if (row >= k.n_rows) return;
  const float dt = k.dt, decay = k.decay;
  for (int c = threadIdx.x; c < k.n_cells; c += TD_TRACE_THREADS) {
    const float fr = k.rates[row * k.ld + c];
    float* prev = k.fr_prev + row * k.ld + c;
    k.deriv[row * k.ld + c] = (fr - *prev) / dt;
    *prev = fr;
  }
  for (int l = 0; l < k.n_inputs; ++l) {
    const int n4 = (k.n_in[l] + 3) >> 2;
    float4* e = reinterpret_cast<float4*>(k.trace[l] + row * k.trace_ld[l]);
    const float4* I = k.in[l] ? reinterpret_cast<const float4*>(k.in[l] + row * k.in_ld[l]) : nullptr;
    for (int q = threadIdx.x; q < n4; q += TD_TRACE_THREADS) {
      const float4 x = I ? I[q] : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 v = e[q];
      v.x = dt * x.x + decay * v.x;
      v.y = dt * x.y + decay * v.y;
      v.z = dt * x.z + decay * v.z;
      v.w = dt * x.w + decay * v.w;
      const int j = 4 * q;                    // the pad columns of an input row are not rates: keep them zero
      if (j + 1 >= k.n_in[l]) v.y = 0.f;
      if (j + 2 >= k.n_in[l]) v.z = 0.f;
      if (j + 3 >= k.n_in[l]) v.w = 0.f;
      e[q] = v;
    }
  }
}

struct TdGK {
  const float* fr;          // fr_prev: the layer's firingrate
  const float* deriv;
  const float* prime;
  const double* reward_shared;   // (n) or NULL
  const float* reward_rows;      // (A, ld) or NULL
  float* td;                     // (A, ld)
  float* g;                      // (A, ldg), pads zero; NULL: td only (per-agent weights)
  long long ld, ldg, n_rows;
  int n_cells;
  double inv_tau;
};

__global__ void k_td_g(const __grid_constant__ TdGK k) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= k.n_rows * k.ldg) return;
  const long long a = idx / k.ldg;
  const int i = (int)(idx - a * k.ldg);
  if (i >= k.n_cells) {
    if (k.g) k.g[idx] = 0.f;
    return;
  }
  const long long o = a * k.ld + i;
  const double r = k.reward_shared ? k.reward_shared[i] : (double)k.reward_rows[o];
  // the reference's order: reward + dVdt - V / tau
  const double td = (r + (double)k.deriv[o]) - (double)k.fr[o] * k.inv_tau;
  k.td[o] = (float)td;
  if (k.g) k.g[idx] = (float)(td * (double)k.prime[o]);
}

constexpr int TD_KC = 32;            // agents staged per shared-memory round
constexpr int TD_THREADS = 256;

struct TdLearnK {
  const float* g;       // (A, ldg)
  const float* e;       // (A, lde)
  double* part;         // (splits, n, n_in)
  long long ldg, lde, n_rows, chunk;
  int n_cells, n_in;
};

// (BM cells x BN inputs) per CTA, TM x TN per thread; (BM / TM) * (BN / TN) == TD_THREADS
template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__(TD_THREADS) k_td_learn(const __grid_constant__ TdLearnK k) {
  static_assert((BM / TM) * (BN / TN) == TD_THREADS, "thread tile");
  __shared__ __align__(16) float gs[TD_KC][BM];
  __shared__ __align__(16) float es[TD_KC][BN];
  constexpr int TX = BN / TN;
  const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
  const int tiles_j = (k.n_in + BN - 1) / BN;
  const int i0 = (blockIdx.x / tiles_j) * BM, j0 = (blockIdx.x % tiles_j) * BN;
  const long long a0 = (long long)blockIdx.y * k.chunk;
  const long long a1 = min(a0 + k.chunk, k.n_rows);
  double acc[TM][TN];
#pragma unroll
  for (int m = 0; m < TM; ++m)
#pragma unroll
    for (int q = 0; q < TN; ++q) acc[m][q] = 0.0;
  for (long long ab = a0; ab < a1; ab += TD_KC) {
    for (int t = threadIdx.x; t < TD_KC * BM; t += TD_THREADS) {
      const int r = t / BM, i = t % BM;
      const long long a = ab + r;
      gs[r][i] = (a < a1 && i0 + i < k.n_cells) ? k.g[a * k.ldg + i0 + i] : 0.f;
    }
    for (int t = threadIdx.x; t < TD_KC * BN; t += TD_THREADS) {
      const int r = t / BN, j = t % BN;
      const long long a = ab + r;
      es[r][j] = (a < a1 && j0 + j < k.n_in) ? k.e[a * k.lde + j0 + j] : 0.f;
    }
    __syncthreads();
    // float32 products summed over KC agents, then promoted: a partial sum of 32 terms is within 32 eps of its
    // terms' absolute sum
    float p[TM][TN];
#pragma unroll
    for (int m = 0; m < TM; ++m)
#pragma unroll
      for (int q = 0; q < TN; ++q) p[m][q] = 0.f;
#pragma unroll 4
    for (int r = 0; r < TD_KC; ++r) {
      float gv[TM], ev[TN];
#pragma unroll
      for (int m = 0; m < TM; ++m) gv[m] = gs[r][ty * TM + m];
#pragma unroll
      for (int q = 0; q < TN; ++q) ev[q] = es[r][tx * TN + q];
#pragma unroll
      for (int m = 0; m < TM; ++m)
#pragma unroll
        for (int q = 0; q < TN; ++q) p[m][q] = fmaf(gv[m], ev[q], p[m][q]);
    }
#pragma unroll
    for (int m = 0; m < TM; ++m)
#pragma unroll
      for (int q = 0; q < TN; ++q) acc[m][q] += (double)p[m][q];
    __syncthreads();
  }
  double* dst = k.part + (size_t)blockIdx.y * k.n_cells * k.n_in;
#pragma unroll
  for (int m = 0; m < TM; ++m) {
    const int i = i0 + ty * TM + m;
    if (i >= k.n_cells) continue;
#pragma unroll
    for (int q = 0; q < TN; ++q) {
      const int j = j0 + tx * TN + q;
      if (j < k.n_in) dst[(size_t)i * k.n_in + j] = acc[m][q];
    }
  }
}

// 3xTF32 wgmma contraction over the agent axis: one warpgroup, a 64 (cells) x 64 (inputs) tile, 32 agents per round.
// A (m64 x k8, cells x agents) comes from registers: fragment a0 (r0, c), a1 (r0 + 8, c), a2 (r0, c + 4), a3 (r0 + 8, c + 4)
// with r0 = 16 warp + lane / 4 (a cell) and c = 8 k8 + lane % 4 (an agent), read from gs[agent][cell] (row stride 72
// floats: the 32 lanes' reads hit 32 banks).  B (k8 x n64) is the trace tile transposed into 64 rows (inputs) of 32 agents,
// 128 bytes each, 128-byte swizzled (16-byte chunk q of row r at q ^ (r % 8)), in the layout k_ffl's W tiles have.  The next
// round's global loads are issued before this round's wgmmas, so they overlap.
constexpr int TD_TC_THREADS = 128;
constexpr int TD_GS_LD = 72;

__global__ void __launch_bounds__(TD_TC_THREADS) k_td_learn_tc(const __grid_constant__ TdLearnK k) {
  __shared__ __align__(16) float gs[TD_KC * TD_GS_LD];
  __shared__ __align__(16) uint8_t eraw[2 * 64 * 128 + 1024];
  uint8_t* ehi = eraw + ((1024u - (smem_u32(eraw) & 1023u)) & 1023u);      // swizzle atoms are 1024 bytes
  uint8_t* elo = ehi + 64 * 128;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tiles_j = (k.n_in + 63) / 64;
  const int i0 = (blockIdx.x / tiles_j) * 64, j0 = (blockIdx.x % tiles_j) * 64;
  const long long a0 = (long long)blockIdx.y * k.chunk;
  const long long a1 = min(a0 + k.chunk, k.n_rows);
  // staging: element t + 128 q of a round is (agent (t + 128 q) / 64, column (t + 128 q) % 64): coalesced rows
  float gv[16], ev[16];
  auto load = [&](long long ab) {
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int idx = tid + TD_TC_THREADS * q, r = idx >> 6, c = idx & 63;
      const long long a = ab + r;
      const bool ok = a < a1;
      gv[q] = (ok && i0 + c < k.n_cells) ? k.g[a * k.ldg + i0 + c] : 0.f;
      ev[q] = (ok && j0 + c < k.n_in) ? k.e[a * k.lde + j0 + c] : 0.f;
    }
  };
  double acc[32];
#pragma unroll
  for (int q = 0; q < 32; ++q) acc[q] = 0.0;
  const int r0 = warp * 16 + (lane >> 2);
  if (a0 < a1) load(a0);
  for (long long ab = a0; ab < a1; ab += TD_KC) {
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int idx = tid + TD_TC_THREADS * q, r = idx >> 6, c = idx & 63;
      gs[r * TD_GS_LD + c] = gv[q];
      const uint32_t hi = to_tf32(ev[q]);
      const uint32_t lo = to_tf32(ev[q] - __uint_as_float(hi));
      const int off = c * 128 + ((((r >> 2) ^ (c & 7))) << 4) + (r & 3) * 4;   // row c (input), agent r
      *reinterpret_cast<uint32_t*>(ehi + off) = hi;
      *reinterpret_cast<uint32_t*>(elo + off) = lo;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> wgmma's async-proxy reads
    __syncthreads();
    if (ab + TD_KC < a1) load(ab + TD_KC);
    uint32_t ahi[4][4], alo[4][4];
#pragma unroll
    for (int k8 = 0; k8 < 4; ++k8) {
      const int c = 8 * k8 + (lane & 3);
      const float xs[4] = {gs[c * TD_GS_LD + r0], gs[c * TD_GS_LD + r0 + 8], gs[(c + 4) * TD_GS_LD + r0],
                           gs[(c + 4) * TD_GS_LD + r0 + 8]};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        ahi[k8][j] = to_tf32(xs[j]);
        alo[k8][j] = to_tf32(xs[j] - __uint_as_float(ahi[k8][j]));
      }
    }
    float part[32];
#pragma unroll
    for (int q = 0; q < 32; ++q) part[q] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k8 = 0; k8 < 4; ++k8) {
      const uint64_t dhi = wgmma_desc_sw128(ehi + k8 * 32), dlo = wgmma_desc_sw128(elo + k8 * 32);
      wgmma_tf32(part, alo[k8], dhi);                              // small terms first
      wgmma_tf32(part, ahi[k8], dlo);
      wgmma_tf32(part, ahi[k8], dhi);
    }
    wgmma_commit();
    wgmma_wait0();
#pragma unroll
    for (int q = 0; q < 32; ++q) acc[q] += (double)part[q];
    __syncthreads();                                               // the stage buffers are rewritten next round
  }
  // D fragment d[4 j + 2 h + e] = (cell r0 + 8 h, input 8 j + 2 (lane % 4) + e)
  double* dst = k.part + (size_t)blockIdx.y * k.n_cells * k.n_in;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int i = i0 + r0 + 8 * h;
    if (i >= k.n_cells) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = j0 + 8 * j + 2 * (lane & 3) + e;
        if (col < k.n_in) dst[(size_t)i * k.n_in + col] = acc[4 * j + 2 * h + e];
      }
  }
}

struct TdApplyK {
  const double* part;   // (splits, n, n_in)
  double* w;            // (n, n_in) master
  float* whi;           // (n_pad, k_pad)
  float* wlo;
  int n_cells, n_in, k_pad, splits;
  double n_rows, c_grad, c_decay;   // c_grad = dt * eta, c_decay = eta * dt * L2 (the reference's products)
};

// WARP: one warp per weight, lane l sums chunks l, l + 32, ... in order, then a fixed shuffle tree (many chunks);
// else one thread per weight summing the chunks in order.
template <bool WARP>
__global__ void k_td_apply(const __grid_constant__ TdApplyK k) {
  const long long idx = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / (WARP ? 32 : 1);
  if (idx >= (long long)k.n_cells * k.n_in) return;
  const size_t nw = (size_t)k.n_cells * k.n_in;
  double s = 0.0;
  if constexpr (WARP) {
    const int lane = threadIdx.x & 31;
    for (int c = lane; c < k.splits; c += 32) s = __dadd_rn(s, k.part[(size_t)c * nw + idx]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_down_sync(0xffffffffu, s, o));
    if (lane != 0) return;
  } else {
    for (int c = 0; c < k.splits; ++c) s = __dadd_rn(s, k.part[(size_t)c * nw + idx]);
  }
  const double w = k.w[idx];
  const double dw = __dsub_rn(__dmul_rn(k.c_grad, __ddiv_rn(s, k.n_rows)), __dmul_rn(k.c_decay, w));
  const double nwv = __dadd_rn(w, dw);
  k.w[idx] = nwv;
  const int i = (int)(idx / k.n_in), j = (int)(idx - (long long)i * k.n_in);
  const float x = (float)nwv;
  uint32_t hi;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  const float xh = __uint_as_float(hi);
  uint32_t lo;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(x - xh));
  k.whi[(size_t)i * k.k_pad + j] = xh;
  k.wlo[(size_t)i * k.k_pad + j] = __uint_as_float(lo);
}

struct TdResetK {
  float* rows[3];                          // fr_prev, deriv, td_error
  long long ld, n_rows;
  float* trace[RIAB_FFL_MAX_INPUTS];
  long long trace_ld[RIAB_FFL_MAX_INPUTS];
  int n_inputs;
  const uint8_t* mask;
};

__global__ void k_td_reset(const __grid_constant__ TdResetK k) {
  const long long row = blockIdx.x;
  if (row >= k.n_rows || (k.mask != nullptr && k.mask[row] == 0)) return;
  for (int b = 0; b < 3; ++b)
    if (k.rows[b])
      for (long long c = threadIdx.x; c < k.ld; c += blockDim.x) k.rows[b][row * k.ld + c] = 0.f;
  for (int l = 0; l < k.n_inputs; ++l)
    for (long long c = threadIdx.x; c < k.trace_ld[l]; c += blockDim.x) k.trace[l][row * k.trace_ld[l] + c] = 0.f;
}

// ---- per-agent weights
struct TdFwdPaK {
  const float* in[RIAB_FFL_MAX_INPUTS];       // input rows (in_ld floats apart, 16-byte aligned); NULL = zeros
  long long in_ld[RIAB_FFL_MAX_INPUTS];
  const double* w[RIAB_FFL_MAX_INPUTS];       // (A, n_cells, n_in[l]) masters
  int n_in[RIAB_FFL_MAX_INPUTS];
  int soff[RIAB_FFL_MAX_INPUTS];              // input l's offset in a staged row (floats, a multiple of 4)
  int n_inputs, n_cells, stage_ld, rows_per_cta;
  ActK act;
  const float* bias;                          // (n_cells)
  const long long* w_row;                     // weight agent of each row, NULL = the row itself
  const long long* in_row;                    // input row of each row, NULL = the row itself
  const double* pos;                          // (n_rows, 2): rows whose x is NaN get zeros and keep their prime; or NULL
  float* rates;                               // (n_rows, ld)
  float* prime;                               // (n_rows, ld) or NULL
  long long ld, n_rows;
};

constexpr int TD_FWD_THREADS = 256;

// STAGED: the CTA's rows_per_cta input rows are copied to shared memory (dynamic, rows_per_cta * stage_ld floats) once and
// read by every cell's warp; otherwise (rows too long to stage) the warps read them from global memory.  Both sum in the
// same order.
template <bool STAGED>
__global__ void __launch_bounds__(TD_FWD_THREADS) k_td_forward_pa(const __grid_constant__ TdFwdPaK k) {
  extern __shared__ __align__(16) float td_xs[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r0 = (long long)blockIdx.x * k.rows_per_cta;
  const int R = (int)min((long long)k.rows_per_cta, k.n_rows - r0);
  if constexpr (STAGED) {
    for (int rr = 0; rr < R; ++rr) {
      const long long ir = k.in_row ? k.in_row[r0 + rr] : r0 + rr;
      for (int l = 0; l < k.n_inputs; ++l) {
        float4* dst = reinterpret_cast<float4*>(td_xs + (size_t)rr * k.stage_ld + k.soff[l]);
        const float4* src = k.in[l] ? reinterpret_cast<const float4*>(k.in[l] + ir * k.in_ld[l]) : nullptr;
        const int n4 = (k.n_in[l] + 3) >> 2;
        for (int q = threadIdx.x; q < n4; q += TD_FWD_THREADS) dst[q] = src ? src[q] : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    __syncthreads();
  }
  const int pairs = R * k.n_cells;
  for (int p = warp; p < pairs; p += TD_FWD_THREADS / 32) {
    const int rr = p / k.n_cells, j = p - rr * k.n_cells;
    const long long row = r0 + rr;
    const long long a = k.w_row ? k.w_row[row] : row;
    double acc = 0.0;
    for (int l = 0; l < k.n_inputs; ++l) {
      if (k.in[l] == nullptr) continue;
      const int n_in = k.n_in[l];
      const double* w = k.w[l] + ((size_t)a * k.n_cells + j) * n_in;
      const float* x;
      if constexpr (STAGED) x = td_xs + (size_t)rr * k.stage_ld + k.soff[l];
      else x = k.in[l] + (k.in_row ? k.in_row[row] : row) * k.in_ld[l];
#pragma unroll 4
      for (int i = lane; i < n_in; i += 32) acc = fma(__ldcs(w + i), (double)x[i], acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
    if (lane == 0) {
      const bool nan_row = k.pos != nullptr && isnan(k.pos[2 * row]);
      float v, dv;
      layer_activate(k.act, (float)__dadd_rn(acc, (double)k.bias[j]), v, dv);
      k.rates[row * k.ld + j] = nan_row ? 0.f : v;
      if (k.prime != nullptr && !nan_row) k.prime[row * k.ld + j] = dv;
    }
  }
}

struct TdLearnPaK {
  const float* td;        // (A, ld) td_error, written by k_td_g
  const float* prime;     // (A, ld)
  const float* e;         // (A, lde) the input's traces
  double* w;              // (A, n_cells, n_in) masters
  long long ld, lde;
  int n_cells, n_in;
  double c_grad, c_decay; // dt * eta, eta * dt * L2 (the reference's products)
};

constexpr int TD_LEARN_PA_THREADS = 128;

// one CTA per agent, its n_cells x n_in block in order; dw = (dt eta) (g e) - (eta dt L2) w, w + dw, as the reference
// evaluates np.outer and its two products, with g = td phi' formed in float64 from the float32 td and phi'
__global__ void __launch_bounds__(TD_LEARN_PA_THREADS) k_td_learn_pa(const __grid_constant__ TdLearnPaK k) {
  const long long a = blockIdx.x;
  const int nw = k.n_cells * k.n_in;
  double* w = k.w + (size_t)a * nw;
  const float* e = k.e + a * k.lde;
  for (int idx = threadIdx.x; idx < nw; idx += TD_LEARN_PA_THREADS) {
    const int j = idx / k.n_in, i = idx - j * k.n_in;
    const double g = __dmul_rn((double)k.td[a * k.ld + j], (double)k.prime[a * k.ld + j]);
    const double wv = __ldcs(w + idx);
    const double dw = __dsub_rn(__dmul_rn(k.c_grad, __dmul_rn(g, (double)e[i])), __dmul_rn(k.c_decay, wv));
    __stcs(w + idx, __dadd_rn(wv, dw));
  }
}

}  // namespace riab

// FeedForwardLayer GEMM on sm_90a: rates[a, i] = phi(sum_l sum_j W_l[i, j] I_l[a, j] + b[i]) with error-compensated
// ("3xTF32") wgmma and fp32 accumulation.  x = hi + lo with hi = tf32(x) and lo = tf32(x - hi); the three products
// hi.hi + hi.lo + lo.hi keep ~2^-21 relative accuracy per term (single-pass TF32 keeps 2^-11).
//
// Layout (FFL_BM = 128 agents x BN = 8, 32 or 64 cells per CTA, K in steps of FFL_BK = 32 floats = one 128-byte swizzle row):
//   * one producer warp issues 2-D TMA loads of the input tile (FFL_BM x 32) and the W_hi / W_lo tiles (BN x 32), all
//     128-byte swizzled, into a ring of FFL_STAGES stages guarded by full / empty mbarriers;
//   * two consumer warpgroups (64 agents each) read their A fragments from shared memory, split them into hi / lo in
//     registers (A-from-registers wgmma) and issue m64nBNk8 wgmmas whose B operand is the swizzled W tile (K-major);
//   * the epilogue adds the bias, applies the activation in accurate float32 and stores the n real columns.
// The input tensor maps have inner dimension n_in, not the row stride: TMA's out-of-bounds zero fill covers the K tail
// and the agent tail, and the pad columns of a rate row (uninitialised memory, possibly NaN) are never read.
#pragma once
#include <cuda.h>
#include "riab_common.cuh"

namespace riab {

constexpr int FFL_BM = 128;
constexpr int FFL_BK = 32;
constexpr int FFL_STAGES = 4;
constexpr int FFL_CONSUMER_WARPS = 8;
constexpr int FFL_THREADS = 32 * FFL_CONSUMER_WARPS + 32;

struct FflK {
  CUtensorMap in[RIAB_FFL_MAX_INPUTS];    // (n_rows, n_in) input rows, box (32, FFL_BM)
  CUtensorMap whi[RIAB_FFL_MAX_INPUTS];   // (n_pad, k_pad) W_hi, box (32, BN)
  CUtensorMap wlo[RIAB_FFL_MAX_INPUTS];   // (n_pad, k_pad) W_lo, box (32, BN)
  int ktiles[RIAB_FFL_MAX_INPUTS];
  int n_inputs, n_cells, n_tiles, act;
  long long n_rows, ld;
  float* rates;
  float* prime;
  const float* bias;
  const double* pos;
  float p0, p1, p2, p3;
};

template <int BN>
constexpr int ffl_stage_bytes() { return FFL_BM * FFL_BK * 4 + 2 * BN * FFL_BK * 4; }
template <int BN>
constexpr int ffl_smem_bytes() { return FFL_STAGES * ffl_stage_bytes<BN>() + 1024; }   // + alignment slack

RIAB_DEV void tma_2d(void* smem_dst, const CUtensorMap* map, int x, int y, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(smem_u32(bar))
               : "memory");
}

RIAB_DEV uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

// wgmma shared-memory matrix descriptor: K-major, 128-byte swizzle, 8-row groups 1024 bytes apart (SBO), LBO unused.
RIAB_DEV uint64_t wgmma_desc_sw128(const void* smem) {
  const uint64_t addr = smem_u32(smem);
  return ((addr & 0x3FFFFull) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
RIAB_DEV void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
RIAB_DEV void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
RIAB_DEV void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// m64nNk8 tf32 wgmma, A from registers, D += A.B (one overload per N tile)
RIAB_DEV void wgmma_tf32(float (&d)[4], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %9, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3}, "
      "{%4,%5,%6,%7}, %8, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
}
RIAB_DEV void wgmma_tf32(float (&d)[16], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, "
      "{%16,%17,%18,%19}, %20, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
}
RIAB_DEV void wgmma_tf32(float (&d)[32], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "{%32,%33,%34,%35}, %36, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
}

// 1 - tanh(x)^2 without cancellation: 4 e / (1 + e)^2 with e = exp(-2|x|)
RIAB_DEV float sech2f(float x) {
  const float e = expf(-2.f * fabsf(x));
  const float d = 1.f + e;
  return 4.f * e / (d * d);
}

// utils.activate (utils.py:919-1026) and its derivative, accurate float32; `act` is uniform across the grid.  The one
// epilogue of every FeedForwardLayer-like contraction (k_ffl here, k_td_forward_pa in riab_td.cuh).
struct ActK {
  int act;
  float p0, p1, p2, p3;
};
RIAB_DEV void layer_activate(const ActK& k, float x, float& v, float& dv) {
  switch (k.act) {
    case RIAB_ACT_SIGMOID: {          // p0 max_fr, p1 min_fr, p2 mid_x, p3 beta
      const float z = k.p3 * (x - k.p2);
      const float e = expf(-z);
      v = (k.p0 - k.p1) / (1.f + e) + k.p1;
      // beta (f - min)(1 - (f - min)/(max - min)) = beta span s (1 - s), s (1 - s) = e' / (1 + e')^2 with e' = exp(-|z|)
      const float ea = expf(-fabsf(z));
      const float d = 1.f + ea;
      dv = k.p3 * (k.p0 - k.p1) * (ea / (d * d));
      break;
    }
    case RIAB_ACT_RELU:               // p0 gain, p1 threshold
      v = k.p0 * fmaxf(0.f, x - k.p1);
      dv = (x - k.p1 > 0.f) ? k.p0 : 0.f;
      break;
    case RIAB_ACT_TANH:               // the reference's derivative ignores the threshold (utils.py:1001)
      v = k.p0 * tanhf(x - k.p1);
      dv = k.p0 * sech2f(x);
      break;
    case RIAB_ACT_RETANH:             // only retanh masks the derivative by x - threshold > 0 (utils.py:1011-1015)
      v = k.p0 * fmaxf(0.f, tanhf(x - k.p1));
      dv = (x - k.p1 > 0.f) ? k.p0 * sech2f(x) : 0.f;
      break;
    case RIAB_ACT_SOFTPLUS: {         // gain log(1 + exp(z)), overflow-safe; derivative gain / (1 + exp(-z))
      const float z = x - k.p1;
      v = k.p0 * (fmaxf(z, 0.f) + log1pf(expf(-fabsf(z))));
      dv = k.p0 / (1.f + expf(-z));
      break;
    }
    default:
      v = x;
      dv = 1.f;
  }
}
RIAB_DEV void ffl_activate(const FflK& k, float x, float& v, float& dv) {
  layer_activate(ActK{k.act, k.p0, k.p1, k.p2, k.p3}, x, v, dv);
}

template <int BN>
__global__ void __launch_bounds__(FFL_THREADS, 1) k_ffl(const __grid_constant__ FflK k) {
  constexpr int A_BYTES = FFL_BM * FFL_BK * 4, W_BYTES = BN * FFL_BK * 4;
  extern __shared__ uint8_t ffl_smem_raw[];
  __shared__ __align__(8) uint64_t full[FFL_STAGES], empty[FFL_STAGES];
  // 128-byte swizzle atoms are 1024 bytes: align the stage buffers to them
  uint8_t* smem = ffl_smem_raw + ((1024u - (smem_u32(ffl_smem_raw) & 1023u)) & 1023u);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = (int)(blockIdx.x % (unsigned)k.n_tiles);          // output tiles of one agent tile are adjacent (L2)
  const long long m0 = (long long)(blockIdx.x / (unsigned)k.n_tiles) * FFL_BM;
  const int n0 = nt * BN;
  if (threadIdx.x == 0) {
    for (int s = 0; s < FFL_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], FFL_CONSUMER_WARPS); }
    mbar_fence_init();
  }
  __syncthreads();
  int total = 0;
  for (int l = 0; l < k.n_inputs; ++l) total += k.ktiles[l];

  if (warp == FFL_CONSUMER_WARPS) {                                // ---- producer warp
    if (lane == 0) {
      int it = 0;
      for (int l = 0; l < k.n_inputs; ++l) {
        for (int kt = 0; kt < k.ktiles[l]; ++kt, ++it) {
          const int s = it % FFL_STAGES;
          if (it >= FFL_STAGES) mbar_wait(&empty[s], ((it / FFL_STAGES) - 1) & 1);
          uint8_t* st = smem + (size_t)s * ffl_stage_bytes<BN>();
          mbar_expect_tx(&full[s], A_BYTES + 2 * W_BYTES);
          tma_2d(st, &k.in[l], kt * FFL_BK, (int)m0, &full[s]);
          tma_2d(st + A_BYTES, &k.whi[l], kt * FFL_BK, n0, &full[s]);
          tma_2d(st + A_BYTES + W_BYTES, &k.wlo[l], kt * FFL_BK, n0, &full[s]);
        }
      }
    }
    return;
  }

  // ---- consumers: warpgroup g owns agents m0 + 64 g .. +63, warp w of it rows 16 w .. 16 w + 15
  float acc[BN / 2], part[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  const int g = warp >> 2, w = warp & 3;
  const int r0 = g * 64 + w * 16 + (lane >> 2);                    // tile rows of a0 / a2; a1 / a3 are r0 + 8
  for (int it = 0; it < total; ++it) {
    const int s = it % FFL_STAGES;
    mbar_wait(&full[s], (it / FFL_STAGES) & 1);
    const uint8_t* st = smem + (size_t)s * ffl_stage_bytes<BN>();
    uint32_t ahi[4][4], alo[4][4];
#pragma unroll
    for (int k8 = 0; k8 < 4; ++k8) {
      // A fragment (m64k8 tf32): a0 (r0, c), a1 (r0 + 8, c), a2 (r0, c + 4), a3 (r0 + 8, c + 4), c = 8 k8 + lane % 4.
      // 128-byte swizzle: the 16-byte chunk q of row r sits at chunk q ^ (r % 8); (r0 + 8) % 8 == r0 % 8.
      const int q0 = 2 * k8, q1 = 2 * k8 + 1, sw = r0 & 7, e = (lane & 3) * 4;
      const float x0 = *reinterpret_cast<const float*>(st + r0 * 128 + ((q0 ^ sw) << 4) + e);
      const float x1 = *reinterpret_cast<const float*>(st + (r0 + 8) * 128 + ((q0 ^ sw) << 4) + e);
      const float x2 = *reinterpret_cast<const float*>(st + r0 * 128 + ((q1 ^ sw) << 4) + e);
      const float x3 = *reinterpret_cast<const float*>(st + (r0 + 8) * 128 + ((q1 ^ sw) << 4) + e);
      const float xs[4] = {x0, x1, x2, x3};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        ahi[k8][j] = to_tf32(xs[j]);
        alo[k8][j] = to_tf32(xs[j] - __uint_as_float(ahi[k8][j]));
      }
    }
    // each stage accumulates into a zeroed partial sum that is then added with IEEE round-to-nearest: the tensor cores'
    // fp32 accumulation is not round-to-nearest, and over a long K its rounding errors pile up one-sidedly
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) part[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k8 = 0; k8 < 4; ++k8) {
      // advancing K by 8 tf32 = 32 bytes inside the swizzled 128-byte rows moves the descriptor's start address
      const uint64_t dhi = wgmma_desc_sw128(st + A_BYTES + k8 * 32);
      const uint64_t dlo = wgmma_desc_sw128(st + A_BYTES + W_BYTES + k8 * 32);
      wgmma_tf32(part, alo[k8], dhi);                              // small terms first
      wgmma_tf32(part, ahi[k8], dlo);
      wgmma_tf32(part, ahi[k8], dhi);
    }
    wgmma_commit();
    wgmma_wait0();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }

  // ---- epilogue: D fragment d[4 j + 2 h + e] = (row r0 + 8 h, column 8 j + 2 (lane % 4) + e)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long long row = m0 + r0 + 8 * h;
    if (row >= k.n_rows) continue;
    const bool nan_row = k.pos != nullptr && isnan(k.pos[2 * row]);
    float* dst = k.rates + row * k.ld;
    float* dp = k.prime ? k.prime + row * k.ld : nullptr;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = n0 + 8 * j + 2 * (lane & 3) + e;
        if (col < k.n_cells) {
          float v, dv;
          ffl_activate(k, acc[4 * j + 2 * h + e] + k.bias[col], v, dv);
          dst[col] = nan_row ? 0.f : v;
          if (dp != nullptr && !nan_row) dp[col] = dv;
        }
      }
    }
  }
}

}  // namespace riab

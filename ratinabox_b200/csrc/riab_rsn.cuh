// RandomSpatialNeurons.get_state (ratinabox/Neurons.py:2916-2941) on sm_90a:
//   rate[a, i] = sum_j k[a, j] T[j, i] / sum_j k[a, j],   k[a, j] = exp(-d(pos_a, X_j)^2 / 2 l^2)
// in ONE kernel: k_ffl's pipeline (riab_ffl.cuh) with the A operand generated in registers instead of loaded.
//
//   * CTA = 64 CWG agents (CWG consumer warpgroups) x BN output columns, K in stages of FFL_BK = 32 sample points.
//     One producer warp TMA-loads the T_hi / T_lo tiles (BN x 32, 128-byte swizzle) into a ring of RSN_STAGES stages,
//     exactly as k_ffl loads W_hi / W_lo.  The sample points' parameters are read by the consumers through L1 (the
//     block is a few KB per stage, shared by every CTA), not staged.
//   * A consumer thread's A fragments of a stage are its two agent rows (r0, r0 + 8) at the 8 columns 8 k8 + lane % 4
//     (+ 4).  riab_rsn_pack lays X out so that these 8 columns are the packed points 8 (lane % 4) .. + 7 of the stage:
//     two runs of 4, each one place_rates4 call (riab_place.cuh, DEFER = false: a flagged line-of-sight group takes
//     the exact float64 path at once) per agent row on the agent records built once per CTA by place_agent_record.
//     The first run gives the fragments of k8 = 0, 1, the second those of k8 = 2, 3.
//   * The kernel values are split into tf32 hi / lo and contracted 3xTF32 like k_ffl, each stage into a zeroed partial
//     sum that is then added with IEEE FADD.  The normaliser sum_j k[a, j] is accumulated in float64 from the same
//     float32 values, per thread in a fixed order, then over the quad in lane order: deterministic, no atomics.
//   * Sample points past |X| (the K tail of the last stage) are zeroed before both sums.
//   * Epilogue: num / den in float64, rounded once; zeros for NaN positions; the n real columns are stored.
// Registers: the 288 threads of two consumer warpgroups + the producer put 3 warps on one SM sub-partition, which caps a
// thread at 168 registers; the point registers of 4 and 8 inner walls (PlaceCellRegs) do not fit next to the
// accumulators there, so those geometries run one consumer warpgroup (160 threads: 255 registers).
#pragma once
#include "riab_ffl.cuh"
#include "riab_place.cuh"

namespace riab {

constexpr int RSN_STAGES = 4;

struct RsnK {
  CUtensorMap thi, tlo;            // (n_pad8, k_pad) T_hi / T_lo, box (32, BN)
  PlaceConst pc;                   // the sample points (n_cells = k_pad), gaussian, [0, 1], direct (not expanded) form
  const double* walls;             // env walls (float64), the inner ones from pc.wall0
  int n_cells, n_tiles, ktiles, n_points;
  long long n_rows, ld;
  float* rates;
  const double* pos;               // (n_rows, 2) f64
};

template <int BN>
constexpr int rsn_stage_bytes() { return 2 * BN * FFL_BK * 4; }
template <int BN>
constexpr int rsn_smem_bytes() { return RSN_STAGES * rsn_stage_bytes<BN>() + 1024; }   // + alignment slack

// packed position p (0..31) of a stage -> the K column of the stage it holds (riab_rsn_pack uses the same map):
// p = 8 q + 2 k8 + h  ->  column 8 k8 + q + 4 h
RIAB_HD int rsn_k_of_packed(int p) { return 8 * ((p & 7) >> 1) + (p >> 3) + 4 * (p & 1); }

template <int CWG>
constexpr int rsn_threads() { return 128 * CWG + 32; }

template <int WI, int DESC, int BN, int CWG>
__global__ void __launch_bounds__(rsn_threads<CWG>(), 1) k_rsn(const __grid_constant__ RsnK k) {
  constexpr bool GEO = DESC < 0;      // the run-time profile kernel is the geodesic one (launch_rsn): GEO agent records
  constexpr int BM = 64 * CWG, CONSUMER_WARPS = 4 * CWG;
  constexpr int T_BYTES = BN * FFL_BK * 4;
  constexpr int REC = place_rec(WI, GEO);
  extern __shared__ uint8_t rsn_smem_raw[];
  __shared__ __align__(8) uint64_t full[RSN_STAGES], empty[RSN_STAGES];
  __shared__ __align__(16) float s_rec[BM * REC];
  __shared__ __align__(16) double s_inner[4 * (WI > 0 ? WI : 1)];
  __shared__ double s_aux[2 * PLACE_MAX_WI];
  uint8_t* smem = rsn_smem_raw + ((1024u - (smem_u32(rsn_smem_raw) & 1023u)) & 1023u);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = (int)(blockIdx.x % (unsigned)k.n_tiles);
  const long long m0 = (long long)(blockIdx.x / (unsigned)k.n_tiles) * BM;
  const int n0 = nt * BN;
  const PlaceConst& pc = k.pc;
  const int n_inner = WI > 0 ? pc.n_inner : 0;
  if (threadIdx.x == 0) {
    for (int s = 0; s < RSN_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], CONSUMER_WARPS); }
    mbar_fence_init();
  }
  for (int i = threadIdx.x; i < 4 * n_inner; i += blockDim.x) s_inner[i] = k.walls[4 * pc.wall0 + i];
  __syncthreads();
  place_wall_invariants(s_aux, s_inner, n_inner);
  __syncthreads();
  if (threadIdx.x < BM) {                                      // one record per agent row of the tile
    const long long row = m0 + threadIdx.x;
    const double px = row < k.n_rows ? k.pos[2 * row] : pc.cxm, py = row < k.n_rows ? k.pos[2 * row + 1] : pc.cym;
    place_agent_record<WI, false, GEO>(s_rec + threadIdx.x * REC, px, py, s_inner, s_aux, n_inner, pc.cxm, pc.cym,
                                       pc.band, 0, 0.f, 0.f);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {                                // ---- producer warp
    if (lane == 0) {
      for (int it = 0; it < k.ktiles; ++it) {
        const int s = it % RSN_STAGES;
        if (it >= RSN_STAGES) mbar_wait(&empty[s], ((it / RSN_STAGES) - 1) & 1);
        uint8_t* st = smem + (size_t)s * rsn_stage_bytes<BN>();
        mbar_expect_tx(&full[s], 2 * T_BYTES);
        tma_2d(st, &k.thi, it * FFL_BK, n0, &full[s]);
        tma_2d(st + T_BYTES, &k.tlo, it * FFL_BK, n0, &full[s]);
      }
    }
    return;
  }

  // ---- consumers: warpgroup g owns agents m0 + 64 g .. +63, warp w of it rows 16 w .. 16 w + 15
  float acc[BN / 2], part[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  double den[2] = {0.0, 0.0};
  const int g = warp >> 2, w = warp & 3, q = lane & 3;
  const int r0 = g * 64 + w * 16 + (lane >> 2);
  const float* rec0 = s_rec + r0 * REC;
  const float* rec1 = s_rec + (r0 + 8) * REC;
  const uint32_t inner_s = smem_u32(s_inner);
  for (int it = 0; it < k.ktiles; ++it) {
    const int s = it % RSN_STAGES;
    // the kernel values of this stage (before waiting for its targets: the generation overlaps the TMA)
    uint32_t ahi[4][4], alo[4][4];
    const bool tail = (it + 1) * FFL_BK > k.n_points;             // the last stage holds pad points
#pragma unroll
    for (int run = 0; run < 2; ++run) {                            // packed points 8 q + 4 run .. + 3: k8 = 2 run, 2 run + 1
      const int cell0 = it * FFL_BK + 8 * q + 4 * run;
      PlaceCellRegs<WI> r;
      place_load_cells<WI, false, GEO>(r, pc, cell0);
      float v0[4], v1[4];
      bool unsure = false;
      place_rates4<WI, DESC, false, 0, false, GEO>(v0, r, pc, cell0, rec0, inner_s, unsure);
      place_rates4<WI, DESC, false, 0, false, GEO>(v1, r, pc, cell0, rec1, inner_s, unsure);
      if (tail) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (it * FFL_BK + rsn_k_of_packed(8 * q + 4 * run + i) >= k.n_points) { v0[i] = 0.f; v1[i] = 0.f; }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) { den[0] += (double)v0[i]; den[1] += (double)v1[i]; }
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        // a0 (r0, c), a1 (r0 + 8, c), a2 (r0, c + 4), a3 (r0 + 8, c + 4): packed 2 kk (column c), 2 kk + 1 (c + 4)
        const float xs[4] = {v0[2 * kk], v1[2 * kk], v0[2 * kk + 1], v1[2 * kk + 1]};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          ahi[2 * run + kk][j] = to_tf32(xs[j]);
          alo[2 * run + kk][j] = to_tf32(xs[j] - __uint_as_float(ahi[2 * run + kk][j]));
        }
      }
    }
    mbar_wait(&full[s], (it / RSN_STAGES) & 1);
    const uint8_t* st = smem + (size_t)s * rsn_stage_bytes<BN>();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) part[i] = 0.f;
    __syncwarp();                                                  // reconverge after the exact fall-back
    wgmma_fence();
#pragma unroll
    for (int k8 = 0; k8 < 4; ++k8) {
      const uint64_t dhi = wgmma_desc_sw128(st + k8 * 32);
      const uint64_t dlo = wgmma_desc_sw128(st + T_BYTES + k8 * 32);
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

  // ---- epilogue: the quad's normaliser in lane order, then D fragment d[4 j + 2 h + e] = (row r0 + 8 h, col 8 j + 2 q + e)
  const int base = lane & ~3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const double d0 = __shfl_sync(0xffffffffu, den[h], base), d1 = __shfl_sync(0xffffffffu, den[h], base + 1);
    const double d2 = __shfl_sync(0xffffffffu, den[h], base + 2), d3 = __shfl_sync(0xffffffffu, den[h], base + 3);
    den[h] = ((d0 + d1) + d2) + d3;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long long row = m0 + r0 + 8 * h;
    if (row >= k.n_rows) continue;
    const bool nan_row = isnan(k.pos[2 * row]);
    float* dst = k.rates + row * k.ld;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = n0 + 8 * j + 2 * q + e;
        if (col < k.n_cells) dst[col] = nan_row ? 0.f : (float)((double)acc[4 * j + 2 * h + e] / den[h]);
      }
    }
  }
}

}  // namespace riab

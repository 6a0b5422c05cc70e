// NeuralNetworkNeurons kernels (see riab_nnn.cuh).
#include "riab_nnn.cuh"

namespace riab {

RIAB_DEV float nnn_activate(int act, float x) {
  switch (act) {
    case RIAB_NNN_RELU: return fmaxf(x, 0.f);
    case RIAB_NNN_SIGMOID: return 1.f / (1.f + expf(-x));
    case RIAB_NNN_TANH: return tanhf(x);
    default: return x;
  }
}

RIAB_DEV void nnn_consumer_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

template <int BN>
__global__ void __launch_bounds__(NNN_THREADS) k_nnn(const __grid_constant__ NnnK k) {
  constexpr int A_BYTES = NNN_BM * FFL_BK * 4, W_BYTES = BN * FFL_BK * 4;
  extern __shared__ uint8_t nnn_smem_raw[];
  __shared__ __align__(8) uint64_t full[NNN_STAGES], empty[NNN_STAGES];
  uint8_t* smem = nnn_smem_raw + ((1024u - (smem_u32(nnn_smem_raw) & 1023u)) & 1023u);
  float* hbuf = reinterpret_cast<float*>(smem + NNN_STAGES * nnn_stage_bytes<BN>());
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long m0 = (long long)blockIdx.x * NNN_BM;
  if (threadIdx.x == 0) {
    for (int s = 0; s < NNN_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    mbar_fence_init();
  }
  __syncthreads();
  int per_chunk = 0;
  for (int l = 0; l < k.n_inputs; ++l) per_chunk += k.ktiles[l];

  if (warp == 4) {                                                 // ---- producer warp
    if (lane == 0) {
      int it = 0;
      for (int c = 0; c < k.n_chunks; ++c)
        for (int l = 0; l < k.n_inputs; ++l)
          for (int kt = 0; kt < k.ktiles[l]; ++kt, ++it) {
            const int s = it % NNN_STAGES;
            if (it >= NNN_STAGES) mbar_wait(&empty[s], ((it / NNN_STAGES) - 1) & 1);
            uint8_t* st = smem + (size_t)s * nnn_stage_bytes<BN>();
            mbar_expect_tx(&full[s], A_BYTES + 2 * W_BYTES);
            tma_2d(st, &k.in[l], kt * FFL_BK, (int)m0, &full[s]);
            tma_2d(st + A_BYTES, &k.whi[l], kt * FFL_BK, c * BN, &full[s]);
            tma_2d(st + A_BYTES + W_BYTES, &k.wlo[l], kt * FFL_BK, c * BN, &full[s]);
          }
    }
    return;
  }

  // ---- layer 1: warp w owns tile rows 16 w .. 16 w + 15 (the fragment layout of k_ffl)
  const int r0 = warp * 16 + (lane >> 2);
  const int h1 = k.widths[1];
  const bool single = k.n_layers == 1;
  float acc[BN / 2], part[BN / 2];
  int it = 0;
  for (int c = 0; c < k.n_chunks; ++c) {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int j = 0; j < per_chunk; ++j, ++it) {
      const int s = it % NNN_STAGES;
      mbar_wait(&full[s], (it / NNN_STAGES) & 1);
      const uint8_t* st = smem + (size_t)s * nnn_stage_bytes<BN>();
      uint32_t ahi[4][4], alo[4][4];
#pragma unroll
      for (int k8 = 0; k8 < 4; ++k8) {
        const int q0 = 2 * k8, q1 = 2 * k8 + 1, sw = r0 & 7, e = (lane & 3) * 4;
        const float xs[4] = {*reinterpret_cast<const float*>(st + r0 * 128 + ((q0 ^ sw) << 4) + e),
                             *reinterpret_cast<const float*>(st + (r0 + 8) * 128 + ((q0 ^ sw) << 4) + e),
                             *reinterpret_cast<const float*>(st + r0 * 128 + ((q1 ^ sw) << 4) + e),
                             *reinterpret_cast<const float*>(st + (r0 + 8) * 128 + ((q1 ^ sw) << 4) + e)};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          ahi[k8][q] = to_tf32(xs[q]);
          alo[k8][q] = to_tf32(xs[q] - __uint_as_float(ahi[k8][q]));
        }
      }
      // a zeroed partial sum per stage, added with round-to-nearest (see k_ffl)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) part[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int k8 = 0; k8 < 4; ++k8) {
        const uint64_t dhi = wgmma_desc_sw128(st + A_BYTES + k8 * 32);
        const uint64_t dlo = wgmma_desc_sw128(st + A_BYTES + W_BYTES + k8 * 32);
        wgmma_tf32(part, alo[k8], dhi);
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
    // chunk epilogue: D fragment d[4 j + 2 h + e] = (row r0 + 8 h, column c BN + 8 j + 2 (lane % 4) + e)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + 8 * h;
      const long long row = m0 + r;
      const bool nan_row = single && row < k.n_rows && k.pos != nullptr && isnan(k.pos[2 * row]);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = c * BN + 8 * j + 2 * (lane & 3) + e;
          if (col >= h1) continue;
          const float v = nnn_activate(k.act[0], acc[4 * j + 2 * h + e] + k.bias1[col]);
          if (!single) hbuf[r * k.h_ld + col] = v;
          else if (row < k.n_rows) k.rates[row * k.ld + col] = nan_row ? 0.f : v;
        }
      }
    }
  }
  if (single) return;

  // ---- layers 2..L: thread t owns agent t % 64 and the 8-column blocks 8 (t / 64) + 16 m
  const int a = threadIdx.x & (NNN_BM - 1), half = threadIdx.x >> 6;
  const long long row = m0 + a;
  const bool live = row < k.n_rows;
  const bool nan_row = live && k.pos != nullptr && isnan(k.pos[2 * row]);
  const float* wl = k.bias1 + ((h1 + 7) & ~7);
  float* hin = hbuf;
  float* hout = hbuf + NNN_BM * k.h_ld;
  for (int l = 2; l <= k.n_layers; ++l) {
    nnn_consumer_sync();                                           // layer l - 1's activations are complete
    const int ni = k.widths[l - 1], no = k.widths[l], no8 = (no + 7) & ~7, act = k.act[l - 1];
    const float* b = wl + (size_t)ni * no8;
    const bool out_layer = l == k.n_layers;
    const float* x = hin + a * k.h_ld;
    for (int j0 = 8 * half; j0 < no; j0 += 16) {
      float s[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) s[q] = 0.f;
      const float* w = wl + j0;
#pragma unroll 4
      for (int i = 0; i < ni; ++i, w += no8) {
        const float xi = x[i];
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(w)), w1 = __ldg(reinterpret_cast<const float4*>(w) + 1);
        s[0] = fmaf(w0.x, xi, s[0]); s[1] = fmaf(w0.y, xi, s[1]); s[2] = fmaf(w0.z, xi, s[2]); s[3] = fmaf(w0.w, xi, s[3]);
        s[4] = fmaf(w1.x, xi, s[4]); s[5] = fmaf(w1.y, xi, s[5]); s[6] = fmaf(w1.z, xi, s[6]); s[7] = fmaf(w1.w, xi, s[7]);
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int col = j0 + q;
        if (col >= no) break;
        const float v = nnn_activate(act, s[q] + b[col]);
        if (!out_layer) hout[a * k.h_ld + col] = v;
        else if (live) k.rates[row * k.ld + col] = nan_row ? 0.f : v;
      }
    }
    wl = b + no8;
    float* t = hin; hin = hout; hout = t;
  }
}

// n_layers == 0: rates the caller computed, copied into the rate rows with the NaN-position mask
__global__ void __launch_bounds__(256) k_nnn_rows(const float* __restrict__ in, long long ld_in, float* out, long long ld,
                                                  int n, long long n_rows, const double* pos) {
  const long long row = blockIdx.x;
  if (row >= n_rows) return;
  const bool nan_row = pos != nullptr && isnan(pos[2 * row]);
  for (int c = threadIdx.x; c < n; c += blockDim.x) out[row * ld + c] = nan_row ? 0.f : in[row * ld_in + c];
}


template <int BN>
cudaError_t nnn_launch_bn(NnnK& k, cudaStream_t s) {
  const size_t smem = nnn_smem_bytes<BN>(k.h_ld);
  cudaError_t e = cudaFuncSetAttribute(k_nnn<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k.n_chunks = (k.widths[1] + BN - 1) / BN;
  k_nnn<BN><<<(unsigned)((k.n_rows + NNN_BM - 1) / NNN_BM), NNN_THREADS, smem, s>>>(k);
  return cudaGetLastError();
}

cudaError_t nnn_launch(NnnK& k, int bn, cudaStream_t s) { return bn == 32 ? nnn_launch_bn<32>(k, s) : nnn_launch_bn<64>(k, s); }

cudaError_t nnn_rows_launch(const float* in, long long ld_in, float* out, long long ld, int n, long long n_rows,
                            const double* pos, cudaStream_t s) {
  k_nnn_rows<<<(unsigned)n_rows, 256, 0, s>>>(in, ld_in, out, ld, n, n_rows, pos);
  return cudaGetLastError();
}

}  // namespace riab

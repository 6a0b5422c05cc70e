// NeuralNetworkNeurons on sm_90a: a chain of Linear layers and elementwise activations over the concatenated input rows,
// one launch per evaluation, NNN_BM = 64 agents per CTA.
//   * layer 1 (K = the inputs' total width, up to thousands): the FeedForwardLayer's error-compensated TF32 wgmma
//     (riab_ffl.cuh).  One producer warp streams the input tile (64 x 32, straight from the input populations' rows) and
//     the W_hi / W_lo tiles (BN x 32) by TMA through an mbarrier ring; one consumer warpgroup splits A into hi / lo in
//     registers.  Layer 1's outputs are produced BN columns at a time (the producer re-streams the input tiles per
//     column chunk; they come from L2 after the first), activated and written to a shared-memory buffer -- or, for a
//     single Linear, straight to the rate rows.
//   * layers 2..L: float32 FMA on the CUDA cores, the activations ping-ponging between two (64, h_ld) shared-memory
//     buffers.  Hidden widths are small (20 for the default MLP): a wgmma would pad them to the N tile, need the 3-pass
//     split for float32 accuracy, and route the activations through swizzled operand tiles, while one thread per
//     (agent, 8 outputs) reads each activation once from shared memory and the weights as warp-uniform float4 loads.
//     Each sum runs in input order with round-to-nearest FMAs, i.e. plain float32 accuracy.
// Hidden activations never leave shared memory; the output rows are written once.
// The kernels live in their own translation unit (riab_nnn.cu): riab_b200.cu, which fills NnnK and launches them through
// the functions below, then compiles to the same device code as without them.
#pragma once
#include "riab_ffl.cuh"

namespace riab {

constexpr int NNN_BM = 64;
constexpr int NNN_STAGES = 4;
constexpr int NNN_THREADS = 128 + 32;          // one consumer warpgroup + the producer warp

struct NnnK {
  CUtensorMap in[RIAB_FFL_MAX_INPUTS];         // (n_rows, n_in) input rows, box (32, NNN_BM)
  CUtensorMap whi[RIAB_FFL_MAX_INPUTS];        // (n_pad, k_pad) W_hi of layer 1's columns of the input, box (32, BN)
  CUtensorMap wlo[RIAB_FFL_MAX_INPUTS];
  int ktiles[RIAB_FFL_MAX_INPUTS];
  int n_inputs, n_layers, n_chunks, h_ld;      // h_ld: row stride of the activation buffers (odd: conflict-free columns)
  int widths[RIAB_NNN_MAX_LAYERS + 1];
  int act[RIAB_NNN_MAX_LAYERS];
  const float* bias1;                          // b_1, then per layer l >= 2: W_l^T (widths[l-1], pad8(widths[l])), b_l
  long long n_rows, ld;
  float* rates;
  const double* pos;
};

template <int BN>
constexpr int nnn_stage_bytes() { return NNN_BM * FFL_BK * 4 + 2 * BN * FFL_BK * 4; }
template <int BN>
constexpr size_t nnn_smem_bytes(int h_ld) { return (size_t)NNN_STAGES * nnn_stage_bytes<BN>() + 2 * (size_t)NNN_BM * h_ld * 4 + 1024; }

// k_nnn<BN> over ceil(k.n_rows / NNN_BM) CTAs (bn 32 or 64; sets k.n_chunks), and k_nnn_rows (n_layers == 0)
cudaError_t nnn_launch(NnnK& k, int bn, cudaStream_t s);
cudaError_t nnn_rows_launch(const float* in, long long ld_in, float* out, long long ld, int n, long long n_rows,
                            const double* pos, cudaStream_t s);

}  // namespace riab

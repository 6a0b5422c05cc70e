// Shared device helpers: non-contracting float64 wrapper, Philox4x32-10, TMA bulk
// copy + mbarrier primitives (sm_90a), cache-hinted stores.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/riab_b200.h"

#define RIAB_DEV __device__ __forceinline__
#define RIAB_HD __host__ __device__ __forceinline__

namespace riab {

// ---------------------------------------------------------------------------
// D: a float64 whose + - * / are the IEEE round-to-nearest operations and are
// never contracted into FMAs, so that expressions written in the order NumPy
// evaluates them give bit-identical results (the geometry predicates that
// decide wall collisions depend on this).
struct D {
  double v;
  RIAB_DEV D() {}
  RIAB_DEV D(double x) : v(x) {}
};
RIAB_DEV D operator+(D a, D b) { return D(__dadd_rn(a.v, b.v)); }
RIAB_DEV D operator-(D a, D b) { return D(__dsub_rn(a.v, b.v)); }
RIAB_DEV D operator*(D a, D b) { return D(__dmul_rn(a.v, b.v)); }
RIAB_DEV D operator/(D a, D b) { return D(__ddiv_rn(a.v, b.v)); }
RIAB_DEV D operator-(D a) { return D(-a.v); }
RIAB_DEV bool operator<(D a, D b) { return a.v < b.v; }
RIAB_DEV bool operator>(D a, D b) { return a.v > b.v; }
RIAB_DEV bool operator<=(D a, D b) { return a.v <= b.v; }
RIAB_DEV bool operator>=(D a, D b) { return a.v >= b.v; }
RIAB_DEV bool operator==(D a, D b) { return a.v == b.v; }
RIAB_DEV D dsqrt(D a) { return D(__dsqrt_rn(a.v)); }

// ---------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11).  Known-answer vectors are checked in
// tests/test_philox.py against a NumPy implementation of the same rounds.
RIAB_HD void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint64_t p0 = (uint64_t)0xD2511F53u * c[0];
  const uint64_t p1 = (uint64_t)0xCD9E8D57u * c[2];
  const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
  const uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
  c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
}
RIAB_HD void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}

// Philox4x32-R with the round keys precomputed (warp-uniform): 2 wide multiplies + 2 three-input
// XORs per round.
template <int R>
RIAB_DEV void philox_keyed(uint32_t (&c)[4], const uint32_t (&rk)[2 * R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) {
    unsigned long long p0, p1;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(p0) : "r"(c[0]), "r"(0xD2511F53u));
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(p1) : "r"(c[2]), "r"(0xCD9E8D57u));
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ rk[2 * i], n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ rk[2 * i + 1];
    c[1] = (uint32_t)p1; c[3] = (uint32_t)p0; c[0] = n0; c[2] = n2;
  }
}
template <int R>
RIAB_DEV void philox_round_keys(uint32_t (&rk)[2 * R], unsigned long long seed) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int i = 0; i < R; ++i) { rk[2 * i] = k0; rk[2 * i + 1] = k1; k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
}

// Stream ids (third counter word, top byte)
enum : uint32_t { RIAB_STREAM_AGENT_OU = 0, RIAB_STREAM_CELL_NOISE = 1, RIAB_STREAM_SPIKES = 2, RIAB_STREAM_MEASURE = 3,
                  RIAB_STREAM_THIN = 4,            // thinned spikes: calls n = 0, 1, ... of a (row, 128-cell block), n in bits 16.. of the sub-index
                  RIAB_STREAM_THETA_FWD = 5,       // ThetaSequenceAgent forward rollouts: sub-index = rollout, step = rollout step
                  RIAB_STREAM_DUMB = 6,            // DumbAgent: sub 0 = the displacement normals, 1 + k = k-th re-drawn position
                  RIAB_STREAM_REPLAY = 7,          // ReplayAgent decisions: sub 0, 1 = uniforms, 2 + k = k-th start position
                  RIAB_STREAM_REPLAY_FWD = 8 };    // ReplayAgent rollouts: sub-index = replay index, step = rollout step

// counter = (agent id lo32, sub-index, step lo32, (step hi & 0xffff) | stream<<24 | population<<16)
RIAB_HD void philox_ctr(uint32_t (&c)[4], uint64_t agent, uint32_t sub, uint64_t step, uint32_t stream, uint32_t pop) {
  c[0] = (uint32_t)agent;
  c[1] = sub ^ ((uint32_t)(agent >> 32) << 24);
  c[2] = (uint32_t)step;
  c[3] = ((uint32_t)(step >> 32) & 0xffffu) | ((pop & 0xffu) << 16) | (stream << 24);
}

// two uint32 -> uniform double in (0,1) with 53 random bits
RIAB_HD double u01_53(uint32_t hi, uint32_t lo) {
  const uint64_t x = (((uint64_t)hi << 32) | lo) >> 11;
  return ((double)x + 0.5) * (1.0 / 9007199254740992.0);
}
RIAB_HD float u01_24(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }

// Two standard normals of the Philox counter c (the agent OU draws): Philox4x32-10 -> two 32-bit uniforms ->
// Box-Muller in float32 (logf / sqrtf / sincospif are the accurate single-precision routines),
// widened to double.  The draws are noise: their float32 resolution is irrelevant to the
// dynamics, and float32 keeps ~150 dependent float64 operations off the motion chain.
RIAB_DEV void philox_normals(uint32_t (&c)[4], uint64_t seed, double& n1, double& n2) {
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  const float u1 = fmaf(__uint2float_rn(c[0]), 2.3283064365386963e-10f, 1.1641532182693481e-10f);   // (0,1]
  const float u2 = __uint2float_rn(c[2]) * 2.3283064365386963e-10f;                                  // [0,1]
  const float r = sqrtf(-2.0f * logf(u1));
  float s, co;
  sincospif(2.0f * u2, &s, &co);
  n1 = (double)(r * co); n2 = (double)(r * s);
}
RIAB_DEV void agent_normals(uint64_t seed, uint64_t step, uint64_t agent, double& n1, double& n2) {
  uint32_t c[4];
  philox_ctr(c, agent, 0u, step, RIAB_STREAM_AGENT_OU, 0u);
  philox_normals(c, seed, n1, n2);
}

// ---------------------------------------------------------------------------
// mbarrier + 1-D TMA bulk copy (cp.async.bulk, SASS: UBLKCP) helpers.
RIAB_DEV uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
RIAB_DEV void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
RIAB_DEV void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
RIAB_DEV void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
RIAB_DEV void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
RIAB_DEV void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// bytes must be a multiple of 16; src/dst 16-byte aligned.
RIAB_DEV void tma_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// 4 consecutive floats of a packed array (16-byte vector load)
RIAB_DEV void ldv(float (&d)[4], const float* __restrict__ p) {
  const float4 v = *reinterpret_cast<const float4*>(p);
  d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
}

// Streaming (evict-first) vector stores for the write-once rate rows.
RIAB_DEV void st_cs_f4(float* p, float a, float b, float c, float d) {
  asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
RIAB_DEV void st_cs_f4(float* p, const float (&o)[4]) { st_cs_f4(p, o[0], o[1], o[2], o[3]); }
RIAB_DEV void st_cs_f1(float* p, float a) { asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(p), "f"(a) : "memory"); }

RIAB_DEV float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// NumPy's floating remainder (result takes the sign of the divisor) -- np.mod
RIAB_DEV double np_mod(double x, double m) {
  double r = fmod(x, m);
  if (r != 0.0 && ((r < 0.0) != (m < 0.0))) r += m;
  return r;
}

}  // namespace riab

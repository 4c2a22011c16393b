// Counter-based normal stream of the throughput mode (replaces the reference's global
// np.random.randn stream, SURVEY.md 3.6): Philox4x32-10 (Salmon et al. 2011) + Box-Muller
// evaluated in fp32.  Restated in numpy by oracle/philox.py; tests compare the two.
#pragma once
#include <stdint.h>

namespace ptar {

// The ten round keys (k + i*W) depend only on the seed: computed once per kernel and kept in
// registers / uniform registers so a round is 2 IMAD.WIDE + 2 LOP3.
struct PhiloxKeys {
  uint32_t k0[10], k1[10];
};

__host__ __device__ inline PhiloxKeys philox_keys(uint64_t seed) {
  PhiloxKeys K;
  uint32_t a = static_cast<uint32_t>(seed), b = static_cast<uint32_t>(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    K.k0[i] = a;
    K.k1[i] = b;
    a += 0x9E3779B9u;
    b += 0xBB67AE85u;
  }
  return K;
}

#ifndef PHILOX_ROUNDS
#define PHILOX_ROUNDS 10
#endif
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, const PhiloxKeys& K) {
#pragma unroll
  for (int i = 0; i < PHILOX_ROUNDS; ++i) {
    const uint64_t p0 = static_cast<uint64_t>(0xD2511F53u) * c.x;
    const uint64_t p1 = static_cast<uint64_t>(0xCD9E8D57u) * c.z;
    c = make_uint4(static_cast<uint32_t>(p1 >> 32) ^ c.y ^ K.k0[i], static_cast<uint32_t>(p1),
                   static_cast<uint32_t>(p0 >> 32) ^ c.w ^ K.k1[i], static_cast<uint32_t>(p0));
  }
  return c;
}

// Two standard normals from two 32-bit words.  u1 = (a + 0.5) 2^-32 in (0, 1] (rounded to fp32), angle =
// 2 pi (b + 0.5) 2^-32 - pi in [-pi, pi) -- the range on which MUFU.SIN / MUFU.COS are accurate to 2^-21.4;
// radius^2 = -2 ln2 * log2(u1), with log2 taken of u1 itself (not of a + 0.5): for u1 in [0.5, 1), where the
// radius is small and -2 ln u1 cancels, MUFU.LG2 is then accurate to 2^-22 ABSOLUTE, so |error(z)| ~ 2e-7 / radius
// instead of 3e-6 / radius -- same instruction count.
// PTAR_BM_MODE selects the evaluation (timing variants of bench.py; the shipped library is mode 0):
//   0  fp32 MUFU intrinsics (default; measured against float64 by tests/test_gpu_statistics.py)
//   1  fp32 library accuracy: log2f + sincospif (1-2 ulp)
//   2  float64 log / sincospi, rounded to fp32 at the end (the consumer interface stays float)
#ifndef PTAR_BM_MODE
#define PTAR_BM_MODE 0
#endif
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& n0, float& n1) {
#if PTAR_BM_MODE == 0
  const float u1 = fmaf(static_cast<float>(a), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
  const float r2 = fmaxf(__log2f(u1) * -1.3862943611198906f, 1e-30f);
  const float r = r2 * rsqrtf(r2);
  const float th = fmaf(static_cast<float>(b), 1.4629180792671596e-9f, -3.1415926535897931f);   // + pi 2^-32 is below fp32 resolution
  n0 = r * __cosf(th);
  n1 = r * __sinf(th);
#elif PTAR_BM_MODE == 1
  const float u1 = fmaf(static_cast<float>(a), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
  const float r = sqrtf(fmaxf(log2f(u1) * -1.3862943611198906f, 0.f));
  float s, c;
  sincospif(fmaf(static_cast<float>(b), 4.656612873077393e-10f, -1.0f), &s, &c);
  n0 = r * c;
  n1 = r * s;
#else
  const double u1 = (static_cast<double>(a) + 0.5) * 2.3283064365386963e-10;
  const double r = sqrt(-2.0 * log(u1));
  double s, c;
  sincospi((static_cast<double>(b) + 0.5) * 4.656612873077393e-10 - 1.0, &s, &c);
  n0 = static_cast<float>(r * c);
  n1 = static_cast<float>(r * s);
#endif
}

// 53-bit uniform in [0, 1) from two Philox words: (a >> 5) 2^26 + (b >> 6), times 2^-53 (exact in fp64).
__device__ __forceinline__ double uniform53(uint32_t a, uint32_t b) {
  return static_cast<double>((static_cast<uint64_t>(a >> 5) << 26) | (b >> 6)) * 1.1102230246251565e-16;
}

// Counter layout: c.x = element index (TOA within the pulsar / ECORR bucket / Fourier column /
// grid column), c.y = kind | psr << 8, (c.z, c.w) = global realization id >> 2.  The 4 outputs
// of a counter are the realizations id&~3 .. +3 of that element.
// The continuous-wave population stream (kind 7, ptar_cwpop.cuh) is keyed per realization instead: c.x = source * 16 +
// parameter pair (4 = the pulsar-term phase), c.y = 7 | psr << 8 (psr only for that phase), (c.z, c.w) = the full global
// realization id; its 4 words are two 53-bit uniforms, (w.x >> 5) 2^26 + (w.y >> 6) and (w.z >> 5) 2^26 + (w.w >> 6)
// times 2^-53.  The common-process population stream (kind 8, ptar_cpop.cuh) is keyed the same way: c.x = Fourier bin
// (normals, c.y = 8 | psr << 8) or PTAR_CPOP_HYPER + hyperparameter pair (c.y = 8), (c.z, c.w) = the full realization id.
// The transient population streams (kinds 9 and 10, ptar_tpop.cuh) are keyed as kind 7: c.x = source * 16 + parameter
// pair, c.y = 9 (burst with memory) or 10 (sine-Gaussian burst), (c.z, c.w) = the full realization id.
__device__ __forceinline__ void normals4(float n[4], uint32_t block, uint32_t kind, uint32_t psr,
                                         uint64_t rfield, const PhiloxKeys& K) {
  const uint4 w = philox4x32_10(make_uint4(block, kind | (psr << 8), static_cast<uint32_t>(rfield),
                                           static_cast<uint32_t>(rfield >> 32)), K);
  box_muller(w.x, w.y, n[0], n[1]);
  box_muller(w.z, w.w, n[2], n[3]);
}

}  // namespace ptar

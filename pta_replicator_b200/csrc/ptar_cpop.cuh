// Per-realization common-process populations (ptar_common_population): every realization gets its own common process,
// its spectrum drawn on the device from the priors of a ptar_cpop_model, injected in the statistics' own Fourier basis
// F_a = (sin, cos)(2 pi f_k t) so that every grid likelihood is the exact likelihood of the injection.
//
// cpop_draw_kernel  one CTA per (realization, bin k).  Thread 0 draws the hyperparameters from the Philox stream
//                   PTAR_K_CPOP (counter layout in ptar.h) and forms sqrt(phi_k); every thread makes the fp64
//                   Box-Muller normals z[b][2k], z[b][2k + 1] of its pulsars into shared memory; then each thread mixes
//                   its pulsars a: c[r][a][2k + s] = sqrt(phi_k) sum_b B_ab z[b][2k + s], b in index order, unfused, so
//                   that tests/cpop_oracle.py restates it operation by operation.
// cpop_add_kernel   rows[r][i] += sum_j c[r][p(i)][j] F_j(t_i) over the packed TOA axis: a CTA covers CPOP_TOAS slots x
//                   CPOP_RB realizations; a thread evaluates its slot's 2K basis values once (argument (2 pi t) f_k, as
//                   engine._sincos_basis rounds it) and keeps them in registers, and walks the realizations with the
//                   coefficient records of the CTA's pulsars staged in shared memory, so each row element is one
//                   coalesced read-modify-write.  Alignment slots (psr < 0) are never touched.
#pragma once
#include <limits.h>
#include <stdint.h>

#include "ptar_cwpop.cuh"
#include "ptar_rng.cuh"

namespace ptar {

constexpr uint32_t K_CPOP = 8;
constexpr int CPOP_DRAW_THREADS = 128;   // threads per (realization, bin) CTA of the draw kernel
constexpr int CPOP_TOAS = 128;           // TOA slots per CTA of the add kernel (one per thread)
constexpr int CPOP_RB = 32;              // realizations per CTA of the add kernel
constexpr int CPOP_UNROLL = 4;           // row elements loaded before their sums are added back
// The CTA's slots span at most CPOP_TOAS / PTAR_TOA_ALIGN pulsars (every segment starts at a multiple of the
// alignment), so one realization's records always fit the stage: 16 KB.
constexpr int CPOP_STAGE = CPOP_TOAS / PTAR_TOA_ALIGN * 2 * PTAR_CPOP_MAX_K;

__device__ __forceinline__ uint4 cpop_words(uint32_t elem, uint32_t psr, uint64_t r, const PhiloxKeys& K) {
  return philox4x32_10(make_uint4(elem, K_CPOP | (psr << 8), static_cast<uint32_t>(r), static_cast<uint32_t>(r >> 32)), K);
}

// Hyperparameter j of realization r (pair j / 2, word pair j & 1) under the prior (kind, lo, width) of slot `s`.
__device__ __forceinline__ double cpop_hyper(const ptar_cpop_model& m, int j, int s, uint64_t r, const PhiloxKeys& K) {
  const uint4 w = cpop_words(PTAR_CPOP_HYPER + j / 2, 0, r, K);
  const double u = (j & 1) ? uniform53(w.z, w.w) : uniform53(w.x, w.y);
  return cwpop_param(m.kind[s], m.lo[s], m.width[s], u);
}

__global__ void __launch_bounds__(CPOP_DRAW_THREADS) cpop_draw_kernel(double* __restrict__ c, double* __restrict__ params,
                                                                       ptar_cpop_model m, int64_t real0, uint64_t seed) {
  extern __shared__ double zs[];   // [n_psr][2]: the normals of this bin
  __shared__ double amp;
  const int k = static_cast<int>(blockIdx.x % m.K);
  const int64_t r = blockIdx.x / m.K;
  const uint64_t rg = static_cast<uint64_t>(real0 + r);
  const PhiloxKeys K = philox_keys(seed);
  const int P = m.n_psr, K2 = 2 * m.K;
  if (threadIdx.x == 0) {
    double a;
    if (m.spectrum == PTAR_CPOP_POWERLAW) {
      const double log10_A = cpop_hyper(m, 0, 0, rg, K), gamma = cpop_hyper(m, 1, 1, rg, K);
      const double A = exp10(log10_A);
      const double pt = __dmul_rn(__ddiv_rn(pow(m.pl_x[k], -gamma), m.pl_den), m.pl_y3);   // _powerlaw_prior
      a = sqrt(__dmul_rn(__dmul_rn(A, A), pt));
      if (params && k == 0) {
        params[2 * r] = log10_A;
        params[2 * r + 1] = gamma;
      }
    } else {
      const double log10_rho = cpop_hyper(m, k, 0, rg, K);
      a = exp10(log10_rho);
      if (params) params[r * m.K + k] = log10_rho;
    }
    amp = a;
  }
  for (int b = threadIdx.x; b < P; b += CPOP_DRAW_THREADS) {
    const uint4 w = cpop_words(static_cast<uint32_t>(k), static_cast<uint32_t>(b), rg, K);
    const double u1 = uniform53(w.x, w.y), u2 = uniform53(w.z, w.w);
    const double rho = sqrt(__dmul_rn(-2.0, log(__dsub_rn(1.0, u1))));   // 1 - u1 in (0, 1], exact
    double s, co;
    sincos(__dmul_rn(6.283185307179586, u2), &s, &co);
    zs[2 * b] = __dmul_rn(rho, co);
    zs[2 * b + 1] = __dmul_rn(rho, s);
  }
  __syncthreads();
  const double a = amp;
  for (int p = threadIdx.x; p < P; p += CPOP_DRAW_THREADS) {
    double c0 = zs[2 * p], c1 = zs[2 * p + 1];
    if (m.Bt) {
      c0 = c1 = 0.0;
      for (int b = 0; b < P; ++b) {
        const double bb = __ldg(m.Bt + int64_t(b) * P + p);   // B_pb: consecutive threads read consecutive doubles
        c0 = __dadd_rn(c0, __dmul_rn(bb, zs[2 * b]));
        c1 = __dadd_rn(c1, __dmul_rn(bb, zs[2 * b + 1]));
      }
    }
    double* o = c + (r * P + p) * K2 + 2 * k;
    o[0] = __dmul_rn(a, c0);
    o[1] = __dmul_rn(a, c1);
  }
}

// KMAX: the bins held in registers (K <= KMAX); the loops run to KMAX, predicated on k < K, so F stays in registers.
template <int KMAX>
__global__ void __launch_bounds__(CPOP_TOAS) cpop_add_kernel(double* __restrict__ rows, int64_t ld, int32_t nreal,
                                                             const double* __restrict__ c,
                                                             const double* __restrict__ freqs,
                                                             const double* __restrict__ slot_t,
                                                             const int32_t* __restrict__ slot_psr, int n_psr, int K) {
  __shared__ __align__(16) double sq[CPOP_STAGE];
  __shared__ int prange[2];
  const int64_t i = int64_t(blockIdx.x) * CPOP_TOAS + threadIdx.x;
  const int p = i < ld ? slot_psr[i] : -1;
  if (threadIdx.x == 0) prange[0] = INT_MAX, prange[1] = -1;
  __syncthreads();
  if (p >= 0) {
    atomicMin(prange, p);
    atomicMax(prange + 1, p);
  }
  __syncthreads();
  const int p_lo = prange[0], p_hi = prange[1];
  if (p_hi < 0) return;   // alignment slots only: the whole CTA leaves
  double F[2 * KMAX];
  const double tw = p >= 0 ? __dmul_rn(6.283185307179586, slot_t[i]) : 0.0;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    F[2 * k] = F[2 * k + 1] = 0.0;
    if (k < K) sincos(__dmul_rn(tw, __ldg(freqs + k)), &F[2 * k], &F[2 * k + 1]);
  }
  const int K2 = 2 * K;
  const int rec = (p_hi - p_lo + 1) * K2;   // doubles of one realization's records (<= CPOP_STAGE)
  const int per_stage = CPOP_STAGE / rec;
  const int off = (p - p_lo) * K2;
  const int64_t rstride = int64_t(n_psr) * K2;
  const double* q0 = c + int64_t(p_lo) * K2;
  const int r_begin = blockIdx.y * CPOP_RB;
  const int r_end = min(nreal, r_begin + CPOP_RB);
  for (int r0 = r_begin; r0 < r_end; r0 += per_stage) {
    const int cnt = min(per_stage, r_end - r0);
    __syncthreads();
    for (int e = threadIdx.x; e < cnt * rec; e += CPOP_TOAS) {
      const int j = e / rec;
      sq[e] = q0[(r0 + j) * rstride + (e - j * rec)];
    }
    __syncthreads();
    if (p < 0) continue;
    for (int j = 0; j < cnt; j += CPOP_UNROLL) {
      double v[CPOP_UNROLL];
#pragma unroll
      for (int u = 0; u < CPOP_UNROLL; ++u)
        if (j + u < cnt) v[u] = rows[int64_t(r0 + j + u) * ld + i];
#pragma unroll
      for (int u = 0; u < CPOP_UNROLL; ++u) {
        if (j + u >= cnt) break;
        const double* q = sq + (j + u) * rec + off;
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
          if (k < K) {
            const double2 cc = *reinterpret_cast<const double2*>(q + 2 * k);
            acc = fma(cc.x, F[2 * k], acc);
            acc = fma(cc.y, F[2 * k + 1], acc);
          }
        }
        rows[int64_t(r0 + j + u) * ld + i] = v[u] + acc;
      }
    }
  }
}

}  // namespace ptar

// Per-frequency optimal statistic (ptar_os_pf): per realization and GW frequency k, the pair correlations of the
// (sin, cos) columns 2k, 2k+1 of the per-pulsar projections X that os_sum wrote, and their template sums.
//
// Per realization r, frequency k = 0..K-1 (K = nc / 2), pair q = (a < b) of os.pairs and template o, with X unscaled:
//   d_qk = X_a,2k X_b,2k + X_a,2k+1 X_b,2k+1;  rho[r][k][q] = d_qk / t[k][q];  b_ok = sum_q Gamma^o_q d_qk
//   phi[r][o][k] = b_ok / dnorm[o][k];  snr[r][o][k] = b_ok / dsqrt[o][k];  phi_mc[r][o][k] = sum_o' finv[k][o][o'] b_o'k
// One CTA per realization.  X[r] is staged transposed, xs[j][p], so that the lanes of a warp, which walk consecutive
// pairs (a fixed, b consecutive), read consecutive doubles.  Warp w takes the frequencies k = w and w + 8 in one pass
// over the pairs (the template weights are read once for both); lane l takes the pairs q = l, l + 32, ...; the lane
// sums are added by a fixed xor-shuffle tree.  Every sum runs in an order fixed by q and k only, so outputs are
// bit-identical whatever nreal, chunking or real0.  No atomics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ptar.h"

namespace ptar {

constexpr int PF_THREADS = 256;
constexpr int PF_WARPS = PF_THREADS / 32;
static_assert(PTAR_OS_MAX_NC / 2 <= 2 * PF_WARPS, "every frequency is one of the two of some warp");

// phi, snr and phi_mc of realization r at frequency k from the template sums b[o] = b_ok.
__device__ __forceinline__ void os_pf_write(int64_t r, int k, int K, int no, const double (&b)[PTAR_OS_MAX_ORF],
                                            const ptar_os_pf_model& pf, double* phi, double* snr, double* phi_mc) {
  const double* fk = pf.finv + int64_t(k) * no * no;
#pragma unroll
  for (int o = 0; o < PTAR_OS_MAX_ORF; ++o)
    if (o < no) {
      const int64_t out = (r * no + o) * K + k;
      phi[out] = __ddiv_rn(b[o], pf.dnorm[o * K + k]);
      snr[out] = __ddiv_rn(b[o], pf.dsqrt[o * K + k]);
      double m = 0.0;
#pragma unroll
      for (int o2 = 0; o2 < PTAR_OS_MAX_ORF; ++o2)
        if (o2 < no) m = fma(fk[o * no + o2], b[o2], m);
      phi_mc[out] = m;
    }
}

__global__ void __launch_bounds__(PF_THREADS) os_pf_kernel(const double* __restrict__ X, ptar_os_model os,
                                                           ptar_os_pf_model pf, double* __restrict__ rho,
                                                           double* __restrict__ phi, double* __restrict__ snr,
                                                           double* __restrict__ phi_mc) {
  extern __shared__ __align__(16) double os_pf_smem[];
  const int P = os.n_psr, ncp = os.ncp, nc = os.nc, K = nc >> 1, no = os.n_orf, npr = os.n_pairs;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r = blockIdx.x;
  double* xs = os_pf_smem;   // [nc][P]
  const double* xr = X + r * P * ncp;
  for (int e = tid; e < P * ncp; e += PF_THREADS) {
    const int p = e / ncp, j = e - p * ncp;
    if (j < nc) xs[j * P + p] = xr[e];
  }
  __syncthreads();
  const int k0 = warp, k1 = warp + PF_WARPS;
  if (k0 >= K) return;
  const bool two = k1 < K;   // warp-uniform
  const double* s0 = xs + 2 * k0 * P;
  const double* c0 = s0 + P;
  const double* s1 = xs + 2 * (two ? k1 : k0) * P;
  const double* c1 = s1 + P;
  double b0[PTAR_OS_MAX_ORF] = {0.0, 0.0, 0.0, 0.0}, b1[PTAR_OS_MAX_ORF] = {0.0, 0.0, 0.0, 0.0};
  for (int q = lane; q < npr; q += 32) {
    const int a = os.pairs[2 * q], b = os.pairs[2 * q + 1];
    const double d0 = fma(c0[a], c0[b], __dmul_rn(s0[a], s0[b]));
    const double d1 = two ? fma(c1[a], c1[b], __dmul_rn(s1[a], s1[b])) : 0.0;
    if (rho) {
      rho[(r * K + k0) * npr + q] = __ddiv_rn(d0, pf.t[int64_t(k0) * npr + q]);
      if (two) rho[(r * K + k1) * npr + q] = __ddiv_rn(d1, pf.t[int64_t(k1) * npr + q]);
    }
#pragma unroll
    for (int o = 0; o < PTAR_OS_MAX_ORF; ++o)
      if (o < no) {
        const double g = os.orf[int64_t(o) * npr + q];
        b0[o] = fma(g, d0, b0[o]);
        b1[o] = fma(g, d1, b1[o]);
      }
  }
  // butterfly: lanes i and i ^ m add the same two values, so every lane ends with the same sum in the same order
#pragma unroll
  for (int m = 16; m > 0; m >>= 1)
#pragma unroll
    for (int o = 0; o < PTAR_OS_MAX_ORF; ++o)
      if (o < no) {
        b0[o] = __dadd_rn(b0[o], __shfl_xor_sync(0xffffffffu, b0[o], m));
        if (two) b1[o] = __dadd_rn(b1[o], __shfl_xor_sync(0xffffffffu, b1[o], m));
      }
  if (lane != 0) return;
  os_pf_write(r, k0, K, no, b0, pf, phi, snr, phi_mc);
  if (two) os_pf_write(r, k1, K, no, b1, pf, phi, snr, phi_mc);
}

}  // namespace ptar

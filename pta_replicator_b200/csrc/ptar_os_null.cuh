// Null distributions of the optimal statistic (ptar_os_null): phase shifts and sky scrambles of one template,
// evaluated for every realization from the per-pulsar projections X that os_sum wrote.
//
// The null set is realization-independent (engine.PulsarBatch._plan_os_null), so both methods are one GEMM:
//   S/N[r][s] = (U[r] . V[:, s]) / sqrt(D_s),   s = 0..n (column 0 = the unshifted, unscrambled template)
//   phase shift   U[r][(q, k, 0)] = x_a,2k x_b,2k + x_a,2k+1 x_b,2k+1      V = Gamma_q cos(phi_s,a,k - phi_s,b,k)
//                 U[r][(q, k, 1)] = x_a,2k+1 x_b,2k - x_a,2k x_b,2k+1      V = Gamma_q sin(phi_s,a,k - phi_s,b,k)
//   sky scramble  U[r][q] = x_a . x_b                                        V = Gamma^s_q
// with x = X phi~^{1/2} and q = (a < b) in the order of os.pairs.
//
// os_null_prepare  one CTA per realization (x in shared memory, as os_pairs): writes U[r][0..kdp), zero past kd.
// os_null_gemm     64 x 64 output tiles on DMMA (mma.sync.m8n8k4.f64).  U rows and V^T rows (both kd-major) are staged
//                  32 kd at a time by bulk-async copies into a 3-stage mbarrier ring (the os_project idiom, row pitch
//                  36 doubles: conflict-free fragment gathers).  Warp w owns the 32 x 32 quarter (w & 1, (w >> 1) & 1)
//                  and the k-half w >> 2 of every 32-kd chunk; the two k-halves are added in a fixed order at the end.
//                  Every output is therefore summed in an order fixed by kd alone -- not by its r- or s-block, so
//                  results do not depend on nreal, chunking or real0.  No split-K across CTAs, no atomics.
// os_null_count    one CTA per realization: #{s >= 1 : not S/N_s < S/N_0} (integer, order-free; a NaN null column
//                  counts) and the p-value (NaN when S/N_0 is NaN).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_os.cuh"

namespace ptar {

constexpr int NL_THREADS = 256;
constexpr int NL_BM = 64;                                 // realizations per CTA
constexpr int NL_BN = 64;                                 // columns per CTA
constexpr int NL_BK = 32;                                 // kd per stage (256-byte bulk copies)
constexpr int NL_P = NL_BK + 4;                           // smem row pitch (doubles): conflict-free fragment gathers
constexpr int NL_STAGES = 3;
constexpr int NL_STAGE_DOUBLES = (NL_BM + NL_BN) * NL_P;  // 36,864 B per stage
constexpr size_t NL_SMEM = sizeof(double) * NL_STAGES * NL_STAGE_DOUBLES + 64;   // + barriers: 2 CTAs per SM
static_assert(2 * NL_BM * NL_BN <= NL_STAGES * NL_STAGE_DOUBLES, "k-half reduction must fit in the ring");

__global__ void __launch_bounds__(NL_THREADS) os_null_prepare_kernel(const double* __restrict__ X, ptar_os_model os,
                                                                     ptar_os_null_model nl, double* __restrict__ U) {
  extern __shared__ __align__(16) double nl_prep_smem[];
  const int P = os.n_psr, ncp = os.ncp, nc = os.nc, K = os.nc / 2, tid = threadIdx.x;
  double* xs = nl_prep_smem;   // [P][ncp]
  const int64_t r = blockIdx.x;
  const double* xr = X + r * P * ncp;
  for (int e = tid; e < P * ncp; e += NL_THREADS) xs[e] = __dmul_rn(xr[e], os.sqrt_phi[e % ncp]);
  __syncthreads();
  double* ur = U + r * nl.kdp;
  if (nl.method == PTAR_OS_NULL_PHASE_SHIFT) {
    const int64_t ne = int64_t(os.n_pairs) * K;
    for (int64_t e = tid; e < ne; e += NL_THREADS) {
      const int q = static_cast<int>(e / K), k = static_cast<int>(e % K);
      const double* xa = xs + os.pairs[2 * q] * ncp + 2 * k;
      const double* xb = xs + os.pairs[2 * q + 1] * ncp + 2 * k;
      double2 v;
      v.x = __fma_rn(xa[0], xb[0], __dmul_rn(xa[1], xb[1]));
      v.y = __fma_rn(xa[1], xb[0], -__dmul_rn(xa[0], xb[1]));
      reinterpret_cast<double2*>(ur)[e] = v;
    }
  } else {
    for (int q = tid; q < os.n_pairs; q += NL_THREADS) {
      const double* xa = xs + os.pairs[2 * q] * ncp;
      const double* xb = xs + os.pairs[2 * q + 1] * ncp;
      double d = 0.0;
      for (int j = 0; j < nc; ++j) d = fma(xa[j], xb[j], d);
      ur[q] = d;
    }
  }
  for (int64_t e = nl.kd + tid; e < nl.kdp; e += NL_THREADS) ur[e] = 0.0;
}

// Warp 0 fills stage `st` with kd chunk `c`: U rows r0 .. r0 + nrow - 1, then V^T rows s0 .. s0 + 63.
__device__ __forceinline__ void os_null_issue(double* st, uint64_t* bar, const double* Ub, const double* Vb, int64_t kdp,
                                              int c, int nrow, int lane) {
  constexpr uint32_t bytes = NL_BK * 8u;
  if (lane == 0) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(os_smem_u32(bar)), "r"(bytes * (nrow + NL_BN))
                 : "memory");
  }
  __syncwarp();
  const int64_t k0 = int64_t(c) * NL_BK;
  for (int m = lane; m < nrow + NL_BN; m += 32) {
    const double* src = m < nrow ? Ub + int64_t(m) * kdp + k0 : Vb + int64_t(m - nrow) * kdp + k0;
    const int row = m < nrow ? m : NL_BM + (m - nrow);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     os_smem_u32(st + row * NL_P)),
                 "l"(src), "r"(bytes), "r"(os_smem_u32(bar))
                 : "memory");
  }
}

__global__ void __launch_bounds__(NL_THREADS, 2) os_null_gemm_kernel(const double* __restrict__ U, int nreal,
                                                                     ptar_os_null_model nl, double* __restrict__ snr) {
  extern __shared__ __align__(16) double nl_smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(nl_smem + NL_STAGES * NL_STAGE_DOUBLES);
  const int s0 = blockIdx.x * NL_BN, r0 = blockIdx.y * NL_BM;
  const int nrow = min(NL_BM, nreal - r0);
  const int nch = static_cast<int>(nl.kdp / NL_BK);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double* Ub = U + int64_t(r0) * nl.kdp;
  const double* Vb = nl.V + int64_t(s0) * nl.kdp;
  if (tid == 0) {
    for (int s = 0; s < NL_STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(os_smem_u32(bars + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == 0)
    for (int c = 0; c < NL_STAGES && c < nch; ++c) os_null_issue(nl_smem + c * NL_STAGE_DOUBLES, bars + c, Ub, Vb, nl.kdp, c, nrow, lane);

  const int wm = warp & 1, wn = (warp >> 1) & 1, kh = warp >> 2;
  const int fr = lane >> 2, fk = lane & 3;
  double acc[4][4][2];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b][0] = acc[a][b][1] = 0.0;

  for (int c = 0; c < nch; ++c) {
    const int s = c % NL_STAGES;
    const double* As = nl_smem + s * NL_STAGE_DOUBLES;
    const double* Bs = As + NL_BM * NL_P;
    os_mbar_wait(bars + s, (c / NL_STAGES) & 1);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int kk = kh * 16 + q * 4 + fk;
      double af[4], bf[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) af[t] = As[(wm * 32 + t * 8 + fr) * NL_P + kk];
#pragma unroll
      for (int t = 0; t < 4; ++t) bf[t] = Bs[(wn * 32 + t * 8 + fr) * NL_P + kk];
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) PTAR_OS_DMMA(acc[mt][nt][0], acc[mt][nt][1], af[mt], bf[nt]);
    }
    __syncthreads();   // every warp is done with stage s
    if (warp == 0 && c + NL_STAGES < nch)
      os_null_issue(nl_smem + s * NL_STAGE_DOUBLES, bars + s, Ub, Vb, nl.kdp, c + NL_STAGES, nrow, lane);
  }
  // k-halves in a fixed order: red[kh][m][n] (reuses the ring; every copy has landed and been consumed)
  double* red = nl_smem;
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      double* d = red + (kh * NL_BM + wm * 32 + mt * 8 + fr) * NL_BN + wn * 32 + nt * 8 + 2 * fk;
      d[0] = acc[mt][nt][0];
      d[1] = acc[mt][nt][1];
    }
  __syncthreads();
  const int ncol = min(NL_BN, nl.n_col - s0);
  for (int e = tid; e < nrow * NL_BN; e += NL_THREADS) {
    const int m = e / NL_BN, n = e % NL_BN;
    if (n < ncol) {
      const double v = __dadd_rn(red[m * NL_BN + n], red[(NL_BM + m) * NL_BN + n]);
      snr[int64_t(r0 + m) * nl.n_col + s0 + n] = __ddiv_rn(v, nl.dsqrt[s0 + n]);
    }
  }
}

__global__ void __launch_bounds__(NL_THREADS) os_null_count_kernel(const double* __restrict__ snr, int n_col,
                                                                   int64_t* __restrict__ exceed, double* __restrict__ fap) {
  __shared__ int cnt[NL_THREADS];
  const int64_t r = blockIdx.x;
  const double* row = snr + r * n_col;
  const double s0 = row[0];
  int c = 0;
  // a NaN null column counts as an exceedance (the conservative side): !(a < b) is a >= b for numbers, true for NaN
  for (int s = 1 + threadIdx.x; s < n_col; s += NL_THREADS) c += !(row[s] < s0);
  cnt[threadIdx.x] = c;
  __syncthreads();
  for (int h = NL_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) cnt[threadIdx.x] += cnt[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    exceed[r] = cnt[0];
    // the p-value of a NaN observed S/N is NaN, not the 1 / n_col that zero exceedances would report
    fap[r] = s0 != s0 ? s0 : __ddiv_rn(1.0 + cnt[0], static_cast<double>(n_col));
  }
}

}  // namespace ptar

// Hellings-Downs (ORF-correlated) common-process likelihood (ptar_hd_grid): per realization, the log-likelihood ratio
// of a power law in (A, gamma) whose cross-pulsar covariance is Gamma_ab phi~(gamma) against the noise-only model, on
// the grid of the CURN likelihood, from the X[r][a] = C_a^T r_a of ptar_os_project.  The summaries are
// ptar_curn_reduce's, run on this map.
//
// The noise-model work is realization-independent and done once on the host (engine.PulsarBatch._plan_hd): with
// Gamma = B B^T and G = B (x) phi~^{1/2}, per grid gamma the eigendecomposition G^T Z G = U diag(lambda) U^T of size
// N = n_psr nc (Z = blockdiag(Z_a)), V(gamma) = U^T G^T and ldet(A, gamma) = sum_j log1p(A^2 lambda_j).  Per realization:
//   hd_grid  y = V(gamma) X  (X stacked over the pulsars);  w_j(A) = A^2 / (1 + A^2 lambda_j);
//            Q(A, gamma) = sum_j w_j(A) y_j^2;  lnL = 1/2 Q - 1/2 ldet             fused two-GEMM chain on DMMA
//
// grid = (realization blocks of 64, gamma), realization block fastest, so the CTAs of one gamma run together and
// V(gamma) crosses HBM about once.  A CTA walks every block of 32 eigen-rows j in index order.  Per j-block it runs a
// k-loop over the stacked X axis (n_psr ncp columns) in chunks of 64: warp 0 stages X [64 x 64] and V [32 x 64] through
// an mbarrier ring (os_issue_chunk, two arrivals per stage; the ring runs on across j-blocks) and warp w accumulates
// the Y tile of rows 16 (w & 3) .. +15 and eigen-rows 16 (w >> 2) .. +15 on DMMA.  The squared Y tile goes to shared
// memory next to the W tile [32 x NAp] that every thread formed before the k-loop, and warp w adds Y^2 W to its Q of
// rows 16 (w & 3) .. +15 and amplitudes NAp / 2 (w >> 2) .. +NAp / 2, held in registers across j-blocks.  A row's Q
// depends on its own X row, the statics and the fixed j and k orders only -- not on the realization block, nreal,
// chunking or real0.  No partial sums, no atomics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_os.cuh"

namespace ptar {

constexpr int HD_THREADS = 256;
constexpr int HD_RB = 64;                                     // realizations per CTA (4 warp rows of 16)
constexpr int HD_JB = PTAR_HD_JB;                             // eigen-rows per j-block (2 warp columns of 16)
constexpr int HD_KC = OS_KC;                                  // stacked X columns per chunk (os_issue_chunk's pitch)
constexpr int HD_STAGE_DOUBLES = (HD_RB + HD_JB) * OS_XP;     // X rows then V rows: 52,224 B
constexpr int HD_YP = HD_JB + 4;                              // Y^2 pitch: rows 32 B apart -> conflict-free A gathers
// QN = n-tiles of 8 amplitudes per warp: NAp = 16 QN amplitudes per CTA (64, 128 or 256)
__host__ __device__ constexpr int hd_stages(int QN) { return QN > 8 ? 2 : 3; }
__host__ __device__ constexpr int hd_wp(int QN) { return 16 * QN + 8; }   // W pitch: k rows 64 B apart
__host__ __device__ constexpr size_t hd_smem(int QN) {
  return sizeof(double) * (size_t(hd_stages(QN)) * HD_STAGE_DOUBLES + HD_RB * HD_YP + HD_JB * hd_wp(QN)) + 32;
}   // QN = 4: 177,952 B;  8: 209,952 B;  16: 190,496 B (+ barriers)

template <int QN>
__global__ void __launch_bounds__(HD_THREADS, 1) hd_grid_kernel(const double* __restrict__ X, int nreal,
                                                               ptar_hd_model hm, double* __restrict__ lnL) {
  extern __shared__ __align__(16) double hd_smem_buf[];
  constexpr int S = hd_stages(QN), WP = hd_wp(QN), NAP = 16 * QN;
  double* ys = hd_smem_buf + S * HD_STAGE_DOUBLES;
  double* ws = ys + HD_RB * HD_YP;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ws + HD_JB * WP);
  const int rb0 = blockIdx.x * HD_RB, g = blockIdx.y;
  const int nrow = min(HD_RB, nreal - rb0);
  const int NA = hm.n_amp, NG = hm.n_gamma;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  const int mg = warp & 3, ng = warp >> 2;
  const int64_t kx = int64_t(hm.n_psr) * hm.ncp;                 // stacked X axis = row pitch of X and V
  const int nkc = static_cast<int>((kx + HD_KC - 1) / HD_KC);
  const int njb = hm.np / HD_JB;
  const int total = njb * nkc;
  const double* xblk = X + int64_t(rb0) * kx;
  const double* vg = hm.V + int64_t(g) * hm.np * kx;
  const double* lam = hm.lam + int64_t(g) * hm.np;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 2;" ::"r"(os_smem_u32(bars + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int c) {   // warp 0: chunk c = (j-block c / nkc, column chunk c % nkc)
    double* st = hd_smem_buf + (c % S) * HD_STAGE_DOUBLES;
    uint64_t* bar = bars + c % S;
    const int jb = c / nkc;
    const int64_t base = int64_t(c % nkc) * HD_KC;
    const int cnt = static_cast<int>(min(int64_t(HD_KC), kx - base));
    os_issue_chunk(st, bar, xblk, kx, base, nrow, cnt, lane);
    os_issue_chunk(st + HD_RB * OS_XP, bar, vg + int64_t(jb) * HD_JB * kx, kx, base, HD_JB, cnt, lane);
  };
  if (warp == 0)
    for (int c = 0; c < S && c < total; ++c) issue(c);

  double q[2][QN][2];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int t = 0; t < QN; ++t) q[m][t][0] = q[m][t][1] = 0.0;
  int c = 0;
  for (int jb = 0; jb < njb; ++jb) {
    // w_j(A) = A^2 / (1 + A^2 lambda_j), the IEEE expression of the host statics (no contraction); 0 past n_amp
    for (int e = tid; e < HD_JB * NAP; e += HD_THREADS) {
      const int j = e / NAP, n = e % NAP;
      const double a2 = n < NA ? __ldg(hm.a2 + n) : 0.0;
      ws[j * WP + n] = __ddiv_rn(a2, __dadd_rn(1.0, __dmul_rn(a2, __ldg(lam + jb * HD_JB + j))));
    }
    double y[2][2][2];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int t = 0; t < 2; ++t) y[m][t][0] = y[m][t][1] = 0.0;
    for (int kc = 0; kc < nkc; ++kc, ++c) {
      const int s = c % S;
      const double* xs = hd_smem_buf + s * HD_STAGE_DOUBLES;
      const double* vs = xs + HD_RB * OS_XP;
      const int cnt = static_cast<int>(min(int64_t(HD_KC), kx - int64_t(kc) * HD_KC));   // a multiple of 8
      os_mbar_wait(bars + s, (c / S) & 1);
#pragma unroll 4
      for (int kk = 0; kk < cnt; kk += 4) {
        double af[2], bf[2];
#pragma unroll
        for (int m = 0; m < 2; ++m) af[m] = xs[(mg * 16 + m * 8 + fr) * OS_XP + kk + fk];
#pragma unroll
        for (int t = 0; t < 2; ++t) bf[t] = vs[(ng * 16 + t * 8 + fr) * OS_XP + kk + fk];
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int t = 0; t < 2; ++t) PTAR_OS_DMMA(y[m][t][0], y[m][t][1], af[m], bf[t]);
      }
      __syncthreads();   // every warp is done with stage s (and, at kc = 0, W is complete)
      if (warp == 0 && c + S < total) issue(c + S);
    }
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        double* yr = ys + (mg * 16 + m * 8 + fr) * HD_YP + ng * 16 + t * 8 + 2 * fk;
        yr[0] = __dmul_rn(y[m][t][0], y[m][t][0]);
        yr[1] = __dmul_rn(y[m][t][1], y[m][t][1]);
      }
    __syncthreads();   // Y^2 complete
#pragma unroll
    for (int kk = 0; kk < HD_JB; kk += 4) {
      double af[2];
#pragma unroll
      for (int m = 0; m < 2; ++m) af[m] = ys[(mg * 16 + m * 8 + fr) * HD_YP + kk + fk];
#pragma unroll
      for (int t = 0; t < QN; ++t) {
        const double bf = ws[(kk + fk) * WP + ng * (NAP / 2) + t * 8 + fr];
#pragma unroll
        for (int m = 0; m < 2; ++m) PTAR_OS_DMMA(q[m][t][0], q[m][t][1], af[m], bf);
      }
    }
    __syncthreads();   // Y^2 and W are free
  }
  const double* ld = hm.ldet + int64_t(g) * NA;
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    const int r = mg * 16 + m * 8 + fr;
    if (r >= nrow) continue;
    double* out = lnL + (int64_t(rb0 + r) * NG + g) * NA;
#pragma unroll
    for (int t = 0; t < QN; ++t)
#pragma unroll
      for (int cc = 0; cc < 2; ++cc) {
        const int k = ng * (NAP / 2) + t * 8 + 2 * fk + cc;
        if (k < NA) out[k] = __dmul_rn(0.5, __dsub_rn(q[m][t][cc], __ldg(ld + k)));
      }
  }
}

}  // namespace ptar

// Factorised free-spectrum likelihood (ptar_fs_grid): per realization and GW frequency bin k, the log-likelihood ratio
// of a common process in bin k alone, phi_k = rho^2 per Fourier coefficient, against the noise-only model, on a grid in
// log10 rho, from the X[r][a] = C_a^T r_a of ptar_os_project.  The summaries are ptar_curn_reduce's, one map per
// (realization, bin).
//
// The noise-model work is realization-independent and done once on the host (engine.PulsarBatch._plan_fs): per bin k
// the stacked eigendecomposition G^T Z[k] G = U diag(lambda) U^T of size n = 2 n_psr (Z[k] = blockdiag_a Z_a[k], G = I
// for the uncorrelated model, B (x) I_2 with Gamma = B B^T for an ORF), V_k = U^T G^T on the gathered axis (pulsar a,
// column i of bin k) and ldet[k][i] = sum_j log1p(rho_i^2 lambda_j).  Per realization:
//   fs_grid  y = V_k X_k  (X_k[2a + i] = X[r][a][2k + i]);  w_j(rho) = rho^2 / (1 + rho^2 lambda_j);
//            lnL[r][k][i] = 1/2 sum_j w_j(rho_i) y_j^2 - 1/2 ldet[k][i]             fused two-GEMM chain on DMMA
//
// grid = (amplitude blocks of 64, realization blocks of 64, bins), amplitude block fastest.  A CTA walks the blocks of
// 32 eigen-rows j in index order.  Per j-block it runs a k-loop over the gathered axis (n2p = 2 n_psr rounded up to 8
// columns) in chunks of 64 = 32 pulsars x 2: every thread gathers the bin-k column pairs of the chunk's pulsars from X's
// [n_psr][ncp] rows (one 16-byte load per realization and pulsar, zero past n_psr) while warp 0's bulk-async copy of the
// V_k chunk [32 x 64] lands through a 2-stage mbarrier ring that runs on across j-blocks.  Warp w owns the realization
// rows 8w .. 8w + 7: Y = X_k V_k^T (M = 8, N = 32) accumulates over the chunks, then Y^2 goes to its own shared rows and
// Q += Y^2 W (M = 8, N = 64, K = 32) in registers across j-blocks, with ptar_curn.cuh's W tile, Q step and store.  So
// the GEMM depth is 2 n_psr, not n_psr ncp.  A row's Q depends on its own X row, the statics and the fixed j and column
// orders only -- not on the realization block, nreal, chunking or real0.  No atomics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_curn.cuh"
#include "ptar_os.cuh"

namespace ptar {

constexpr int FS_THREADS = CURN_THREADS;                    // the CTA shape of the body shared with curn_grid_kernel
constexpr int FS_RB = CURN_RB;                              // realizations per CTA (one m-tile of 8 per warp)
constexpr int FS_AB = CURN_AB;                              // amplitudes per CTA (8 n-tiles)
constexpr int FS_JB = PTAR_FS_JB;                           // eigen-rows per j-block (4 n-tiles)
constexpr int FS_KC = OS_KC;                                // gathered columns per chunk: 32 pulsars x 2
constexpr int FS_STAGES = 2;
constexpr int FS_STAGE_DOUBLES = (FS_RB + FS_JB) * OS_XP;   // gathered X rows then V rows, pitch OS_XP: 52,224 B
constexpr int FS_YP = FS_JB + 4;                            // Y^2 pitch: rows 32 B apart -> conflict-free A gathers
constexpr size_t FS_SMEM = sizeof(double) * (FS_STAGES * FS_STAGE_DOUBLES + FS_RB * FS_YP + FS_JB * CURN_WP) + 16;
// = 141,328 B (+ 2 barriers)

// Warp 0: chunk c = (j-block c / nkc, column chunk c % nkc) of V_k into stage c % FS_STAGES of the ring
__device__ __forceinline__ void fs_issue_v(double* smem, uint64_t* bars, const double* vk, int n2p, int nkc, int c,
                                           int lane) {
  const int64_t base = int64_t(c % nkc) * FS_KC;
  os_issue_chunk(smem + (c % FS_STAGES) * FS_STAGE_DOUBLES + FS_RB * OS_XP, bars + c % FS_STAGES,
                 vk + int64_t(c / nkc) * FS_JB * n2p, n2p, base, FS_JB, static_cast<int>(min(int64_t(FS_KC), n2p - base)),
                 lane);
}

// The warp's rows of Y = X_k V_k^T on one j-block (M = 8, N = 32, K = n2p), the first GEMM of fs_grid_kernel and the
// whole of fs_y2_kernel: per column chunk every thread gathers the bin-k pairs of the chunk's pulsars for the block's
// rows while the chunk c of V_k lands; c runs on across j-blocks, and warp 0 refills each stage once all warps are done.
__device__ __forceinline__ void fs_y_block(double (&y)[4][2], int& c, double* smem, uint64_t* bars, const double* xblk,
                                           const double* vk, const ptar_fs_model& m, int nrow, int nkc, int total,
                                           int tid, int lane, int warp, int fr, int fk) {
  const int P = m.n_psr, n2p = m.n2p;
  const int64_t ldx = int64_t(P) * m.ncp;
#pragma unroll
  for (int t = 0; t < 4; ++t) y[t][0] = y[t][1] = 0.0;
  for (int kc = 0; kc < nkc; ++kc, ++c) {
    const int s = c % FS_STAGES;
    double* xs = smem + s * FS_STAGE_DOUBLES;
    const double* vs = xs + FS_RB * OS_XP;
    // the bin-k pair of pulsars 32 kc .. 32 kc + 31 for every row of the block; zero past n_psr and nrow
    for (int e = tid; e < FS_RB * (FS_KC / 2); e += FS_THREADS) {
      const int r = e / (FS_KC / 2), p = e % (FS_KC / 2), a = kc * (FS_KC / 2) + p;
      double2 v = make_double2(0.0, 0.0);
      if (r < nrow && a < P) v = __ldg(reinterpret_cast<const double2*>(xblk + int64_t(r) * ldx + int64_t(a) * m.ncp));
      *reinterpret_cast<double2*>(xs + r * OS_XP + 2 * p) = v;
    }
    os_mbar_wait(bars + s, (c / FS_STAGES) & 1);
    __syncthreads();   // gathered X complete (and, at kc = 0, the caller's W)
    const int cnt = min(FS_KC, n2p - kc * FS_KC);   // a multiple of 8
#pragma unroll 4
    for (int kk = 0; kk < cnt; kk += 4) {
      const double af = xs[(warp * 8 + fr) * OS_XP + kk + fk];
#pragma unroll
      for (int t = 0; t < 4; ++t) PTAR_OS_DMMA(y[t][0], y[t][1], af, vs[(t * 8 + fr) * OS_XP + kk + fk]);
    }
    __syncthreads();   // every warp is done with stage s
    if (warp == 0 && c + FS_STAGES < total) fs_issue_v(smem, bars, vk, n2p, nkc, c + FS_STAGES, lane);
  }
}

// The V_k ring's barriers and its first FS_STAGES chunks
__device__ __forceinline__ void fs_ring_start(double* smem, uint64_t* bars, const double* vk, int n2p, int nkc, int total,
                                              int tid, int lane, int warp) {
  if (tid == 0) {
    for (int s = 0; s < FS_STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(os_smem_u32(bars + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == 0)
    for (int c = 0; c < FS_STAGES && c < total; ++c) fs_issue_v(smem, bars, vk, n2p, nkc, c, lane);
}

__global__ void __launch_bounds__(FS_THREADS, 1) fs_grid_kernel(const double* __restrict__ X, int nreal, ptar_fs_model m,
                                                                double* __restrict__ lnL) {
  extern __shared__ __align__(16) double fs_smem[];
  double* ys = fs_smem + FS_STAGES * FS_STAGE_DOUBLES;
  double* ws = ys + FS_RB * FS_YP;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ws + FS_JB * CURN_WP);
  const int k0 = blockIdx.x * FS_AB, rb0 = blockIdx.y * FS_RB, kb = blockIdx.z;
  const int nrow = min(FS_RB, nreal - rb0);
  const int NA = m.n_amp, n2p = m.n2p;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  const int nkc = (n2p + FS_KC - 1) / FS_KC, njb = m.np / FS_JB, total = njb * nkc;
  const double* xblk = X + int64_t(rb0) * m.n_psr * m.ncp + 2 * kb;
  const double* vk = m.V + int64_t(kb) * m.np * n2p;
  const double* lam = m.lam + int64_t(kb) * m.np;
  fs_ring_start(fs_smem, bars, vk, n2p, nkc, total, tid, lane, warp);

  double q[8][2];
#pragma unroll
  for (int t = 0; t < 8; ++t) q[t][0] = q[t][1] = 0.0;
  double* yw = ys + warp * 8 * FS_YP;
  int c = 0;
  for (int jb = 0; jb < njb; ++jb) {
    grid_w_tile<FS_JB>(ws, lam + jb * FS_JB, m.a2, k0, NA, tid);
    double y[4][2];
    fs_y_block(y, c, fs_smem, bars, xblk, vk, m, nrow, nkc, total, tid, lane, warp, fr, fk);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      yw[fr * FS_YP + t * 8 + 2 * fk] = __dmul_rn(y[t][0], y[t][0]);
      yw[fr * FS_YP + t * 8 + 2 * fk + 1] = __dmul_rn(y[t][1], y[t][1]);
    }
    __syncwarp();
    grid_q_add<FS_JB, FS_YP>(q, yw, ws, fr, fk);
    __syncthreads();   // W is free for the next j-block
  }
  const int r = warp * 8 + fr;
  if (r >= nrow) return;
  grid_store(lnL + (int64_t(rb0 + r) * m.n_bin + kb) * NA, m.ldet + int64_t(kb) * NA, q, k0, NA, fk);
}

}  // namespace ptar

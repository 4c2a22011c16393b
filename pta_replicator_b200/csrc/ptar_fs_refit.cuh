// Spectral refit of the factorised free spectrum (ptar_fs_y2, ptar_fs_refit): per realization, the sum over the bins of
// the free spectrum's per-bin log-likelihood ratios at rho_k(t)^2, for every template t of a spectral model on a grid,
// from the X[r][a] = C_a^T r_a of ptar_os_project and the statics of one free-spectrum model (ptar_fs.cuh: V_k, lambda).
//   fs_y2     y2[r][k][j] = (V_k X_k)_j^2, j < np (zero past 2 n_psr: V_k's pad rows are zero)
//   fs_refit  w_kj(t) = rho_k(t)^2 / (1 + rho_k(t)^2 lambda_kj);
//             lnL[r][t] = 1/2 sum_k sum_j y2[r][k][j] w_kj(t) - 1/2 ldet[t]                 one GEMM of depth K np on DMMA
// The summaries of the maps are ptar_curn_reduce's.
//
// fs_y2: grid = (realization blocks of 64, bins), the j-block loop of fs_grid_kernel (fs_y_block) without its W and Q
// steps; a thread stores the squares of its own Y fragment.  Written once per realization, Y^2 is read by every template
// block of every refit model, where recomputing Y per 64-template block would cost more than the refit GEMM itself.
// fs_refit: grid = (template blocks of 64, realization blocks of 64), template block fastest so that the CTAs that read
// the same Y^2 rows run back to back.  The depth axis d = k np + j is walked in chunks of 64 columns (the last may hold
// 32): warp 0 stages the block's Y^2 chunk [64 x 64] through a 2-stage bulk-async mbarrier ring while every thread forms
// the chunk's W [64 x 64] (two 32-row tiles of ptar_curn.cuh's grid_w_tile, each on its bin's row of rho^2); warp w then
// adds Q += Y^2 W on its realization rows 8w .. 8w + 7 (grid_q_add) and grid_store writes 1/2 (Q - ldet).  A row's Q
// depends on its own X row, the statics and the fixed d order only -- not on the realization block, nreal, chunking or
// real0.  No atomics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_curn.cuh"
#include "ptar_fs.cuh"
#include "ptar_os.cuh"

namespace ptar {

constexpr size_t FS_Y2_SMEM = sizeof(double) * FS_STAGES * FS_STAGE_DOUBLES + 16;   // the V_k ring: 104,464 B

__global__ void __launch_bounds__(FS_THREADS, 2) fs_y2_kernel(const double* __restrict__ X, int nreal, ptar_fs_model m,
                                                              double* __restrict__ y2) {
  extern __shared__ __align__(16) double fs_smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(fs_smem + FS_STAGES * FS_STAGE_DOUBLES);
  const int rb0 = blockIdx.x * FS_RB, kb = blockIdx.y;
  const int nrow = min(FS_RB, nreal - rb0);
  const int n2p = m.n2p;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  const int nkc = (n2p + FS_KC - 1) / FS_KC, njb = m.np / FS_JB, total = njb * nkc;
  const double* xblk = X + int64_t(rb0) * m.n_psr * m.ncp + 2 * kb;
  const double* vk = m.V + int64_t(kb) * m.np * n2p;
  fs_ring_start(fs_smem, bars, vk, n2p, nkc, total, tid, lane, warp);
  const int r = warp * 8 + fr;
  double* out = y2 + (int64_t(rb0 + r) * m.n_bin + kb) * m.np + 2 * fk;
  int c = 0;
  for (int jb = 0; jb < njb; ++jb) {
    double y[4][2];
    fs_y_block(y, c, fs_smem, bars, xblk, vk, m, nrow, nkc, total, tid, lane, warp, fr, fk);
    if (r < nrow)
#pragma unroll
      for (int t = 0; t < 4; ++t)
        *reinterpret_cast<double2*>(out + jb * FS_JB + t * 8) =
            make_double2(__dmul_rn(y[t][0], y[t][0]), __dmul_rn(y[t][1], y[t][1]));
  }
}

constexpr int RF_THREADS = CURN_THREADS;              // the CTA shape of grid_w_tile / grid_q_add / grid_store
constexpr int RF_RB = CURN_RB;                        // realizations per CTA (one m-tile of 8 per warp)
constexpr int RF_TB = CURN_AB;                        // templates per CTA (8 n-tiles)
constexpr int RF_KC = 2 * FS_JB;                      // depth columns per chunk: two 32-row W tiles
constexpr int RF_STAGES = 2;
constexpr int RF_STAGE_DOUBLES = RF_RB * OS_XP;       // Y^2 rows at pitch OS_XP: 34,816 B
constexpr size_t RF_SMEM = sizeof(double) * (RF_STAGES * RF_STAGE_DOUBLES + RF_KC * CURN_WP) + 16;
// = 106,512 B (+ 2 barriers): two CTAs per SM

__global__ void __launch_bounds__(RF_THREADS, 2) fs_refit_kernel(const double* __restrict__ y2, int nreal,
                                                                 ptar_fs_refit_model m, double* __restrict__ lnL) {
  extern __shared__ __align__(16) double rf_smem[];
  double* ws = rf_smem + RF_STAGES * RF_STAGE_DOUBLES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ws + RF_KC * CURN_WP);
  const int t0 = blockIdx.x * RF_TB, rb0 = blockIdx.y * RF_RB;
  const int nrow = min(RF_RB, nreal - rb0);
  const int NT = m.n_tmpl, depth = m.n_bin * m.np;
  const int nch = (depth + RF_KC - 1) / RF_KC;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  const double* yblk = y2 + int64_t(rb0) * depth;
  if (tid == 0) {
    for (int s = 0; s < RF_STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(os_smem_u32(bars + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int c) {   // warp 0: the depth columns 64 c .. 64 c + 63 of the block's Y^2 rows
    os_issue_chunk(rf_smem + (c % RF_STAGES) * RF_STAGE_DOUBLES, bars + c % RF_STAGES, yblk, depth, int64_t(c) * RF_KC,
                   nrow, min(RF_KC, depth - c * RF_KC), lane);
  };
  if (warp == 0)
    for (int c = 0; c < RF_STAGES && c < nch; ++c) issue(c);

  double q[8][2];
#pragma unroll
  for (int t = 0; t < 8; ++t) q[t][0] = q[t][1] = 0.0;
  for (int c = 0; c < nch; ++c) {
    const int s = c % RF_STAGES, cnt = min(RF_KC, depth - c * RF_KC);   // 32 or 64
    for (int h = 0; h < cnt; h += FS_JB) {   // a 32-row tile lies in one bin: np is a multiple of 32
      const int d = c * RF_KC + h;
      grid_w_tile<FS_JB>(ws + h * CURN_WP, m.lam + d, m.rho2 + int64_t(d / m.np) * NT, t0, NT, tid);
    }
    os_mbar_wait(bars + s, (c / RF_STAGES) & 1);
    __syncthreads();   // W complete
    const double* yw = rf_smem + s * RF_STAGE_DOUBLES + warp * 8 * OS_XP;
    for (int h = 0; h < cnt; h += FS_JB) grid_q_add<FS_JB, OS_XP>(q, yw + h, ws + h * CURN_WP, fr, fk);
    __syncthreads();   // stage s and W are free
    if (warp == 0 && c + RF_STAGES < nch) issue(c + RF_STAGES);
  }
  const int r = warp * 8 + fr;
  if (r >= nrow) return;
  grid_store(lnL + int64_t(rb0 + r) * NT, m.ldet, q, t0, NT, fk);
}

}  // namespace ptar

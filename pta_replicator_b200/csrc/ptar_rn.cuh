// Single-pulsar intrinsic red-noise likelihood (ptar_rn_grid): per realization and pulsar, the log-likelihood ratio of
// a power law in (A, gamma) on the pulsar's own red-noise basis against the white + ECORR (+ common) noise model, on a
// grid, from the X[r][a] = C_a^T r_a of ptar_os_project.  The summaries are ptar_curn_reduce's, one map per
// (realization, pulsar).
//
// The noise-model work is realization-independent and done once on the host (engine.PulsarBatch._plan_rn): per pulsar
// a and grid gamma, the eigendecomposition phi~_a^{1/2} Z_a phi~_a^{1/2} = U diag(lambda) U^T, V_a(gamma) =
// U^T phi~_a^{1/2} and ldet[a][g][k] = sum_j log1p(A_k^2 lambda_j).  Per realization:
//   rn_grid  y = V_a(gamma) X_a;  w_j(A) = A^2 / (1 + A^2 lambda_j);  lnL[r][a][g][k] = 1/2 sum_j w_j(A_k) y_j^2 - 1/2 ldet
//            fused two-GEMM chain on DMMA, as curn_grid, with no pulsar sum and ncp up to 64
//
// grid = (amplitude blocks of 64, realization blocks of 64, pulsars x groups of RN_GB gammas), amplitude block fastest
// so that the CTAs that share X_a and V_a run back to back; the gamma groups give a realization sub-block of the
// engine (a few hundred realizations) several waves of CTAs.  A CTA stages its X_a [64 x ncp] once, then loops over
// the gammas of its group with V_a(gamma) [ncp x ncp] double-buffered through a bulk-async mbarrier ring
// (os_issue_chunk) while every thread forms w_j(A) [ncp x 64] in shared memory.  Warp w owns the realization rows 8w .. 8w + 7 of both GEMMs: Y = X_a V_a^T (M = 8,
// N = ncp, K = ncp), Y^2 to shared memory (its own rows only: a __syncwarp, no CTA barrier), then Q = Y^2 W (M = 8,
// N = 64, K = ncp) in registers, stored per gamma.  Shared memory is sized for ncp = 64 at every instantiation:
// X 34,816 B + 2 V stages 69,632 B + Y^2 34,816 B + W 36,864 B + barriers = 176,160 B, one CTA per SM.  An output
// depends on its own X row and the statics only -- not on the realization block, nreal, chunking or real0.  No atomics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_curn.cuh"
#include "ptar_os.cuh"

namespace ptar {

constexpr int RN_THREADS = CURN_THREADS;                     // the CTA shape of the body shared with curn_grid_kernel
constexpr int RN_RB = CURN_RB;                               // realizations per CTA (one m-tile of 8 per warp)
constexpr int RN_AB = CURN_AB;                               // amplitudes per CTA (8 n-tiles)
constexpr int RN_STAGES = 2;                                 // V_a(gamma) buffers
constexpr int RN_GB = 16;                                    // gammas per CTA
constexpr int RN_YP = PTAR_RN_MAX_NC + 4;                    // Y^2 pitch: rows 32 B apart -> conflict-free A gathers
constexpr size_t RN_SMEM = sizeof(double) * (RN_RB * OS_XP + RN_STAGES * PTAR_RN_MAX_NC * OS_XP + RN_RB * RN_YP +
                                             PTAR_RN_MAX_NC * CURN_WP) + 32;   // + 3 barriers: 176,160 B

template <int NT>   // n-tiles of 8 basis columns: ncp = 8 NT
__global__ void __launch_bounds__(RN_THREADS, 1) rn_grid_kernel(const double* __restrict__ X, int nreal, ptar_rn_model m,
                                                               double* __restrict__ lnL) {
  extern __shared__ __align__(16) double rn_smem[];
  constexpr int NCP = 8 * NT;
  double* xs = rn_smem;
  double* vring = xs + RN_RB * OS_XP;
  double* ys = vring + RN_STAGES * PTAR_RN_MAX_NC * OS_XP;
  double* ws = ys + RN_RB * RN_YP;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ws + PTAR_RN_MAX_NC * CURN_WP);   // [0, RN_STAGES) V stages, then X
  const int P = m.n_psr, NA = m.n_amp, NG = m.n_gamma, ngg = (NG + RN_GB - 1) / RN_GB;
  const int k0 = blockIdx.x * RN_AB, rb0 = blockIdx.y * RN_RB, a = blockIdx.z / ngg;
  const int g0 = (blockIdx.z % ngg) * RN_GB, ng = min(RN_GB, NG - g0);
  const int nrow = min(RN_RB, nreal - rb0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  const int64_t ldx = int64_t(P) * NCP;
  const double* va = m.V + int64_t(a) * NG * NCP * NCP;
  if (tid == 0) {
    for (int s = 0; s <= RN_STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(os_smem_u32(bars + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int i) {   // warp 0: the ncp rows of V_a(gamma_{g0 + i})
    os_issue_chunk(vring + (i % RN_STAGES) * PTAR_RN_MAX_NC * OS_XP, bars + i % RN_STAGES,
                   va + int64_t(g0 + i) * NCP * NCP, NCP, 0, NCP, NCP, lane);
  };
  if (warp == 0) {
    os_issue_chunk(xs, bars + RN_STAGES, X + int64_t(rb0) * ldx, ldx, int64_t(a) * NCP, nrow, NCP, lane);
    for (int i = 0; i < RN_STAGES && i < ng; ++i) issue(i);
  }

  double* yw = ys + warp * 8 * RN_YP;
  const int r = warp * 8 + fr;
  for (int i = 0; i < ng; ++i) {
    const int g = g0 + i, s = i % RN_STAGES;
    const double* vs = vring + s * PTAR_RN_MAX_NC * OS_XP;
    grid_w_tile<NCP>(ws, m.lam + (int64_t(a) * NG + g) * NCP, m.a2, k0, NA, tid);
    if (i == 0) os_mbar_wait(bars + RN_STAGES, 0);
    os_mbar_wait(bars + s, (i / RN_STAGES) & 1);
    __syncthreads();   // W complete
    grid_y2_rows<NT, RN_YP>(yw, xs, vs, warp, fr, fk);
    __syncwarp();
    double q[8][2];
#pragma unroll
    for (int t = 0; t < 8; ++t) q[t][0] = q[t][1] = 0.0;
    grid_q_add<NCP, RN_YP>(q, yw, ws, fr, fk);
    if (r < nrow)
      grid_store(lnL + ((int64_t(rb0 + r) * P + a) * NG + g) * NA, m.ldet + (int64_t(a) * NG + g) * NA, q, k0, NA, fk);
    __syncthreads();   // stage s, W and Y^2 are free
    if (warp == 0 && i + RN_STAGES < ng) issue(i + RN_STAGES);
  }
}

}  // namespace ptar

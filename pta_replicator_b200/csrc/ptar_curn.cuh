// Common uncorrelated red process (CURN) likelihood (ptar_curn_grid, ptar_curn_reduce): per realization, the
// log-likelihood ratio of a power law in (A, gamma) shared by every pulsar against the noise-only model, on a grid, and
// its summaries, from the X[r][a] = C_a^T r_a of ptar_os_project.
//
// The noise-model work is realization-independent and done once on the host (engine.PulsarBatch._plan_curn): per
// pulsar a and grid gamma, the eigendecomposition phi~^{1/2} Z_a phi~^{1/2} = U diag(lambda) U^T, V_a(gamma) =
// U^T phi~^{1/2} and ldet(A, gamma) = sum_a sum_j log1p(A^2 lambda_j).  Per realization:
//   curn_grid    y = V_a(gamma) X_a;  w_j(A) = A^2 / (1 + A^2 lambda_j);  Q(A, gamma) = sum_a sum_j w_j(A) y_j^2;
//                lnL = 1/2 Q - 1/2 ldet                                          fused two-GEMM chain on DMMA
//   curn_reduce  max, first argmax (gamma-major), ln B, the marginal densities in log10 A and gamma, the upper limit
//
// curn_grid: grid = (amplitude blocks of 64, realization blocks of 64, gamma), amplitude block fastest so that the CTAs
// that share X and V run back to back.  Per pulsar, in index order, warp 0 stages X_a [64 x ncp] and V_a(gamma)
// [ncp x ncp] through a 2-stage bulk-async mbarrier ring (os_issue_chunk, two arrivals per stage) while every thread
// forms w_j(A) [ncp x 64] in shared memory.  Warp w owns the realization rows 8w .. 8w + 7 of both GEMMs:
// Y = X_a V_a^T (M = 8, N = ncp, K = ncp), Y^2 to shared memory (its own rows only: a __syncwarp, no CTA barrier),
// then Q += Y^2 W (M = 8, N = 64, K = ncp) in registers across all pulsars.  A row's Q depends on its own X row, the
// statics and the pulsar order only -- not on the realization block, nreal, chunking or real0.  No atomics.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_os.cuh"

namespace ptar {

constexpr int CURN_THREADS = 256;
constexpr int CURN_RB = 64;                                  // realizations per CTA (one m-tile of 8 per warp)
constexpr int CURN_AB = 64;                                  // amplitudes per CTA (8 n-tiles)
constexpr int CURN_STAGES = 2;
constexpr int CURN_STAGE_DOUBLES = (CURN_RB + PTAR_OS_MAX_NC) * OS_XP;   // X rows then V rows, pitch OS_XP: 52,224 B
constexpr int CURN_YP = PTAR_OS_MAX_NC + 4;                  // Y^2 pitch: rows 32 B apart -> conflict-free A gathers
constexpr int CURN_WP = CURN_AB + 8;                         // W pitch: k rows 64 B apart -> conflict-free B gathers
constexpr size_t CURN_SMEM = sizeof(double) * (CURN_STAGES * CURN_STAGE_DOUBLES + CURN_RB * CURN_YP +
                                               PTAR_OS_MAX_NC * CURN_WP) + 16;   // + barriers: 141,328 B
constexpr int CURN_RED_THREADS = 256;                        // >= PTAR_CURN_MAX_NA and PTAR_CURN_MAX_NG

// The per-pulsar body of curn_grid_kernel and rn_grid_kernel (ptar_rn.cuh): a CTA of CURN_THREADS threads over
// CURN_RB realizations x CURN_AB amplitudes, warp w owning the realization rows 8w .. 8w + 7.

// w_j(A) = A^2 / (1 + A^2 lambda_j) [ncp x 64] of the amplitudes k0 .. k0 + 63, the IEEE expression of the host oracle
// (no contraction); 0 past n_amp
template <int NCP>
__device__ __forceinline__ void grid_w_tile(double* ws, const double* lam, const double* a2s, int k0, int NA, int tid) {
  for (int e = tid; e < NCP * CURN_AB; e += CURN_THREADS) {
    const int j = e / CURN_AB, n = e % CURN_AB;
    const double a2 = k0 + n < NA ? __ldg(a2s + k0 + n) : 0.0;
    ws[j * CURN_WP + n] = __ddiv_rn(a2, __dadd_rn(1.0, __dmul_rn(a2, __ldg(lam + j))));
  }
}

// The warp's rows of Y = X_a V_a^T (M = 8, N = ncp, K = ncp) from X_a and V_a staged at pitch OS_XP, squared into its
// own rows yw of Y^2 (pitch YP); the caller's __syncwarp publishes them
template <int NT, int YP>
__device__ __forceinline__ void grid_y2_rows(double* yw, const double* xs, const double* vs, int warp, int fr, int fk) {
  constexpr int NCP = 8 * NT;
  double y[NT][2];
#pragma unroll
  for (int t = 0; t < NT; ++t) y[t][0] = y[t][1] = 0.0;
#pragma unroll
  for (int kk = 0; kk < NCP; kk += 4) {
    const double af = xs[(warp * 8 + fr) * OS_XP + kk + fk];
#pragma unroll
    for (int t = 0; t < NT; ++t) PTAR_OS_DMMA(y[t][0], y[t][1], af, vs[(t * 8 + fr) * OS_XP + kk + fk]);
  }
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    yw[fr * YP + t * 8 + 2 * fk] = __dmul_rn(y[t][0], y[t][0]);
    yw[fr * YP + t * 8 + 2 * fk + 1] = __dmul_rn(y[t][1], y[t][1]);
  }
}

// Q += Y^2 W (M = 8, N = 64, K = ncp) on the warp's rows of Y^2
template <int NCP, int YP>
__device__ __forceinline__ void grid_q_add(double (&q)[8][2], const double* yw, const double* ws, int fr, int fk) {
#pragma unroll
  for (int kk = 0; kk < NCP; kk += 4) {
    const double af = yw[fr * YP + kk + fk];
#pragma unroll
    for (int t = 0; t < 8; ++t) PTAR_OS_DMMA(q[t][0], q[t][1], af, ws[(kk + fk) * CURN_WP + t * 8 + fr]);
  }
}

// out[k] = 1/2 (Q - ldet[k]) of the thread's row at its amplitudes k0 + 8t + 2 fk + c < n_amp
__device__ __forceinline__ void grid_store(double* out, const double* ld, const double (&q)[8][2], int k0, int NA, int fk) {
#pragma unroll
  for (int t = 0; t < 8; ++t)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int k = k0 + t * 8 + 2 * fk + c;
      if (k < NA) out[k] = __dmul_rn(0.5, __dsub_rn(q[t][c], __ldg(ld + k)));
    }
}

template <int NT>   // n-tiles of 8 basis columns: ncp = 8 NT
__global__ void __launch_bounds__(CURN_THREADS, 1) curn_grid_kernel(const double* __restrict__ X, int nreal,
                                                                   ptar_curn_model cm, double* __restrict__ lnL) {
  extern __shared__ __align__(16) double curn_smem[];
  constexpr int NCP = 8 * NT;
  double* ys = curn_smem + CURN_STAGES * CURN_STAGE_DOUBLES;
  double* ws = ys + CURN_RB * CURN_YP;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ws + PTAR_OS_MAX_NC * CURN_WP);
  const int k0 = blockIdx.x * CURN_AB, rb0 = blockIdx.y * CURN_RB, g = blockIdx.z;
  const int nrow = min(CURN_RB, nreal - rb0);
  const int P = cm.n_psr, NA = cm.n_amp, NG = cm.n_gamma;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  const int64_t ldx = int64_t(P) * NCP;
  const double* xblk = X + int64_t(rb0) * ldx;
  if (tid == 0) {
    for (int s = 0; s < CURN_STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 2;" ::"r"(os_smem_u32(bars + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int a) {   // warp 0: X_a rows of the realization block, then the ncp rows of V_a(gamma)
    double* st = curn_smem + (a % CURN_STAGES) * CURN_STAGE_DOUBLES;
    uint64_t* bar = bars + a % CURN_STAGES;
    os_issue_chunk(st, bar, xblk, ldx, int64_t(a) * NCP, nrow, NCP, lane);
    os_issue_chunk(st + CURN_RB * OS_XP, bar, cm.V + (int64_t(a) * NG + g) * NCP * NCP, NCP, 0, NCP, NCP, lane);
  };
  if (warp == 0)
    for (int a = 0; a < CURN_STAGES && a < P; ++a) issue(a);

  double q[8][2];
#pragma unroll
  for (int t = 0; t < 8; ++t) q[t][0] = q[t][1] = 0.0;
  double* yw = ys + warp * 8 * CURN_YP;
  for (int a = 0; a < P; ++a) {
    const int s = a % CURN_STAGES;
    const double* xs = curn_smem + s * CURN_STAGE_DOUBLES;
    const double* vs = xs + CURN_RB * OS_XP;
    grid_w_tile<NCP>(ws, cm.lam + (int64_t(a) * NG + g) * NCP, cm.a2, k0, NA, tid);
    os_mbar_wait(bars + s, (a / CURN_STAGES) & 1);
    __syncthreads();   // W complete
    grid_y2_rows<NT, CURN_YP>(yw, xs, vs, warp, fr, fk);
    __syncwarp();
    grid_q_add<NCP, CURN_YP>(q, yw, ws, fr, fk);
    __syncthreads();   // stage s, W and Y^2 are free
    if (warp == 0 && a + CURN_STAGES < P) issue(a + CURN_STAGES);
  }
  const int r = warp * 8 + fr;
  if (r >= nrow) return;
  grid_store(lnL + (int64_t(rb0 + r) * NG + g) * NA, cm.ldet + int64_t(g) * NA, q, k0, NA, fk);
}

// One CTA per realization, over its map lnL[g][k] (k = log10 A index).  Every sum runs in a fixed order: per-thread
// sequences in index order, then fixed-shape trees.
//   m = max lnL, first (g, k) attaining it (gamma-major);  e = exp(lnL - m)
//   s_k = sum_g wg_g e_gk (in g order);  t_g = sum_k wx_k prior_k e_gk (in k order);  B' = tree_k wx_k prior_k s_k
//   ln_bayes = m + ln B';  post_log10_A_k = prior_k s_k / B';  post_gamma_g = t_g / B'
//   ul: the quantile `ul` of the trapezoid CDF of post_log10_A (normalised by its last node), linear between nodes.
// Non-finite maps: the maximum ranks by fe_better (the first NaN above every number).  -inf among finite entries is a
// zero likelihood; a NaN or +inf anywhere makes ln_bayes, both posteriors and ul NaN; an all -inf map gives m = -inf at
// (0, 0), ln_bayes = -inf, posteriors and ul NaN.
__global__ void __launch_bounds__(CURN_RED_THREADS) curn_reduce_kernel(const double* __restrict__ lnL, int nreal,
                                                                       ptar_curn_model cm, double* __restrict__ lmax,
                                                                       int64_t* __restrict__ ml_g, int64_t* __restrict__ ml_a,
                                                                       double* __restrict__ lnb, double* __restrict__ post_a,
                                                                       double* __restrict__ post_g, double* __restrict__ ul) {
  __shared__ double rv[CURN_RED_THREADS];
  __shared__ int ri[CURN_RED_THREADS];
  __shared__ double pa[PTAR_CURN_MAX_NA];
  const int NA = cm.n_amp, NG = cm.n_gamma, n = NA * NG, tid = threadIdx.x;
  const int64_t r = blockIdx.x;
  const double* m = lnL + r * n;
  double best = -INFINITY;
  int bi = INT32_MAX;   // ranks below every entry: a -inf entry still wins on its index
  for (int e = tid; e < n; e += CURN_RED_THREADS) {
    const double v = m[e];
    if (fe_better(v, e, best, bi)) best = v, bi = e;
  }
  rv[tid] = best;
  ri[tid] = bi;
  __syncthreads();
  for (int h = CURN_RED_THREADS / 2; h > 0; h >>= 1) {
    if (tid < h && fe_better(rv[tid + h], ri[tid + h], rv[tid], ri[tid])) {
      rv[tid] = rv[tid + h];
      ri[tid] = ri[tid + h];
    }
    __syncthreads();
  }
  // A NaN or +inf maximum makes every e below NaN (NaN - m, inf - inf), and with them every integral; so does an
  // all -inf map (-inf - -inf), whose ln_bayes is -inf by definition.
  const double mx = rv[0];
  const int am = ri[0];
  __syncthreads();   // rv is reused below
  double sk = 0.0;
  if (tid < NA) {
    for (int g = 0; g < NG; ++g) sk = __dadd_rn(sk, __dmul_rn(__ldg(cm.wg + g), exp(__dsub_rn(m[g * NA + tid], mx))));
    rv[tid] = __dmul_rn(__dmul_rn(__ldg(cm.wx + tid), __ldg(cm.prior + tid)), sk);
  } else {
    rv[tid] = 0.0;
  }
  double tg = 0.0;
  if (tid < NG)
    for (int k = 0; k < NA; ++k)
      tg = __dadd_rn(tg, __dmul_rn(__dmul_rn(__ldg(cm.wx + k), __ldg(cm.prior + k)), exp(__dsub_rn(m[tid * NA + k], mx))));
  __syncthreads();
  for (int h = CURN_RED_THREADS / 2; h > 0; h >>= 1) {
    if (tid < h) rv[tid] = __dadd_rn(rv[tid], rv[tid + h]);
    __syncthreads();
  }
  const double B = rv[0];
  if (tid < NA) {
    const double p = __ddiv_rn(__dmul_rn(__ldg(cm.prior + tid), sk), B);
    pa[tid] = p;
    post_a[r * NA + tid] = p;
  }
  if (tid < NG) post_g[r * NG + tid] = __ddiv_rn(tg, B);
  __syncthreads();
  if (tid == 0) {
    lmax[r] = mx;
    ml_g[r] = am / NA;
    ml_a[r] = am % NA;
    lnb[r] = mx == -INFINITY ? mx : __dadd_rn(mx, log(B));
    const double* x = cm.log10_A;
    double c = 0.0;
    for (int k = 1; k < NA; ++k)
      c = __dadd_rn(c, __dmul_rn(__dmul_rn(0.5, __dsub_rn(x[k], x[k - 1])), __dadd_rn(pa[k - 1], pa[k])));
    const double target = __dmul_rn(cm.ul, c);
    // a posterior that is not finite has no quantile: NaN, never the last node (c >= target is false for every NaN)
    double lo = 0.0, q = isfinite(target) ? x[NA - 1] : NAN;
    c = 0.0;
    for (int k = 1; k < NA; ++k) {
      c = __dadd_rn(c, __dmul_rn(__dmul_rn(0.5, __dsub_rn(x[k], x[k - 1])), __dadd_rn(pa[k - 1], pa[k])));
      if (c >= target) {
        q = __dadd_rn(x[k - 1], __dmul_rn(__dsub_rn(x[k], x[k - 1]), __ddiv_rn(__dsub_rn(target, lo), __dsub_rn(c, lo))));
        break;
      }
      lo = c;
    }
    ul[r] = q;
  }
}

}  // namespace ptar

// Incoherent Fp-statistic (ptar_fp_project, ptar_fp_reduce): per-realization continuous-wave detection statistics of
// the pulsars of a batch, from rows the generator wrote, without the rows leaving the device.
//
// The noise-model work is realization-independent and done once on the host (engine.PulsarBatch._plan_fp): the
// whitened basis C~_a(f) = P_a^{-1} F_f L_a(f)^{-T} for every pulsar a and search frequency f, 2 Nf columns on the
// packed TOA axis.  Per realization:
//   fp_project  amps[r][a][j] = sum_{i in pulsar a} C~[i][j] row_r[i]      fp64 GEMM, M = realizations, N = 2 Nf, K = TOAs
//   fp_reduce   Fp[r][f] = 1/2 sum_a (amps[r][a][2f]^2 + amps[r][a][2f+1]^2)  (pulsar order);  max_f and first argmax
//
// fp_project: one CTA per (pulsar, block of 64 realizations, block of 64 columns) walks ALL TOAs of its pulsar and
// writes its 64 x 64 outputs directly -- no tile partials, no second pass.  The grid is pulsar-major in descending TOA
// count (the longest CTAs start first), then realization block, then column block fastest: the CTAs that share a chunk
// of rows run side by side, and so do the CTAs that share a chunk of C~, so both cross HBM about once.  Per 64-TOA
// chunk, warp 0 stages the rows with os_issue_chunk (one bulk copy per realization row, row pitch OS_XP: conflict-free
// A gathers) and the C~ chunk with ONE bulk copy (Ct is [column block][ld][64]; TOA i's 64 columns are rotated by
// 8 (i & 1) on the host so that the B gathers of the four k-rows of a fragment hit every bank once per wavefront) into
// a 3-stage mbarrier ring (count 2: one arrival for each copy group).  DMMA (mma.sync.m8n8k4.f64): warp w owns the
// 32 x 32 quarter (w & 1, (w >> 1) & 1) and the k-half w >> 2 of every chunk; the two k-halves are added in a fixed order
// at the end.  An output is therefore summed in an order fixed by the TOA index alone -- not by the realization block
// slot, nreal, chunking or real0.  No atomics anywhere.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_os.cuh"

namespace ptar {

constexpr int FP_THREADS = 256;
constexpr int FP_BN = 64;                                        // columns per CTA (one column block of Ct)
constexpr int FP_A_DOUBLES = OS_RB * OS_XP;                      // staged rows: 64 realizations x 64 TOAs, pitch 68
constexpr int FP_STAGE_DOUBLES = FP_A_DOUBLES + OS_KC * FP_BN;   // + the C~ chunk: 67,584 B per stage
constexpr int FP_STAGES = 3;
constexpr size_t FP_SMEM = sizeof(double) * FP_STAGES * FP_STAGE_DOUBLES + 64;   // + barriers: 1 CTA per SM
static_assert(2 * OS_RB * FP_BN <= FP_STAGES * FP_STAGE_DOUBLES, "k-half reduction must fit in the ring");
constexpr int FP_REDUCE_THREADS = PTAR_FP_MAX_FREQ;              // one thread per frequency

// Warp 0 fills stage `st` with the chunk of cnt4 TOAs at packed index `base`: the rows (os_issue_chunk, first arrival)
// and the C~ chunk of this CTA's column block (second arrival, one bulk copy of cnt4 x 64 doubles).
__device__ __forceinline__ void fp_issue_chunk(double* st, uint64_t* bar, const double* rblk, int64_t ld, const double* ctb,
                                               int64_t base, int nrow, int cnt4, int lane) {
  os_issue_chunk(st, bar, rblk, ld, base, nrow, cnt4, lane);
  if (lane == 0) {
    const uint32_t bytes = static_cast<uint32_t>(cnt4) * FP_BN * 8u;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(os_smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     os_smem_u32(st + FP_A_DOUBLES)),
                 "l"(ctb + base * FP_BN), "r"(bytes), "r"(os_smem_u32(bar))
                 : "memory");
  }
}

__global__ void __launch_bounds__(FP_THREADS, 1) fp_project_kernel(const double* __restrict__ rows, int64_t ld, int nreal,
                                                                   ptar_fp_model fp, double* __restrict__ amps) {
  extern __shared__ __align__(16) double fp_smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(fp_smem + FP_STAGES * FP_STAGE_DOUBLES);
  const int nrb = (nreal + OS_RB - 1) / OS_RB;
  const int cb = blockIdx.x % fp.n_cb;
  const int rb = (blockIdx.x / fp.n_cb) % nrb;
  const int p = fp.psr_order[blockIdx.x / (fp.n_cb * nrb)];
  const int64_t s0 = fp.seg_off[p];
  const int n = fp.seg_len[p], nch = (n + OS_KC - 1) / OS_KC;
  const int r0 = rb * OS_RB, nrow = min(OS_RB, nreal - r0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double* rblk = rows + int64_t(r0) * ld;
  const double* ctb = fp.Ct + int64_t(cb) * fp.ld * FP_BN;
  if (tid == 0) {
    for (int s = 0; s < FP_STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 2;" ::"r"(os_smem_u32(bars + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto cnt_of = [&](int c) { return min(OS_KC, n - c * OS_KC); };
  if (warp == 0)
    for (int c = 0; c < FP_STAGES && c < nch; ++c)
      fp_issue_chunk(fp_smem + c * FP_STAGE_DOUBLES, bars + c, rblk, ld, ctb, s0 + c * OS_KC, nrow, (cnt_of(c) + 3) & ~3, lane);

  const int wm = warp & 1, wn = (warp >> 1) & 1, kh = warp >> 2;
  const int fr = lane >> 2, fk = lane & 3;
  double acc[4][4][2];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b][0] = acc[a][b][1] = 0.0;

  for (int c = 0; c < nch; ++c) {
    const int s = c % FP_STAGES;
    double* xs = fp_smem + s * FP_STAGE_DOUBLES;
    const double* cs = xs + FP_A_DOUBLES;
    const int cnt = cnt_of(c), cnt4 = (cnt + 3) & ~3;
    os_mbar_wait(bars + s, (c / FP_STAGES) & 1);
    if (cnt < cnt4) {   // the pulsar's alignment slots: whatever the rows hold there must not reach the sums
      for (int e = tid; e < OS_RB * 4; e += FP_THREADS) {
        const int m = e >> 2, k = cnt + (e & 3);
        if (k < cnt4) xs[m * OS_XP + k] = 0.0;
      }
      __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < OS_KC / 8; ++q) {
      const int kk = kh * (OS_KC / 2) + q * 4;
      if (kk < cnt4) {
        const int kl = kk + fk;
        const int sw = (kl & 1) * 8;   // the host's rotation of odd TOAs (chunks start at even packed indices)
        double af[4], bf[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) af[t] = xs[(wm * 32 + t * 8 + fr) * OS_XP + kl];
#pragma unroll
        for (int t = 0; t < 4; ++t) bf[t] = cs[kl * FP_BN + ((wn * 32 + t * 8 + fr + sw) & (FP_BN - 1))];
#pragma unroll
        for (int mt = 0; mt < 4; ++mt)
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) PTAR_OS_DMMA(acc[mt][nt][0], acc[mt][nt][1], af[mt], bf[nt]);
      }
    }
    __syncthreads();   // every warp is done with stage s
    if (warp == 0 && c + FP_STAGES < nch) {
      const int cn = c + FP_STAGES;
      fp_issue_chunk(xs, bars + s, rblk, ld, ctb, s0 + cn * OS_KC, nrow, (cnt_of(cn) + 3) & ~3, lane);
    }
  }
  // k-halves in a fixed order: red[kh][m][n] (reuses the ring; every copy has landed and been consumed)
  double* red = fp_smem;
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      double* d = red + (kh * OS_RB + wm * 32 + mt * 8 + fr) * FP_BN + wn * 32 + nt * 8 + 2 * fk;
      d[0] = acc[mt][nt][0];
      d[1] = acc[mt][nt][1];
    }
  __syncthreads();
  const int nc = 2 * fp.n_freq;
  const int ncol = min(FP_BN, nc - cb * FP_BN);
  const int64_t ldo = int64_t(fp.n_psr) * nc;
  double* out = amps + int64_t(r0) * ldo + int64_t(p) * nc + cb * FP_BN;
  for (int e = tid; e < nrow * FP_BN; e += FP_THREADS) {
    const int m = e / FP_BN, j = e % FP_BN;
    if (j < ncol) out[m * ldo + j] = __dadd_rn(red[m * FP_BN + j], red[(OS_RB + m) * FP_BN + j]);
  }
}

// Q(P, x) = Gamma(P, x) / Gamma(P) for an integer shape P >= 1: the single-frequency false-alarm probability of Fp
// (Fp ~ Gamma(P, 1) under the null).  For integer P, Q(P, x) = sum_{k < P} t_k with t_k = e^{-x} x^k / k!, every term
// positive.  The largest term t_m, m = min(P - 1, floor(x)), is evaluated in log space; the others follow from it by
// the ratios k / x (down) and x / (k + 1) (up), all <= 1, so nothing overflows and nothing cancels:
//   ln t_m = m ln(x / m) + (m - x) - 1/2 ln(2 pi m) - delta(m),   delta(m) = ln m! - (m + 1/2) ln m + m - 1/2 ln(2 pi)
// with ln(x / m) = log1p((x - m) / m) (x - m exact for x < 2m) and delta by its Stirling series for m >= 16 (truncation
// < 1e-16), ln m! of the exact m! below.  Relative error ~ (x + P) u, the conditioning of Q itself; no branch of a
// general-shape algorithm (the DLMF 8.12 asymptotic series of Cephes igammac loses ~1e-9 where Fp ~ P).  A fixed loop of
// P - 1 steps per (realization, frequency): the value depends on x and P only.
__device__ __forceinline__ double fp_q_int(int P, double x) {
  if (!(x > 0.0)) return x == 0.0 ? 1.0 : x;   // Q(P, 0) = 1; NaN stays NaN (Fp >= 0 otherwise)
  if (x == INFINITY) return 0.0;
  const int m = x < double(P - 1) ? static_cast<int>(floor(x)) : P - 1;
  const double dm = double(m);
  double L;
  if (m == 0) {
    L = -x;
  } else if (m < 16) {
    double f = 1.0;
    for (int k = 2; k <= m; ++k) f *= double(k);   // exact: 15! < 2^53
    L = fma(dm, log(x), -x) - log(f);
  } else {
    const double i1 = 1.0 / dm, i2 = i1 * i1;
    const double delta = i1 * (1.0 / 12 - i2 * (1.0 / 360 - i2 * (1.0 / 1260 - i2 * (1.0 / 1680 - i2 * (1.0 / 1188)))));
    L = dm * log1p((x - dm) / dm) + (dm - x) - (0.9189385332046727418 + 0.5 * log(dm)) - delta;
  }
  double s = 1.0, r = 1.0;
  for (int k = m; k > 0; --k) {
    r *= double(k) / x;
    s += r;
  }
  r = 1.0;
  for (int k = m + 1; k < P; ++k) {
    r *= x / double(k);
    s += r;
  }
  return exp(L) * s;
}

// One CTA per realization, thread f = frequency: Fp in pulsar order, then (max, first argmax) by a fixed tree of
// fe_better (the first NaN above every number, wherever it sits); with `fap` also the false-alarm probability
// Q(n_psr, Fp) per frequency (NaN for a NaN Fp, 0 for +inf).
__global__ void __launch_bounds__(FP_REDUCE_THREADS) fp_reduce_kernel(const double* __restrict__ amps, int nreal,
                                                                      ptar_fp_model fp, double* __restrict__ Fp,
                                                                      double* __restrict__ Fp_max,
                                                                      int64_t* __restrict__ Fp_argmax,
                                                                      double* __restrict__ fap) {
  __shared__ double sv[FP_REDUCE_THREADS];
  __shared__ int si[FP_REDUCE_THREADS];
  const int64_t r = blockIdx.x;
  const int nf = fp.n_freq, f = threadIdx.x;
  const int64_t nc = 2 * nf;
  double v = -INFINITY;
  if (f < nf) {
    const double* a = amps + r * fp.n_psr * nc + 2 * f;
    double s = 0.0;
    for (int q = 0; q < fp.n_psr; ++q) {
      const double2 x = *reinterpret_cast<const double2*>(a + q * nc);
      s = __dadd_rn(s, __fma_rn(x.y, x.y, __dmul_rn(x.x, x.x)));
    }
    v = __dmul_rn(0.5, s);
    Fp[r * nf + f] = v;
    if (fap) fap[r * nf + f] = fp_q_int(fp.n_psr, v);
  }
  sv[f] = v;
  si[f] = f;
  __syncthreads();
  for (int h = FP_REDUCE_THREADS / 2; h > 0; h >>= 1) {
    if (f < h) {
      const double b = sv[f + h];
      const int bi = si[f + h];
      if (fe_better(b, bi, sv[f], si[f])) {
        sv[f] = b;
        si[f] = bi;
      }
    }
    __syncthreads();
  }
  if (f == 0) {
    Fp_max[r] = sv[0];
    Fp_argmax[r] = si[0];
  }
}

}  // namespace ptar

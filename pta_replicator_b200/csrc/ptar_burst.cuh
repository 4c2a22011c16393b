// Sine-Gaussian burst search over a t0 x f0 x Q bank and the sky (ptar_burst_ninv, ptar_burst_project, ptar_burst_reduce):
// per-realization whitened wavelet amplitudes X^ in the layout of ptar_fp_project, which ptar_fe_sky turns into the
// coherent statistic per (template, sky), and the maxima over the whole bank.
//
// Template j = (t0, f0, Q), tau = Q / (2 pi f0): W_j(t) = exp(-(t - t0)^2 / tau^2) (cos, sin)(2 pi f0 (t - t0)) on the TOAs of
// the static range [lo, hi) that spans |t - t0| <= 6 tau, zero elsewhere.  The noise-model work is realization-independent
// and done once on the host (engine.PulsarBatch._plan_burst): with P_a^-1 = N^-1 - N^-1 T S^-1 T^T N^-1 (N white + ECORR,
// T the timing model, red noise and common basis, S = L_S L_S^T), the z columns N^-1 T L_S^-T (projected by the unchanged
// ptar_fp_project: z_a = L_S^-1 T^T N^-1 r_a), H_a(j) = L_S^-1 T^T N^-1 W_j [rank x 2] and the closed-form 2 x 2 inverse
// factor of M_a(j) = W_j^T P_a^-1 W_j.  Per realization r:
//   burst_ninv     y = N^-1 r on the packed axis: y_i = (r_i - coef_run sum_{k in run} r_k / d_k) / d_i, one Sherman-Morrison
//                  term per ECORR run (a run of one TOA, coef 0, without ECORR); a run is summed in TOA order
//   burst_project  N_a(j) = W_j^T y_a - H_a(j)^T z_a,  X^_a(j) = L^-1 N_a(j)  (0 for an unseen cell)
//
// burst_project: one CTA per (pulsar, 64 realizations, 16 templates = 32 columns) walks only the union of its templates'
// windows (static per-(pulsar, block) TOA range; the bank is sorted by (tau, t0), so a block's windows are neighbours).
// Per 64-TOA chunk, warp 0 stages y with os_issue_chunk into a 2-stage bulk-async ring while the CTA generates the
// 64 x 32 W chunk in shared memory: one exp and one sincospi (fp64) per (TOA, template) for the two columns, 4 per
// thread, amortised over the CTA's 64 realizations (2 x 64 DMMA multiply-adds per generated pair).  DMMA (mma.sync.m8n8k4.f64):
// warp w owns rows 32 (w & 1) .. +31 and TOA quarter w >> 1 of every chunk (4 k-steps); the quarters are added in a fixed
// order at the end, then the epilogue subtracts H^T z (k in increasing order) and whitens.  Every sum runs in an order
// fixed by the TOA and z index alone: outputs are bit-identical whatever nreal, chunking or real0.  No atomics anywhere.
//
// burst_reduce: one thread per realization takes the maximum of ptar_fe_sky's per-template maxima over the bank (ties to
// the lower template, whose sky index is fe_sky's first), re-forms N4 there in pulsar order and gives a^ = M4^-1 N4; one
// thread per (realization, pulsar) takes the per-pulsar transient statistic 1/2 |X^|^2 over the templates the pulsar sees
// and a^_a = M_a^-1 N_a = L^-T X^ at its maximum.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_fe.cuh"
#include "ptar_os.cuh"

namespace ptar {

constexpr int BU_THREADS = 256;
constexpr int BU_TB = PTAR_BURST_TB;                          // templates per CTA
constexpr int BU_BN = 2 * BU_TB;                              // columns per CTA
constexpr int BU_WP = BU_BN + 4;                              // W row pitch: conflict-free B gathers
constexpr int BU_STAGES = 2;
constexpr int BU_W_DOUBLES = OS_KC * BU_WP;
constexpr size_t BU_SMEM = sizeof(double) * (BU_STAGES * OS_STAGE_DOUBLES + BU_W_DOUBLES) + 64;   // 88 KB: 2 CTAs per SM
static_assert(4 * OS_RB * BU_BN <= BU_STAGES * OS_STAGE_DOUBLES, "the k-quarter reduction must fit in the ring");
static_assert(PTAR_BURST_GROUP % BU_TB == 0, "a group is whole template blocks");
constexpr int BU_NINV_THREADS = 256;
constexpr int BU_REDUCE_THREADS = 128;

// y = N^-1 r: thread (TOA, realization).  Each thread sums its run in TOA order (the threads of a run read the same
// addresses, so a warp's loads are broadcasts) and writes its own TOA: coalesced rows, and every TOA of a run gets the
// same sum.  Alignment slots (toa_run < 0) are not written.
__global__ void __launch_bounds__(BU_NINV_THREADS) burst_ninv_kernel(const double* __restrict__ rows, int64_t ld, int nreal,
                                                                     ptar_burst_model bm, double* __restrict__ y) {
  const int64_t i = int64_t(blockIdx.x) * BU_NINV_THREADS + threadIdx.x;
  if (i >= ld) return;
  const int q = bm.toa_run[i];
  if (q < 0) return;
  const int64_t s = bm.run_start[q];
  const int len = bm.run_len[q];
  const double coef = bm.run_coef[q], di = bm.dinv[i];
  for (int r = blockIdx.y; r < nreal; r += gridDim.y) {
    const double* x = rows + int64_t(r) * ld;
    double sum = 0.0;
    if (coef != 0.0)
      for (int k = 0; k < len; ++k) sum = __fma_rn(x[s + k], bm.dinv[s + k], sum);
    y[int64_t(r) * ld + i] = __dmul_rn(__dsub_rn(x[i], __dmul_rn(coef, sum)), di);
  }
}

__global__ void __launch_bounds__(BU_THREADS, 2) burst_project_kernel(const double* __restrict__ y, int64_t ld, int nreal,
                                                                      const double* __restrict__ z, ptar_burst_model bm,
                                                                      int group, double* __restrict__ amps) {
  extern __shared__ __align__(16) double bu_smem[];
  double* ws = bu_smem + BU_STAGES * OS_STAGE_DOUBLES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ws + BU_W_DOUBLES);
  __shared__ double tp[BU_TB][3];
  __shared__ int tw[BU_TB][2];
  const int j0g = group * PTAR_BURST_GROUP;
  const int jg = min(PTAR_BURST_GROUP, bm.n_tmpl - j0g);           // templates of this group
  const int ntb = (jg + BU_TB - 1) / BU_TB;
  const int nrb = (nreal + OS_RB - 1) / OS_RB;
  const int tb = blockIdx.x % ntb;
  const int rb = (blockIdx.x / ntb) % nrb;
  const int p = bm.psr_order[blockIdx.x / (ntb * nrb)];
  const int P = bm.n_psr, J = bm.n_tmpl;
  const int jb0 = j0g + tb * BU_TB;                                  // first template of the block (bank index)
  const int nt = min(BU_TB, j0g + jg - jb0);
  const int64_t s0 = bm.seg_off[p];
  const int2 rng = reinterpret_cast<const int2*>(bm.blk)[int64_t(p) * ((J + BU_TB - 1) / BU_TB) + jb0 / BU_TB];
  const int lo = rng.x, n = rng.y - rng.x, nch = n > 0 ? (n + OS_KC - 1) / OS_KC : 0;   // lo: a multiple of 4
  const int r0 = rb * OS_RB, nrow = min(OS_RB, nreal - r0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double* rblk = y + int64_t(r0) * ld;
  if (tid < BU_TB) {
    const bool ok = tid < nt;
    const int j = jb0 + tid;
    tp[tid][0] = ok ? bm.tmpl[4 * j] : 0.0;
    tp[tid][1] = ok ? bm.tmpl[4 * j + 1] : 0.0;
    tp[tid][2] = ok ? bm.tmpl[4 * j + 2] : 0.0;
    const int2 w = ok ? reinterpret_cast<const int2*>(bm.win)[int64_t(p) * J + j] : make_int2(0, 0);
    tw[tid][0] = w.x;
    tw[tid][1] = w.y;
  }
  if (tid == 0) {
    for (int s = 0; s < BU_STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(os_smem_u32(bars + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto cnt_of = [&](int c) { return min(OS_KC, n - c * OS_KC); };
  if (warp == 0)
    for (int c = 0; c < BU_STAGES && c < nch; ++c)
      os_issue_chunk(bu_smem + c * OS_STAGE_DOUBLES, bars + c, rblk, ld, s0 + lo + c * OS_KC, nrow, (cnt_of(c) + 3) & ~3, lane);

  const int wm = warp & 1, kq = warp >> 1;
  const int fr = lane >> 2, fk = lane & 3;
  double acc[4][4][2];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b][0] = acc[a][b][1] = 0.0;

  for (int c = 0; c < nch; ++c) {
    const int s = c % BU_STAGES;
    double* xs = bu_smem + s * OS_STAGE_DOUBLES;
    const int base = lo + c * OS_KC;                                 // local TOA index of the chunk's first row
    const int cnt = cnt_of(c), cnt4 = (cnt + 3) & ~3;
    // W of the chunk: (TOA k, template tl) pairs, one exp and one sincos each; zero outside the template's window
#pragma unroll
    for (int q = 0; q < OS_KC * BU_TB / BU_THREADS; ++q) {
      const int e = tid + q * BU_THREADS, tl = e % BU_TB, k = e / BU_TB, i = base + k;
      double2 w = make_double2(0.0, 0.0);
      if (i >= tw[tl][0] && i < tw[tl][1]) {
        const double x = __dsub_rn(bm.t[s0 + i], tp[tl][0]);
        const double u = __dmul_rn(x, tp[tl][1]);
        const double g = exp(-__dmul_rn(u, u));
        double sn, cs;
        sincospi(__dmul_rn(tp[tl][2], x), &sn, &cs);   // exact reduction by integers: no Payne-Hanek path, no stack
        w = make_double2(__dmul_rn(g, cs), __dmul_rn(g, sn));
      }
      *reinterpret_cast<double2*>(ws + k * BU_WP + 2 * tl) = w;
    }
    os_mbar_wait(bars + s, (c / BU_STAGES) & 1);
    if (cnt < cnt4)   // past the pulsar's last TOA: whatever the scratch holds there must not reach the sums
      for (int e = tid; e < OS_RB * 4; e += BU_THREADS) {
        const int m = e >> 2, k = cnt + (e & 3);
        if (k < cnt4) xs[m * OS_XP + k] = 0.0;
      }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < OS_KC / 16; ++q) {
      const int kk = kq * (OS_KC / 4) + q * 4;
      if (kk < cnt4) {
        const int kl = kk + fk;
        double af[4], bf[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) af[t] = xs[(wm * 32 + t * 8 + fr) * OS_XP + kl];
#pragma unroll
        for (int t = 0; t < 4; ++t) bf[t] = ws[kl * BU_WP + t * 8 + fr];
#pragma unroll
        for (int mt = 0; mt < 4; ++mt)
#pragma unroll
          for (int nt2 = 0; nt2 < 4; ++nt2) PTAR_OS_DMMA(acc[mt][nt2][0], acc[mt][nt2][1], af[mt], bf[nt2]);
      }
    }
    __syncthreads();   // every warp is done with stage s and with W
    if (warp == 0 && c + BU_STAGES < nch) {
      const int cn = c + BU_STAGES;
      os_issue_chunk(xs, bars + s, rblk, ld, s0 + lo + cn * OS_KC, nrow, (cnt_of(cn) + 3) & ~3, lane);
    }
  }
  // k-quarters in a fixed order: red[kq][m][n] (reuses the ring; every copy has landed and been consumed)
  double* red = bu_smem;
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt2 = 0; nt2 < 4; ++nt2) {
      double* d = red + (kq * OS_RB + wm * 32 + mt * 8 + fr) * BU_BN + nt2 * 8 + 2 * fk;
      d[0] = acc[mt][nt2][0];
      d[1] = acc[mt][nt2][1];
    }
  __syncthreads();
  const int nzc = bm.n_zc;
  const int64_t ldo = int64_t(P) * 2 * jg;
  for (int e = tid; e < nrow * BU_TB; e += BU_THREADS) {
    const int m = e / BU_TB, tl = e % BU_TB;
    if (tl >= nt) continue;
    const int j = jb0 + tl;
    double v[2];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int col = 2 * tl + c;
      v[c] = __dadd_rn(__dadd_rn(__dadd_rn(red[m * BU_BN + col], red[(OS_RB + m) * BU_BN + col]),
                                 red[(2 * OS_RB + m) * BU_BN + col]),
                       red[(3 * OS_RB + m) * BU_BN + col]);
    }
    const double* zr = z + (int64_t(r0 + m) * P + p) * nzc;
    const double* h = bm.H + (int64_t(p) * J + j) * 2 * nzc;
    double hz0 = 0.0, hz1 = 0.0;
    for (int k = 0; k < nzc; ++k) {
      const double zk = zr[k];
      hz0 = __fma_rn(h[k], zk, hz0);
      hz1 = __fma_rn(h[nzc + k], zk, hz1);
    }
    const double n0 = __dsub_rn(v[0], hz0), n1 = __dsub_rn(v[1], hz1);
    const double* wl = bm.wl + (int64_t(p) * J + j) * 3;
    double* o = amps + int64_t(r0 + m) * ldo + int64_t(p) * 2 * jg + 2 * (j - j0g);
    o[0] = __dmul_rn(wl[0], n0);
    o[1] = __fma_rn(wl[1], n0, __dmul_rn(wl[2], n1));
  }
}

// Per realization: the maximum over the bank of fe_sky's per-template maxima, and a^ = M4^-1 N4 at that cell.
__global__ void __launch_bounds__(BU_REDUCE_THREADS) burst_reduce_kernel(const double* __restrict__ amps,
                                                                         const double* __restrict__ jmax,
                                                                         const int64_t* __restrict__ jargmax, int nreal,
                                                                         ptar_burst_model bm, double* __restrict__ B_tmpl,
                                                                         int64_t* __restrict__ B_tmpl_sky,
                                                                         double* __restrict__ B_max,
                                                                         int64_t* __restrict__ argmax_tmpl,
                                                                         int64_t* __restrict__ argmax_sky,
                                                                         double* __restrict__ fap, double* __restrict__ amp) {
  const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= nreal) return;
  const int J = bm.n_tmpl, P = bm.n_psr;
  double best = 0.0;
  int bj = -1;
  int64_t bs = 0;
  for (int j = 0; j < J; ++j) {
    const int g = j / PTAR_BURST_GROUP, jg = min(PTAR_BURST_GROUP, J - g * PTAR_BURST_GROUP);
    const int64_t at = int64_t(g) * PTAR_BURST_GROUP * nreal + r * jg + (j - g * PTAR_BURST_GROUP);
    const double v = jmax[at];
    const int64_t s = jargmax[at];
    B_tmpl[r * J + j] = v;
    B_tmpl_sky[r * J + j] = s;
    if (bj < 0 || fe_better(v, j, best, bj)) {
      best = v;
      bj = j;
      bs = s;
    }
  }
  B_max[r] = best;
  argmax_tmpl[r] = bj;
  argmax_sky[r] = bs;
  fap[r] = exp(-best) * (1.0 + best);
  // N4[2 pol + c] = sum_a e_a(s)[pol] (L X^)[c] at (bj, bs), in pulsar order
  const int g = bj / PTAR_BURST_GROUP, jg = min(PTAR_BURST_GROUP, J - g * PTAR_BURST_GROUP);
  const double* ab = amps + int64_t(g) * PTAR_BURST_GROUP * nreal * P * 2 + r * P * 2 * jg + 2 * (bj - g * PTAR_BURST_GROUP);
  double n4[4] = {0.0, 0.0, 0.0, 0.0};
  for (int a = 0; a < P; ++a) {
    const double x0 = ab[int64_t(a) * 2 * jg], x1 = ab[int64_t(a) * 2 * jg + 1];
    const double* l = bm.Lf + (int64_t(bj) * P + a) * 3;
    const double m0 = __dmul_rn(l[0], x0), m1 = __fma_rn(l[1], x0, __dmul_rn(l[2], x1));
    const double* e = bm.antenna + (int64_t(a) * bm.n_sky + bs) * 2;
    n4[0] = __fma_rn(e[0], m0, n4[0]);
    n4[1] = __fma_rn(e[0], m1, n4[1]);
    n4[2] = __fma_rn(e[1], m0, n4[2]);
    n4[3] = __fma_rn(e[1], m1, n4[3]);
  }
  // y = L4^-1 N4 (rows 00, 10, 11, 20, 21, 22, 30 .. 33), a^ = L4^-T y
  const double* L = bm.linv + (int64_t(bj) * bm.n_sb * FE_SB + bs) * FE_LINV;
  double yv[4];
  yv[0] = L[0] * n4[0];
  yv[1] = L[1] * n4[0] + L[2] * n4[1];
  yv[2] = L[3] * n4[0] + L[4] * n4[1] + L[5] * n4[2];
  yv[3] = L[6] * n4[0] + L[7] * n4[1] + L[8] * n4[2] + L[9] * n4[3];
  const double a3 = L[9] * yv[3];
  const double a2 = L[5] * yv[2] + L[8] * yv[3];
  const double a1 = L[2] * yv[1] + L[4] * yv[2] + L[7] * yv[3];
  const double a0 = L[0] * yv[0] + L[1] * yv[1] + L[3] * yv[2] + L[6] * yv[3];
  // the model residual is sum b e_pol W_c; add_burst's is -(F+ h+ + Fx hx): a = -b
  amp[r * 4 + 0] = -a0;
  amp[r * 4 + 1] = -a1;
  amp[r * 4 + 2] = -a2;
  amp[r * 4 + 3] = -a3;
}

// Per (realization, pulsar): Bt = 1/2 |X^|^2 over the templates the pulsar sees, its maximum, template, e^-Bt and
// a^_a = L^-T X^ there; with `maps` every Bt (0 at an unseen template).
__global__ void __launch_bounds__(BU_REDUCE_THREADS) burst_psr_kernel(const double* __restrict__ amps, int nreal,
                                                                      ptar_burst_model bm, double* __restrict__ Bt_max,
                                                                      int64_t* __restrict__ argmax, double* __restrict__ fap,
                                                                      double* __restrict__ amp, double* __restrict__ maps) {
  const int64_t q = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int P = bm.n_psr, J = bm.n_tmpl;
  if (q >= int64_t(nreal) * P) return;
  const int64_t r = q / P;
  const int a = static_cast<int>(q - r * P);
  double best = -INFINITY, bx0 = 0.0, bx1 = 0.0;
  int bj = -1;
  for (int j = 0; j < J; ++j) {
    const int g = j / PTAR_BURST_GROUP, jg = min(PTAR_BURST_GROUP, J - g * PTAR_BURST_GROUP);
    const double* x = amps + int64_t(g) * PTAR_BURST_GROUP * nreal * P * 2 + (r * P + a) * 2 * jg + 2 * (j - g * PTAR_BURST_GROUP);
    const double x0 = x[0], x1 = x[1];
    const double v = __dmul_rn(0.5, __fma_rn(x1, x1, __dmul_rn(x0, x0)));
    if (maps) maps[q * J + j] = v;
    if (bm.seen[int64_t(a) * J + j] && (bj < 0 || fe_better(v, j, best, bj))) {
      best = v;
      bj = j;
      bx0 = x0;
      bx1 = x1;
    }
  }
  Bt_max[q] = best;
  argmax[q] = bj;
  fap[q] = bj < 0 ? NAN : exp(-best);
  if (amp) {
    if (bj < 0) {
      amp[2 * q] = amp[2 * q + 1] = NAN;
    } else {
      const double* l = bm.Lf + (int64_t(bj) * P + a) * 3;
      const double b1 = bx1 / l[2];
      amp[2 * q] = (bx0 - l[1] * b1) / l[0];
      amp[2 * q + 1] = b1;
    }
  }
}

}  // namespace ptar

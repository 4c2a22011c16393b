// Burst-with-memory search over epoch x sky (ptar_bwm_sky, ptar_bwm_combine): per-realization maps of the coherent
// (Earth-term) statistic of a memory ramp, reduced on the device to their maxima, and the pulsar-term statistic, from
// the amplitudes X^ that ptar_fp_project wrote on the whitened ramp basis.
//
// The noise-model work is realization-independent and done once on the host (engine.PulsarBatch._plan_bwm): per pulsar a
// and burst epoch t0 the ramp u = (t - t0) [t >= t0], its Fisher information m_a(t0) = u^T P_a^-1 u, the whitened ramp
// C~_a(t0) = P_a^-1 u / sqrt(m_a(t0)) (the columns ptar_fp_project reduces the rows on, column j = epoch j), the Earth-term
// antenna patterns e_a(s) = (F+, Fx) and, per (t0, s), the inverse Cholesky factor L2^-1 of
// M2(t0, s) = sum_a e_a e_a^T m_a(t0).  Per realization r, epoch t and sky point s:
//   N2[(r, t)][(s, pol)] = sum_a sqrt(m_a(t)) X^[r][a][t] e_a(s)[pol]       fp64 GEMM, K = pulsars
//   B = 1/2 |L2^-1 N2|^2,  t0max[r][t] = max_s B,  t0argmax[r][t] = the first s attaining it
//
// bwm_sky: one CTA per (32 realizations, epoch pair 2q, 2q + 1) runs the staged mainloop of fe_sky_kernel
// (sky_mainloop, csrc/ptar_fe.cuh) with the two GEMM row halves c = 0, 1 holding the two epochs of the pair, each entry
// sqrt(m_a(t)) X^ formed with one multiply while it is staged; each stage carries beside its antenna block the 2 x 3
// packed L2^-1 of the pair at its 32 sky points.  The DMMA fragments put (s, +) and (s, x) of both epochs in one
// thread, whose epilogue forms the two 1/2 |L2^-1 N2|^2 and keeps a running (max, first argmax) per epoch.  With `maps`
// only B is written.  Per thread the sky order is increasing and the (max, lowest index) combine is exact and
// order-free, so every output depends on the realization's amplitudes only.  No atomics anywhere.
//
// bwm_combine: one thread per realization takes the maximum over epochs (lower epoch first on ties) and re-forms N2 at
// the argmax cell in pulsar order to give b^ = M2^-1 N2 = L2^-T L2^-1 N2, the strain |b^| and the polarisation angle
// 1/2 atan2(b^_x, b^_+) mod pi; one thread per (realization, pulsar) takes the pulsar term 1/2 X^2 over the epochs
// the pulsar sees, its slope X^ / sqrt(m) and erfc(sqrt(max)).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_fe.cuh"

namespace ptar {

constexpr int BWM_LINV = 6;               // packed L2^-1 (00, 10, 11) of the two epochs of a pair
constexpr int BWM_COMBINE_THREADS = 256;
static_assert(sky_smem_bytes(PTAR_FE_MAX_PSR, BWM_LINV) <= 227 * 1024, "the BWM tile must fit one SM's shared memory");

__global__ void __launch_bounds__(FE_THREADS, 1) bwm_sky_kernel(const double* __restrict__ amps, int nreal,
                                                                ptar_bwm_model bw, double* __restrict__ t0max,
                                                                int64_t* __restrict__ t0argmax, double* __restrict__ maps) {
  __shared__ double red_v[2][2][FE_RB];
  __shared__ int red_i[2][2][FE_RB];
  const int P = bw.n_psr, T = bw.n_t0;
  const int q = blockIdx.y, r0 = blockIdx.x * FE_RB, nrow = min(FE_RB, nreal - r0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wn = warp >> 2, fk = lane & 3, row = (warp & 3) * 8 + (lane >> 2);
  const int64_t nc = 2 * int64_t((T + 1) >> 1);
  const bool odd = 2 * q + 1 < T;                         // the pair's second epoch exists
  double best0 = -INFINITY, best1 = -INFINITY;
  int bidx0 = 0x7fffffff, bidx1 = 0x7fffffff;
  // rows c: sqrt(m_a(2q + c)) X^[r][a][2q + c]; zero past nreal and n_psr (and for an unseen or absent epoch: sqm = 0)
  auto form = [&](int m, int a, double& n0, double& n1) {
    if (m < nrow && a < P) {
      const double2 x = *reinterpret_cast<const double2*>(amps + (int64_t(r0 + m) * P + a) * nc + 2 * q);
      const double2 w = *reinterpret_cast<const double2*>(bw.sqm + (int64_t(q) * P + a) * 2);
      n0 = __dmul_rn(w.x, x.x);
      n1 = __dmul_rn(w.y, x.y);
    }
  };
  auto epi = [&](int sky, const double* L, double v0, double v1, double v2, double v3) {
    const double y0 = __dmul_rn(L[0], v0), y1 = __fma_rn(L[1], v0, __dmul_rn(L[2], v2));
    const double z0 = __dmul_rn(L[3], v1), z1 = __fma_rn(L[4], v1, __dmul_rn(L[5], v3));
    const double b0 = __dmul_rn(0.5, __fma_rn(y1, y1, __dmul_rn(y0, y0)));
    const double b1 = __dmul_rn(0.5, __fma_rn(z1, z1, __dmul_rn(z0, z0)));
    if (sky < bw.n_sky) {
      if (fe_better(b0, sky, best0, bidx0)) {
        best0 = b0;
        bidx0 = sky;
      }
      if (fe_better(b1, sky, best1, bidx1)) {
        best1 = b1;
        bidx1 = sky;
      }
      if (maps && row < nrow) {
        double* mp = maps + (int64_t(r0 + row) * T + 2 * q) * bw.n_sky + sky;
        mp[0] = b0;
        if (odd) mp[bw.n_sky] = b1;
      }
    }
  };
  sky_mainloop<BWM_LINV>(bw.ant, bw.linv, bw.kp, bw.n_sb, q, form, epi);
  // (max, first argmax) per epoch over the threads of a realization: the quad (fk), then the two column halves (wn)
#pragma unroll
  for (int o = 1; o < 4; o <<= 1) {
    const double ov0 = __shfl_xor_sync(0xffffffffu, best0, o), ov1 = __shfl_xor_sync(0xffffffffu, best1, o);
    const int oi0 = __shfl_xor_sync(0xffffffffu, bidx0, o), oi1 = __shfl_xor_sync(0xffffffffu, bidx1, o);
    if (fe_better(ov0, oi0, best0, bidx0)) {
      best0 = ov0;
      bidx0 = oi0;
    }
    if (fe_better(ov1, oi1, best1, bidx1)) {
      best1 = ov1;
      bidx1 = oi1;
    }
  }
  if (fk == 0) {
    red_v[0][wn][row] = best0;
    red_i[0][wn][row] = bidx0;
    red_v[1][wn][row] = best1;
    red_i[1][wn][row] = bidx1;
  }
  __syncthreads();
  if (tid < 2 * FE_RB) {
    const int c = tid / FE_RB, m = tid % FE_RB, t = 2 * q + c;
    if (m < nrow && t < T) {
      double v = red_v[c][0][m];
      int i = red_i[c][0][m];
      if (fe_better(red_v[c][1][m], red_i[c][1][m], v, i)) {
        v = red_v[c][1][m];
        i = red_i[c][1][m];
      }
      t0max[int64_t(r0 + m) * T + t] = v;
      t0argmax[int64_t(r0 + m) * T + t] = i;
    }
  }
}

// sqrt(m_a(t)) of the pair layout [ceil(T / 2)][n_psr][2]
__device__ __forceinline__ double bwm_sqm(const ptar_bwm_model& bw, int a, int t) {
  return bw.sqm[(int64_t(t >> 1) * bw.n_psr + a) * 2 + (t & 1)];
}

// One thread per realization: the maximum over epochs in epoch order (ties to the lower epoch) and its sky index, then
// b^ at that cell.  N2 is re-formed in pulsar order (2 P multiply-adds); y = L2^-1 N2, b^ = L2^-T y.
__global__ void __launch_bounds__(BWM_COMBINE_THREADS) bwm_combine_kernel(
    const double* __restrict__ amps, const double* __restrict__ t0max, const int64_t* __restrict__ t0argmax, int nreal,
    ptar_bwm_model bw, double* __restrict__ bwm_max, int64_t* __restrict__ argmax_t0, int64_t* __restrict__ argmax_sky,
    double* __restrict__ strain, double* __restrict__ pol, double* __restrict__ fap) {
  const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= nreal) return;
  const int T = bw.n_t0, P = bw.n_psr;
  const int64_t nc = 2 * int64_t((T + 1) >> 1);
  const double* v = t0max + r * T;
  double best = v[0];
  int bt = 0;
  for (int t = 1; t < T; ++t)
    if (fe_better(v[t], t, best, bt)) {
      best = v[t];
      bt = t;
    }
  const int64_t s = t0argmax[r * T + bt];
  bwm_max[r] = best;
  argmax_t0[r] = bt;
  argmax_sky[r] = s;
  fap[r] = exp(-best);
  double np = 0.0, nx = 0.0;
  if (s >= 0 && s < bw.n_sky) {
    for (int a = 0; a < P; ++a) {
      const double w = __dmul_rn(bwm_sqm(bw, a, bt), amps[(r * P + a) * nc + bt]);
      const double* e = bw.antenna + (int64_t(a) * bw.n_sky + s) * 2;
      np = __fma_rn(e[0], w, np);
      nx = __fma_rn(e[1], w, nx);
    }
  }
  const int64_t sp = s >= 0 && s < bw.n_sky ? s : 0;
  const double* L = bw.linv + ((int64_t(bt >> 1) * bw.n_sb * FE_SB) + sp) * BWM_LINV + 3 * (bt & 1);
  const double y0 = __dmul_rn(L[0], np), y1 = __fma_rn(L[1], np, __dmul_rn(L[2], nx));
  const double bx = __dmul_rn(L[2], y1), bp = __fma_rn(L[0], y0, __dmul_rn(L[1], y1));
  strain[r] = hypot(bp, bx);
  double psi = 0.5 * atan2(bx, bp);
  if (psi < 0.0) psi += M_PI;
  if (psi >= M_PI) psi -= M_PI;
  pol[r] = psi;
}

// One thread per (realization, pulsar): Bp = 1/2 X^2 over the epochs the pulsar sees, in epoch order (ties to the
// lower epoch, the first NaN above every number); slope = X^ / sqrt(m) there, fap = erfc(sqrt(max)).  A pulsar that sees
// no epoch gets -inf, index -1 and NaN slope and fap.
__global__ void __launch_bounds__(BWM_COMBINE_THREADS) bwm_psr_kernel(const double* __restrict__ amps, int nreal,
                                                                      ptar_bwm_model bw, double* __restrict__ psr_max,
                                                                      int64_t* __restrict__ psr_argmax,
                                                                      double* __restrict__ slope,
                                                                      double* __restrict__ psr_fap) {
  const int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int P = bw.n_psr, T = bw.n_t0;
  if (e >= int64_t(nreal) * P) return;
  const int a = static_cast<int>(e % P);
  const int64_t nc = 2 * int64_t((T + 1) >> 1);
  const double* x = amps + e * nc;
  const uint8_t* seen = bw.seen + int64_t(a) * T;
  double best = -INFINITY;
  int bt = 0x7fffffff;
  for (int t = 0; t < T; ++t) {
    if (!seen[t]) continue;
    const double v = __dmul_rn(0.5, __dmul_rn(x[t], x[t]));
    if (fe_better(v, t, best, bt)) {
      best = v;
      bt = t;
    }
  }
  psr_max[e] = best;
  if (bt == 0x7fffffff) {
    psr_argmax[e] = -1;
    slope[e] = NAN;
    psr_fap[e] = NAN;
    return;
  }
  psr_argmax[e] = bt;
  slope[e] = x[bt] / bwm_sqm(bw, a, bt);
  psr_fap[e] = erfc(sqrt(best));
}

}  // namespace ptar

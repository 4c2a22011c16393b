// Timing-model projection (ptar_timing_project): post-fit residuals r' = r - W^{-1/2} Q (Q^T W^{1/2} r) per pulsar,
// Q = the orthonormal factor of the whitened design matrix (host QR, engine.PulsarBatch.set_timing_model).
//
// Two kernels over a tile list (<= 1024 time-sorted TOAs of one pulsar per tile), grid = (realization blocks, tiles),
// realization block fastest so the CTAs that share a tile's Q rows run back to back and find them in L2:
//   reduce  partial[t][r][j] = sum_{i in tile t} Q_ij (sqrtw_i r_i)
//   apply   c[r][j] = sum_{tiles t of the pulsar, in order} partial[t][r][j];  r_i -= (sum_j Q_ij c[r][j]) / sqrtw_i
// Thread layout (both kernels): lane = TOA index mod 32, warp = ROWS consecutive realizations; every Q value a thread
// loads serves its ROWS realizations, every Q line a warp loads serves the CTA's 8 warps from L1.  A (realization,
// column) sum is accumulated by one lane over its TOAs i = lane, lane + 32, ... in order and then added across the 32
// lanes by a fixed xor butterfly, so its value depends on the tile and the row's data only -- not on which slot of
// which realization block the row landed in, nor on nreal, chunking or real0.  No atomics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ptar.h"

namespace ptar {

// 8 warps per CTA; realizations per CTA = 8 * ROWS (16 for k <= 16).  Measured on ng15-full (k <= 12, H100): 2 rows per
// warp beat 4 rows (216 registers, one CTA per SM) by 18 %, and 16-warp CTAs at <= 128 registers were slower still.
constexpr int TM_THREADS = 256;
constexpr int TM_WARPS = TM_THREADS / 32;

// realizations per warp for a column bucket KC (KC * ROWS fp64 accumulators per thread)
template <int KC>
struct TmRows {
  static constexpr int v = KC <= 8 ? 4 : 2;
};

template <int KC>
__host__ __device__ constexpr int tm_rb() { return TM_WARPS * TmRows<KC>::v; }

template <int KC>
__global__ void __launch_bounds__(TM_THREADS) timing_reduce_kernel(const double* __restrict__ out, int64_t ld, int nreal,
                                                                   ptar_timing_model tm, double* __restrict__ partial) {
  constexpr int ROWS = TmRows<KC>::v;
  const ptar_tile tile = tm.tiles[blockIdx.y];
  const int p = tile.psr;
  const int k = tm.k[p], n = tile.n_toa, np = tm.seg_len[p];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r0 = blockIdx.x * tm_rb<KC>() + warp * ROWS;
  if (r0 >= nreal) return;
  const double* __restrict__ q = tm.Q + tm.q_off[p] + tile.toa_local0;
  const double* __restrict__ sw = tm.sqrtw + tile.toa_start;
  const double* x = out + int64_t(r0) * ld + tile.toa_start;
  double acc[ROWS][KC];
#pragma unroll
  for (int a = 0; a < ROWS; ++a)
#pragma unroll
    for (int j = 0; j < KC; ++j) acc[a][j] = 0.0;
  for (int i = lane; i < n; i += 32) {
    const double s = __ldg(sw + i);
    double xs[ROWS];
#pragma unroll
    for (int a = 0; a < ROWS; ++a) xs[a] = r0 + a < nreal ? __dmul_rn(x[int64_t(a) * ld + i], s) : 0.0;
#pragma unroll
    for (int j = 0; j < KC; ++j) {
      if (j < k) {
        const double u = __ldg(q + int64_t(j) * np + i);
#pragma unroll
        for (int a = 0; a < ROWS; ++a) acc[a][j] = fma(u, xs[a], acc[a][j]);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < ROWS; ++a)
#pragma unroll
    for (int j = 0; j < KC; ++j)
      if (j < k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[a][j] = __dadd_rn(acc[a][j], __shfl_xor_sync(0xffffffffu, acc[a][j], o));
      }
  if (lane == 0) {
#pragma unroll
    for (int a = 0; a < ROWS; ++a) {
      if (r0 + a >= nreal) break;
      double* dst = partial + (int64_t(blockIdx.y) * nreal + r0 + a) * tm.kmax;
#pragma unroll
      for (int j = 0; j < KC; ++j)
        if (j < k) dst[j] = acc[a][j];
    }
  }
}

template <int KC>
__global__ void __launch_bounds__(TM_THREADS) timing_apply_kernel(double* __restrict__ out, int64_t ld, int nreal,
                                                                  ptar_timing_model tm, const double* __restrict__ partial) {
  constexpr int ROWS = TmRows<KC>::v;
  constexpr int RB = tm_rb<KC>();
  __shared__ double cs[RB][KC];
  const ptar_tile tile = tm.tiles[blockIdx.y];
  const int p = tile.psr;
  const int k = tm.k[p], n = tile.n_toa, np = tm.seg_len[p];
  const int t0 = tm.tile0[p], nt = tm.n_tile[p];
  const int rb0 = blockIdx.x * RB;
  // c[r][j]: the pulsar's tile partials, added in tile order
  for (int e = threadIdx.x; e < RB * KC; e += TM_THREADS) {
    const int rl = e / KC, j = e % KC, r = rb0 + rl;
    double c = 0.0;
    if (j < k && r < nreal)
      for (int t = 0; t < nt; ++t) c = __dadd_rn(c, partial[(int64_t(t0 + t) * nreal + r) * tm.kmax + j]);
    cs[rl][j] = c;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r0 = rb0 + warp * ROWS;
  if (r0 >= nreal) return;
  double c[ROWS][KC];
#pragma unroll
  for (int a = 0; a < ROWS; ++a)
#pragma unroll
    for (int j = 0; j < KC; ++j) c[a][j] = cs[warp * ROWS + a][j];
  const double* __restrict__ q = tm.Q + tm.q_off[p] + tile.toa_local0;
  const double* __restrict__ sw = tm.sqrtw + tile.toa_start;
  double* y = out + int64_t(r0) * ld + tile.toa_start;
  for (int i = lane; i < n; i += 32) {
    const double inv = __ddiv_rn(1.0, __ldg(sw + i));
    double d[ROWS];
#pragma unroll
    for (int a = 0; a < ROWS; ++a) d[a] = 0.0;
#pragma unroll
    for (int j = 0; j < KC; ++j) {
      if (j < k) {
        const double u = __ldg(q + int64_t(j) * np + i);
#pragma unroll
        for (int a = 0; a < ROWS; ++a) d[a] = fma(u, c[a][j], d[a]);
      }
    }
#pragma unroll
    for (int a = 0; a < ROWS; ++a)
      if (r0 + a < nreal) y[int64_t(a) * ld + i] = __dsub_rn(y[int64_t(a) * ld + i], __dmul_rn(d[a], inv));
  }
}

}  // namespace ptar

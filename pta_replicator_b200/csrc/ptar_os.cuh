// Optimal statistic (ptar_os_project, ptar_os_pairs): per-realization Hellings-Downs (and other template) cross-
// correlations of the pulsars of a batch, from rows the generator wrote, without the rows leaving the device.
//
// The noise-model work is realization-independent and done once on the host (engine.PulsarBatch._plan_os):
// C_a = P_a^{-1} F_gw,a (n_a x 2K) on the packed TOA axis, t_ab, the template weights and F^{-1}.  Per realization:
//   os_project  partial[t][r][j] = sum_{i in tile t} C[i][j] row_r[i]      tall-skinny fp64 GEMM, HBM-bound
//   os_sum      X[r][p][j] = sum_{tiles t of pulsar p, in tile order} partial[t][r][j]
//   os_pairs    x = X phi~^{1/2};  d_ab = x_a . x_b;  rho_ab = d_ab / t_ab;  b_o = sum_{a<b} Gamma^o_ab d_ab;
//               A2_o = b_o / D_o;  S/N_o = b_o / sqrt(D_o);  A2_mc = F^{-1} b
//
// os_project: grid = (realization blocks of 64, tiles), realization block fastest, so the CTAs that share a tile's
// C rows run back to back and find them in L2 (C is read at 8 * ncp / 64 = 4 B per output at ncp = 32).  The
// residual rows of a tile are staged 64 TOAs at a time by bulk-async copies (one copy per realization row) into a
// 3-stage mbarrier ring; the products run on DMMA (mma.sync.m8n8k4.f64): M = 64 realizations, N = ncp <= 64 columns,
// K = TOAs.  Warp w owns m-tiles 4 (w & 1) .. +3 and the k-quarter w >> 1 of every 64-TOA chunk; the four
// k-quarters are added in a fixed order at the end.  A partial therefore depends on the tile and the row's data
// only -- not on which slot of which realization block the row landed in, nor on nreal, chunking or real0.  No
// atomics anywhere; os_pairs reduces over pairs with a fixed-shape tree.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ptar.h"

namespace ptar {

constexpr int OS_THREADS = 256;
constexpr int OS_RB = 64;                        // realizations per CTA (8 m-tiles)
constexpr int OS_KC = 64;                        // TOAs per stage
constexpr int OS_XP = OS_KC + 4;                 // smem row pitch (doubles): rows 32 B apart -> conflict-free A gathers
constexpr int OS_STAGES = 3;
constexpr int OS_STAGE_DOUBLES = OS_RB * OS_XP;  // 34,816 B per stage
constexpr size_t OS_SMEM = sizeof(double) * OS_STAGES * OS_STAGE_DOUBLES + 64;   // + barriers: 2 CTAs per SM
// The ring also holds the k-quarter partials red[4][OS_RB][ncp] at the end; past ncp = 32 (NT > 4: the red-noise
// likelihood's bases, up to ncp = 64) they outgrow it, so the barriers move behind them and one CTA runs per SM.
__host__ __device__ constexpr int os_ring_doubles(int nt) {
  return OS_STAGES * OS_STAGE_DOUBLES > 4 * OS_RB * 8 * nt ? OS_STAGES * OS_STAGE_DOUBLES : 4 * OS_RB * 8 * nt;
}
constexpr size_t os_project_smem(int nt) { return sizeof(double) * os_ring_doubles(nt) + 64; }   // == OS_SMEM for nt <= 4
__host__ __device__ constexpr int os_ctas_per_sm(int nt) { return nt <= 4 ? 2 : 1; }
constexpr int OS_PAIR_THREADS = 256;

#define PTAR_OS_DMMA(c0, c1, a, b)                                                                      \
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"          \
               : "+d"(c0), "+d"(c1)                                                                      \
               : "d"(a), "d"(b))

__device__ __forceinline__ uint32_t os_smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void os_mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(os_smem_u32(bar)), "r"(parity)
        : "memory");
  }
}

// The one ranking of every (max, argmax) in the library -- Fp over frequency, Fe over sky and frequency, the radiometer
// over pixels, ln L over the grid: (v, i) ranks above (bv, bi) on a larger value, then on a lower index; NaN ranks above
// every number (the first NaN wins).  A total order on (value, index), so a combine is exact whatever its shape.
__device__ __forceinline__ bool fe_better(double v, int i, double bv, int bi) {
  if (v != v) return !(bv != bv) || i < bi;
  if (bv != bv) return false;
  return v > bv || (v == bv && i < bi);
}

// Warp 0 fills stage `s` with chunk `c` of the tile: one bulk copy of cnt4 doubles per valid realization row.
__device__ __forceinline__ void os_issue_chunk(double* stage, uint64_t* bar, const double* rows, int64_t ld, int64_t base,
                                               int nrow, int cnt4, int lane) {
  const uint32_t bytes = static_cast<uint32_t>(cnt4) * 8u;
  if (lane == 0) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic reads / zero-fills of this stage
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(os_smem_u32(bar)), "r"(bytes * nrow)
                 : "memory");
  }
  __syncwarp();
  for (int m = lane; m < nrow; m += 32)
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     os_smem_u32(stage + m * OS_XP)),
                 "l"(rows + int64_t(m) * ld + base), "r"(bytes), "r"(os_smem_u32(bar))
                 : "memory");
}

template <int NT>   // n-tiles of 8 columns: ncp = 8 NT
__global__ void __launch_bounds__(OS_THREADS, os_ctas_per_sm(NT))
    os_project_kernel(const double* __restrict__ rows, int64_t ld, int nreal, ptar_os_model os,
                      double* __restrict__ partial) {
  extern __shared__ __align__(16) double os_smem[];
  constexpr int NCP = 8 * NT;
  uint64_t* bars = reinterpret_cast<uint64_t*>(os_smem + os_ring_doubles(NT));
  const ptar_tile tile = os.tiles[blockIdx.y];
  const int rb0 = blockIdx.x * OS_RB;
  const int nrow = min(OS_RB, nreal - rb0);
  const int n = tile.n_toa, nch = (n + OS_KC - 1) / OS_KC;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double* rblk = rows + int64_t(rb0) * ld;
  if (tid == 0) {
    for (int s = 0; s < OS_STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(os_smem_u32(bars + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto cnt_of = [&](int c) { return min(OS_KC, n - c * OS_KC); };
  if (warp == 0)
    for (int c = 0; c < OS_STAGES && c < nch; ++c)
      os_issue_chunk(os_smem + c * OS_STAGE_DOUBLES, bars + c, rblk, ld, tile.toa_start + c * OS_KC, nrow, (cnt_of(c) + 3) & ~3, lane);

  const int mh = warp & 1, kq = warp >> 1;
  const int fr = lane >> 2, fk = lane & 3;
  double acc[4][NT][2];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < NT; ++b) acc[a][b][0] = acc[a][b][1] = 0.0;
  const double* __restrict__ Cb = os.C + int64_t(tile.toa_start) * NCP;

  for (int c = 0; c < nch; ++c) {
    const int s = c % OS_STAGES;
    double* xs = os_smem + s * OS_STAGE_DOUBLES;
    const int cnt = cnt_of(c), cnt4 = (cnt + 3) & ~3;
    os_mbar_wait(bars + s, (c / OS_STAGES) & 1);
    if (cnt < cnt4) {   // the pulsar's alignment slots: whatever the rows hold there must not reach the sums
      for (int e = tid; e < OS_RB * 4; e += OS_THREADS) {
        const int m = e >> 2, k = cnt + (e & 3);
        if (k < cnt4) xs[m * OS_XP + k] = 0.0;
      }
      __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int kk = kq * 16 + q * 4;
      if (kk < cnt4) {
        double bf[NT], af[4];
        const double* cr = Cb + int64_t(c * OS_KC + kk + fk) * NCP + fr;
#pragma unroll
        for (int t = 0; t < NT; ++t) bf[t] = __ldg(cr + t * 8);
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) af[mt] = xs[(mh * 32 + mt * 8 + fr) * OS_XP + kk + fk];
#pragma unroll
        for (int mt = 0; mt < 4; ++mt)
#pragma unroll
          for (int t = 0; t < NT; ++t) PTAR_OS_DMMA(acc[mt][t][0], acc[mt][t][1], af[mt], bf[t]);
      }
    }
    __syncthreads();   // every warp is done with stage s
    if (warp == 0 && c + OS_STAGES < nch) {
      const int cn = c + OS_STAGES;
      os_issue_chunk(xs, bars + s, rblk, ld, tile.toa_start + cn * OS_KC, nrow, (cnt_of(cn) + 3) & ~3, lane);
    }
  }
  // k-quarters in a fixed order: red[kq][m][j] (reuses the ring; every copy has landed and been consumed)
  double* red = os_smem;
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      double* d = red + (kq * OS_RB + mh * 32 + mt * 8 + fr) * NCP + t * 8 + 2 * fk;
      d[0] = acc[mt][t][0];
      d[1] = acc[mt][t][1];
    }
  __syncthreads();
  for (int e = tid; e < nrow * NCP; e += OS_THREADS) {
    const int m = e / NCP, j = e % NCP;
    double v = red[m * NCP + j];
#pragma unroll
    for (int q = 1; q < 4; ++q) v = __dadd_rn(v, red[(q * OS_RB + m) * NCP + j]);
    partial[(int64_t(blockIdx.y) * nreal + rb0 + m) * NCP + j] = v;
  }
}

// X[r][p][j] = sum of the tile partials of pulsar p in tile order (one thread per (r, p, j)).
__global__ void os_sum_kernel(const double* __restrict__ partial, int nreal, ptar_os_model os, double* __restrict__ X) {
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int ncp = os.ncp;
  if (idx >= int64_t(nreal) * os.n_psr * ncp) return;
  const int j = static_cast<int>(idx % ncp);
  const int p = static_cast<int>((idx / ncp) % os.n_psr);
  const int64_t r = idx / (int64_t(ncp) * os.n_psr);
  const int t0 = os.tile0[p], nt = os.n_tile[p];
  double v = 0.0;
  for (int t = 0; t < nt; ++t) v = __dadd_rn(v, partial[(int64_t(t0 + t) * nreal + r) * ncp + j]);
  X[idx] = v;
}

// One CTA per realization.  xs[p][j] = X[r][p][j] phi~_j^{1/2} in shared memory; thread `tid` takes the pairs tid,
// tid + 256, ...; per-thread template sums are added by a fixed tree.
__global__ void __launch_bounds__(OS_PAIR_THREADS) os_pairs_kernel(const double* __restrict__ X, int nreal, ptar_os_model os,
                                                                   double* __restrict__ rho, double* __restrict__ a2,
                                                                   double* __restrict__ snr, double* __restrict__ a2_mc) {
  extern __shared__ __align__(16) double os_pair_smem[];
  const int P = os.n_psr, ncp = os.ncp, nc = os.nc, no = os.n_orf, tid = threadIdx.x;
  double* xs = os_pair_smem;                                      // [P][ncp]
  double* red = os_pair_smem + size_t(P) * ncp;                   // [PTAR_OS_MAX_ORF][256]
  const int64_t r = blockIdx.x;
  const double* xr = X + r * P * ncp;
  for (int e = tid; e < P * ncp; e += OS_PAIR_THREADS) xs[e] = __dmul_rn(xr[e], os.sqrt_phi[e % ncp]);
  __syncthreads();
  double bo[PTAR_OS_MAX_ORF] = {0.0, 0.0, 0.0, 0.0};
  for (int q = tid; q < os.n_pairs; q += OS_PAIR_THREADS) {
    const int a = os.pairs[2 * q], b = os.pairs[2 * q + 1];
    const double* xa = xs + a * ncp;
    const double* xb = xs + b * ncp;
    double d = 0.0;
    for (int j = 0; j < nc; ++j) d = fma(xa[j], xb[j], d);
    if (rho) rho[r * os.n_pairs + q] = __ddiv_rn(d, os.t_ab[q]);
#pragma unroll
    for (int o = 0; o < PTAR_OS_MAX_ORF; ++o)
      if (o < no) bo[o] = fma(os.orf[int64_t(o) * os.n_pairs + q], d, bo[o]);
  }
#pragma unroll
  for (int o = 0; o < PTAR_OS_MAX_ORF; ++o) red[o * OS_PAIR_THREADS + tid] = bo[o];
  __syncthreads();
  for (int h = OS_PAIR_THREADS / 2; h > 0; h >>= 1) {
    if (tid < h)
#pragma unroll
      for (int o = 0; o < PTAR_OS_MAX_ORF; ++o)
        red[o * OS_PAIR_THREADS + tid] = __dadd_rn(red[o * OS_PAIR_THREADS + tid], red[o * OS_PAIR_THREADS + tid + h]);
    __syncthreads();
  }
  if (tid < no) {
    const double b = red[tid * OS_PAIR_THREADS];
    a2[r * no + tid] = __ddiv_rn(b, os.dnorm[tid]);
    snr[r * no + tid] = __ddiv_rn(b, os.dsqrt[tid]);
    double m = 0.0;
    for (int o = 0; o < no; ++o) m = fma(os.finv[tid * no + o], red[o * OS_PAIR_THREADS], m);
    a2_mc[r * no + tid] = m;
  }
}

}  // namespace ptar

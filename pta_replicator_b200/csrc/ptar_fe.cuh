// Coherent Fe-statistic over a sky grid (ptar_fe_sky, ptar_fe_combine): per-realization sky maps of the continuous-wave
// statistic (Ellis, Siemens & Creighton 2012), reduced on the device to their maxima, from the amplitudes X^ that
// ptar_fp_project wrote.
//
// The noise-model work is realization-independent and done once on the host (engine.PulsarBatch._plan_fe): L_a(f) of
// the Fp plan's M_a(f), the Earth-term antenna patterns e_a(s) = (F+, Fx) and, per (f, s), the inverse Cholesky factor
// L4^-1 of M4(f, s) = sum_a e_a e_a^T (x) M_a(f).  Per realization r, frequency f and sky point s:
//   N_a(f)    = L_a(f) X^[r][a][f]                                 (= F_f^T P_a^-1 r_a)
//   N4[2p+c]  = sum_a e_a(s)[p] N_a(f)[c]                          fp64 GEMM: rows (f, r, c), K = pulsars, columns (s, p)
//   Fe        = 1/2 |L4^-1 N4|^2,  fmax[r][f] = max_s Fe,  fargmax[r][f] = the first s attaining it
//
// fe_sky: one CTA per (32 realizations, frequency) holds the 64 x kp operand N (rows c = 0 then c = 1 of the same 32
// realizations, pitch kp + 4: conflict-free A gathers) in shared memory for its whole life and walks the sky 32 points
// (64 columns) per stage.  N is formed while it is staged -- three multiplies per element from X^ and L_a(f) -- rather
// than by a launch of its own: the kernel reads X^ once either way, and the fold saves a launch and an Nf x R x 2 kp
// scratch round trip through HBM.  Each stage (the antenna block [kp][64], odd pulsars rotated by 8 so that the four
// k-rows of a B fragment fall on both halves of the banks, plus the 32 x 10 entries of L4^-1) arrives by two bulk-async
// copies into a 2-stage mbarrier ring.  DMMA (mma.sync.m8n8k4.f64): warp w owns realizations 8 (w & 3) .. +7 as the
// m-tile pair (c = 0, c = 1) and columns 32 (w >> 2) .. +31 of the stage, so the four numbers N4 of a cell -- (s, +) and
// (s, x) of both c -- sit in one thread's accumulators; the epilogue forms 1/2 |L4^-1 N4|^2 there and keeps a running
// (max, first argmax) per thread.  The 8 x kp x 64 GEMM product of a stage is never written (with `maps` only Fe is).
// Per thread the sky order is increasing, and the (max, lowest index) combine of the threads that hold a realization is
// exact and order-free, so every output depends on the realization's amplitudes only.  No atomics anywhere.
// The staged mainloop -- ring, barriers, operand staging, fragment gathers and the DMMA loop -- is sky_mainloop, which
// bwm_sky_kernel (csrc/ptar_bwm.cuh) shares: a kernel supplies only its operand former and its per-cell epilogue.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_os.cuh"

namespace ptar {

constexpr int FE_THREADS = 256;
constexpr int FE_RB = 32;                 // realizations per CTA: 64 GEMM rows
constexpr int FE_SB = 32;                 // sky points per stage
constexpr int FE_BN = 2 * FE_SB;          // columns (s, pol) per stage
constexpr int FE_LINV = 10;               // packed lower-triangular L4^-1
constexpr int FE_COMBINE_THREADS = 256;

// A stage of a sky kernel: the antenna block [kp][64] and LINV packed doubles per sky point of the block.
__host__ __device__ constexpr int sky_stage_doubles(int kp, int linv) { return kp * FE_BN + FE_SB * linv; }
// N tile + two stages + two mbarriers
__host__ __device__ constexpr size_t sky_smem_bytes(int kp, int linv) {
  return sizeof(double) * (size_t(2 * FE_RB) * (kp + 4) + 2 * size_t(sky_stage_doubles(kp, linv))) + 64;
}
__host__ __device__ constexpr int fe_stage_doubles(int kp) { return sky_stage_doubles(kp, FE_LINV); }
// 199 KB at kp = 128 (1 CTA per SM), 130 KB at kp = 80
__host__ __device__ constexpr size_t fe_smem_bytes(int kp) { return sky_smem_bytes(kp, FE_LINV); }
static_assert(fe_smem_bytes(PTAR_FE_MAX_PSR) <= 227 * 1024, "the Fe tile must fit one SM's shared memory");
static_assert(PTAR_FE_MAX_PSR % 16 == 0, "kp is a multiple of 16");

// One thread fills stage `st` with sky block `sb`: the antenna block (all kp pulsars x 64 columns) and the LINV packed
// doubles of each of its 32 sky points, row y (this CTA's frequency or epoch pair) of lv [y][32 n_sb][LINV].
template <int LINV>
__device__ __forceinline__ void sky_issue_stage(double* st, uint64_t* bar, const double* ant, const double* lv, int kp, int nsb,
                                                int y, int sb) {
  const uint32_t ab = static_cast<uint32_t>(kp) * FE_BN * 8u, lb = FE_SB * LINV * 8u;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic reads of this stage
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(os_smem_u32(bar)), "r"(ab + lb) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   os_smem_u32(st)),
               "l"(ant + int64_t(sb) * kp * FE_BN), "r"(ab), "r"(os_smem_u32(bar))
               : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   os_smem_u32(st + kp * FE_BN)),
               "l"(lv + (int64_t(y) * nsb + sb) * FE_SB * LINV), "r"(lb), "r"(os_smem_u32(bar))
               : "memory");
}

// The staged mainloop of the sky kernels (fe_sky_kernel, bwm_sky_kernel).  The CTA's 64 x kp operand N is formed
// once by form(m, a, n0, n1) (realization slot m, pulsar a; rows c = 0 and c = 1; both 0 on entry), then the sky is
// walked 32 points per stage through the 2-stage bulk-async ring of antenna blocks `ant` [n_sb][kp][64] and packed
// per-point factors, row y of `lv` [y][32 n_sb][LINV].  After each stage's DMMA loop every thread calls epi(sky, L, v0, v1, v2, v3)
// for its four sky points in increasing order, with L the point's LINV factors and (v0, v1, v2, v3) = N2 of
// (c = 0, +), (c = 1, +), (c = 0, x), (c = 1, x) for its realization slot row = 8 (warp & 3) + (lane >> 2).
template <int LINV, class Form, class Epi>
__device__ __forceinline__ void sky_mainloop(const double* ant, const double* lv, int kp, int nsb, int y, Form form, Epi epi) {
  extern __shared__ __align__(16) double sky_smem[];
  const int ap = kp + 4;
  const int sd = sky_stage_doubles(kp, LINV);
  double* As = sky_smem;                                  // [c][FE_RB][ap]
  double* ring = sky_smem + 2 * FE_RB * ap;               // 2 x [kp][64] antenna + [32][LINV] factors
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + 2 * sd);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    for (int s = 0; s < 2; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(os_smem_u32(bars + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0)
    for (int s = 0; s < 2 && s < nsb; ++s) sky_issue_stage<LINV>(ring + s * sd, bars + s, ant, lv, kp, nsb, y, s);
  for (int e = tid; e < FE_RB * kp; e += FE_THREADS) {
    const int m = e / kp, a = e - m * kp;
    double n0 = 0.0, n1 = 0.0;
    form(m, a, n0, n1);
    As[m * ap + a] = n0;
    As[(FE_RB + m) * ap + a] = n1;
  }
  __syncthreads();

  const int wm = warp & 3, wn = warp >> 2, fr = lane >> 2, fk = lane & 3;
  const int row = wm * 8 + fr;                            // realization slot of this thread's accumulator rows
  const double* a0 = As + row * ap + fk;                  // c = 0
  const double* a1 = As + (FE_RB + row) * ap + fk;        // c = 1
  for (int sb = 0; sb < nsb; ++sb) {
    const int s = sb & 1;
    double* bs = ring + s * sd;
    const double* li = bs + kp * FE_BN;
    os_mbar_wait(bars + s, (sb >> 1) & 1);
    double acc[2][4][2];
#pragma unroll
    for (int t = 0; t < 4; ++t) acc[0][t][0] = acc[0][t][1] = acc[1][t][0] = acc[1][t][1] = 0.0;
    const int sw = (fk & 1) * 8;                          // the host's rotation of odd pulsars (k-steps start even)
    const double* bcol = bs + fk * FE_BN;
#pragma unroll 4
    for (int k = 0; k < kp; k += 4) {
      const double x0 = a0[k], x1 = a1[k];
      double bf[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) bf[t] = bcol[k * FE_BN + ((wn * 32 + t * 8 + fr + sw) & (FE_BN - 1))];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        PTAR_OS_DMMA(acc[0][t][0], acc[0][t][1], x0, bf[t]);
        PTAR_OS_DMMA(acc[1][t][0], acc[1][t][1], x1, bf[t]);
      }
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int sl = wn * 16 + t * 4 + fk;               // columns 2 sl (+), 2 sl + 1 (x) of the stage
      epi(sb * FE_SB + sl, li + sl * LINV, acc[0][t][0], acc[1][t][0], acc[0][t][1], acc[1][t][1]);
    }
    __syncthreads();   // every warp is done with stage s
    if (tid == 0 && sb + 2 < nsb) sky_issue_stage<LINV>(bs, bars + s, ant, lv, kp, nsb, y, sb + 2);
  }
}

__global__ void __launch_bounds__(FE_THREADS, 1) fe_sky_kernel(const double* __restrict__ amps, int nreal, ptar_fe_model fe,
                                                               double* __restrict__ fmax, int64_t* __restrict__ fargmax,
                                                               double* __restrict__ maps) {
  __shared__ double red_v[2][FE_RB];
  __shared__ int red_i[2][FE_RB];
  const int P = fe.n_psr;
  const int f = blockIdx.y, r0 = blockIdx.x * FE_RB, nrow = min(FE_RB, nreal - r0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wn = warp >> 2, fk = lane & 3, row = (warp & 3) * 8 + (lane >> 2);
  const int64_t nc = 2 * int64_t(fe.n_freq);
  double best = -INFINITY;
  int bidx = 0x7fffffff;
  // N = L_a(f) X^ of this CTA's realizations at frequency f; zero past nreal and n_psr
  auto form = [&](int m, int a, double& n0, double& n1) {
    if (m < nrow && a < P) {
      const double2 x = *reinterpret_cast<const double2*>(amps + (int64_t(r0 + m) * P + a) * nc + 2 * f);
      const double* l = fe.Lf + (int64_t(f) * P + a) * 3;
      n0 = __dmul_rn(l[0], x.x);
      n1 = __fma_rn(l[1], x.x, __dmul_rn(l[2], x.y));
    }
  };
  auto epi = [&](int sky, const double* L, double v0, double v1, double v2, double v3) {
    const double y0 = __dmul_rn(L[0], v0);
    const double y1 = __fma_rn(L[1], v0, __dmul_rn(L[2], v1));
    const double y2 = __fma_rn(L[3], v0, __fma_rn(L[4], v1, __dmul_rn(L[5], v2)));
    const double y3 = __fma_rn(L[6], v0, __fma_rn(L[7], v1, __fma_rn(L[8], v2, __dmul_rn(L[9], v3))));
    const double v = __dmul_rn(0.5, __fma_rn(y3, y3, __fma_rn(y2, y2, __fma_rn(y1, y1, __dmul_rn(y0, y0)))));
    if (sky < fe.n_sky) {
      if (fe_better(v, sky, best, bidx)) {
        best = v;
        bidx = sky;
      }
      if (maps && row < nrow) maps[(int64_t(r0 + row) * fe.n_freq + f) * fe.n_sky + sky] = v;
    }
  };
  sky_mainloop<FE_LINV>(fe.ant, fe.linv, fe.kp, fe.n_sb, f, form, epi);
  // (max, first argmax) over the threads of a realization: the quad (fk), then the two column halves (wn)
#pragma unroll
  for (int o = 1; o < 4; o <<= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
    if (fe_better(ov, oi, best, bidx)) {
      best = ov;
      bidx = oi;
    }
  }
  if (fk == 0) {
    red_v[wn][row] = best;
    red_i[wn][row] = bidx;
  }
  __syncthreads();
  if (tid < nrow) {
    double v = red_v[0][tid];
    int i = red_i[0][tid];
    if (fe_better(red_v[1][tid], red_i[1][tid], v, i)) {
      v = red_v[1][tid];
      i = red_i[1][tid];
    }
    fmax[int64_t(r0 + tid) * fe.n_freq + f] = v;
    fargmax[int64_t(r0 + tid) * fe.n_freq + f] = i;
  }
}

// One thread per realization: the maximum over frequency in frequency order (ties to the lower f) and its sky index.
__global__ void __launch_bounds__(FE_COMBINE_THREADS) fe_combine_kernel(const double* __restrict__ fmax,
                                                                        const int64_t* __restrict__ fargmax, int nreal,
                                                                        int nf, double* __restrict__ fe_max,
                                                                        int64_t* __restrict__ argmax_f,
                                                                        int64_t* __restrict__ argmax_sky) {
  const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= nreal) return;
  const double* v = fmax + r * nf;
  double best = v[0];
  int bi = 0;
  for (int f = 1; f < nf; ++f)
    if (fe_better(v[f], f, best, bi)) {
      best = v[f];
      bi = f;
    }
  fe_max[r] = best;
  argmax_f[r] = bi;
  argmax_sky[r] = fargmax[r * nf + bi];
}

}  // namespace ptar

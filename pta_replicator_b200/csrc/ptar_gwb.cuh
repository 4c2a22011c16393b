// GWB stage kernels (red_noise.py:235-285) and the small dense Cholesky.
//
// The reference colours complex white draws with the Cholesky factor of the ORF, scales by
// sqrt(C(f)), Hermitian-packs, inverse-FFTs (length 2Nf-2 = 2 x prime) and keeps npts samples.
// All of that is ONE real linear map per pulsar row:  grid = A . z  with
//   parity mode      A = T  [npts x 2(Nf-2)]  (pruned inverse DFT x sqrt(C)/dt; z = the
//                    reference's own draws, so results match the reference to fp64 rounding)
//   throughput mode  A = L  [npts x npts] lower triangular with L L^T = T T^T (same Gaussian
//                    law from npts instead of 2(Nf-2) draws per pulsar; 10-20x fewer flops)
// and the ORF mixing M commutes with it, so it is applied to the draws first (ptar_gwb_mix).
// Only the grid knots next to a pulsar's TOAs are ever interpolated, so the synthesis evaluates,
// per pulsar, just that sorted subset of rows of A ("knots"; ~60 % of them on ng15-shaped data).
//
// Both GEMMs of the parity mode run on the fp64 tensor path, mma.sync.m8n8k4.f64 (SASS DMMA.8x8x4); the
// throughput-mode synthesis runs on the int8 tensor cores (ptar_gwb_i8.cuh).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_rng.cuh"

namespace ptar {

#define PTAR_DMMA(c0, c1, a, b)                                                                         \
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"          \
               : "+d"(c0), "+d"(c1)                                                                      \
               : "d"(a), "d"(b))

// ---------------------------------------------------------------------------------------
// ORF mixing: Zm[p][r][j] = sum_{q<=p} M[p][q] z[r][q][j]   (output pulsar-major).
// Persistent: each CTA stages the lower triangle of M once in shared memory, then loops over the work items
// blockIdx.x, blockIdx.x + gridDim.x, ... = (32 grid columns, one Philox group of 4 realizations), the column
// block fastest.  The grid is the resident-CTA count (2 per SM at 67 pulsars), so one CTA's draws run under the
// other's MMAs.  Per item: 128 rows (row = l*32 + jj), D[row][p] = sum_q z[q][row] * M[p][q]; K = q padded to a
// multiple of 4, N = p padded to a multiple of 8.  zs[q][row] has row stride 132 and ms[p][q] row stride KP+4 ->
// conflict-free 8x4 fragment gathers.  Warp w owns rows 16w..16w+15 (2 m-tiles) and all n-tiles; k-steps above the
// diagonal are skipped.
constexpr int MIX_JT = 32, MX_ROWS = 128, MX_ZS = MX_ROWS + 4;

// SLICE = true (throughput mode with the int8 tensor-core synthesis, n_psr <= 72): instead of fp64 Zm the kernel emits the
// six signed radix-256 digit slices of Zm[p][r][j] / zscale[p] in the tensor core's K-major core-matrix tile layout
// (ptar_gwb_i8.cuh: ZS[slice][p][r-block][k-chunk of 32][16][2][8][16]).  The accumulators of all n-tiles stay in registers,
// the digits are staged through the shared memory the draws occupied and leave as 16-byte stores.  Digit
// extraction: m = fma(v, 2^48 / zscale, 1.5 * 2^52) holds round(v 2^48 / zscale) in its low mantissa bits; adding
// 0x80 to every byte position turns the balanced digits d in [-128, 127] into the plain bytes d + 128 of that integer.
constexpr int MX_MAXNT = 9;                    // n-tiles kept in registers by the SLICE build (n_psr <= 72)
constexpr int MX_DSTRIDE = 6 * 2 * 4 * 16 + 16;  // bytes per pulsar in the digit staging area (+16: bank skew)

template <bool INJECT, bool SLICE>
__global__ void __launch_bounds__(256, 2) gwb_mix_dmma_kernel(double* __restrict__ Zm, const double* __restrict__ M,
                                                               const double* __restrict__ zin, int P, int J,
                                                               int64_t nreal, const PhiloxKeys K, int64_t real0,
                                                               int8_t* __restrict__ ZS, const double* __restrict__ zinv,
                                                               int Jpad, int64_t rcap) {
  extern __shared__ __align__(16) double mx_smem[];
  const int KP = (P + 3) & ~3, NP = (P + 7) & ~7, MS = KP + 4;
  double* zs = mx_smem;                       // [KP][132]
  double* ms = mx_smem + size_t(KP) * MX_ZS;  // [NP][MS]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int p = tid >> 5; p < NP; p += 8) {      // warp per row of M: no integer division by the run-time pitch
    for (int q = tid & 31; q < MS; q += 32) ms[p * MS + q] = (p < P && q <= p) ? __ldg(M + size_t(p) * P + q) : 0.0;
  }
  const int fr = lane >> 2, fk = lane & 3;
  const int row0 = warp * 16;
  const int n_nt = NP / 8;
  const int n_jb = (J + MIX_JT - 1) / MIX_JT;
  const int64_t n_items = int64_t(n_jb) * ((nreal + 3) / 4);
  for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int j0 = static_cast<int>(item % n_jb) * MIX_JT;
    const int64_t rbase = (item / n_jb) * 4;
    __syncthreads();  // the previous item's draws and digits are consumed (and ms is visible)
    // unrolled: independent Philox chains interleave (each thread draws ~9 of them per item, a long dependent chain each)
#pragma unroll 3
    for (int idx = tid; idx < KP * MIX_JT; idx += 256) {
      const int q = idx / MIX_JT, jj = idx % MIX_JT, j = j0 + jj;
      double z[4] = {0, 0, 0, 0};
      if (q < P && j < J) {
        if (INJECT) {
#pragma unroll
          for (int l = 0; l < 4; ++l)
            if (rbase + l < nreal) z[l] = zin[((rbase + l) * P + q) * J + j];
        } else {
          float n[4];
          normals4(n, j, PTAR_K_GWB, q, static_cast<uint64_t>(real0 + rbase) >> 2, K);
#pragma unroll
          for (int l = 0; l < 4; ++l) z[l] = static_cast<double>(n[l]);
        }
      }
#pragma unroll
      for (int l = 0; l < 4; ++l) zs[size_t(q) * MX_ZS + l * MIX_JT + jj] = z[l];
    }
    __syncthreads();
    double keep[SLICE ? MX_MAXNT : 1][2][2];
#pragma unroll
    for (int nt = 0; nt < (SLICE ? MX_MAXNT : 16); ++nt) {
      if (nt >= n_nt) break;
      double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
      const int kmax = min(KP, (nt * 8 + 8 + 3) & ~3);  // q <= p < nt*8+8
#pragma unroll 4
      for (int k0 = 0; k0 < kmax; k0 += 4) {
        const double b = ms[(nt * 8 + fr) * MS + k0 + fk];
        const double a0 = zs[size_t(k0 + fk) * MX_ZS + row0 + fr];
        const double a1 = zs[size_t(k0 + fk) * MX_ZS + row0 + 8 + fr];
        PTAR_DMMA(acc[0][0], acc[0][1], a0, b);
        PTAR_DMMA(acc[1][0], acc[1][1], a1, b);
      }
      if (SLICE) {
        keep[nt][0][0] = acc[0][0]; keep[nt][0][1] = acc[0][1]; keep[nt][1][0] = acc[1][0]; keep[nt][1][1] = acc[1][1];
      } else {
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int row = row0 + t * 8 + fr;
          const int l = row >> 5, jj = row & 31, j = j0 + jj;
          if (j < J && rbase + l < nreal) {
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int p = nt * 8 + 2 * fk + u;
              if (p < P) Zm[(size_t(p) * nreal + (rbase + l)) * J + j] = acc[t][u];
            }
          }
        }
      }
    }
    if (SLICE) {
      __syncthreads();                                   // every warp is done reading the draws
      unsigned char* ds = reinterpret_cast<unsigned char*>(zs);   // [p][slice][c][l][16] (+ skew)
#pragma unroll
      for (int nt = 0; nt < MX_MAXNT; ++nt) {
        if (nt >= n_nt) break;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int row = row0 + t * 8 + fr;
          const int l = row >> 5, jj = row & 31;
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int p = nt * 8 + 2 * fk + u;
            if (p < P) {
              const double m = fma(keep[nt][t][u], __ldg(zinv + p), 6755399441055744.0);   // 1.5 * 2^52
              // low 48 bits of the mantissa = round(v * zinv) in two's complement; + 0x80 per byte -> bytes d + 128
              const unsigned long long xb = static_cast<unsigned long long>(__double_as_longlong(m)) + 0x0000808080808080ull;
              const uint32_t lo = static_cast<uint32_t>(xb) ^ 0x80808080u;            // digits of slices 5, 4, 3, 2
              const uint32_t hi = static_cast<uint32_t>(xb >> 32) ^ 0x00008080u;      // digits of slices 1, 0
              unsigned char* d = ds + size_t(p) * MX_DSTRIDE + ((jj >> 4) * 4 + l) * 16 + (jj & 15);
              d[5 * 128] = static_cast<unsigned char>(lo);
              d[4 * 128] = static_cast<unsigned char>(lo >> 8);
              d[3 * 128] = static_cast<unsigned char>(lo >> 16);
              d[2 * 128] = static_cast<unsigned char>(lo >> 24);
              d[1 * 128] = static_cast<unsigned char>(hi);
              d[0 * 128] = static_cast<unsigned char>(hi >> 8);
            }
          }
        }
      }
      __syncthreads();
      // 16-byte pieces: (p, slice, c, l) -> ZS[slice][p][rblk][kch][g][c][r8][16] (k-chunks of 32 columns = this CTA's
      // 32 columns); the four rows of a piece are adjacent
      const int64_t n_rblk = rcap / 128, nkch = Jpad / 32;
      const int kch = j0 / 32;
      const int64_t rblk = rbase / 128;
      const int g = static_cast<int>((rbase % 128) / 8), r8 = static_cast<int>(rbase % 8);
      for (int idx = tid; idx < P * 6 * 2 * 4; idx += 256) {
        const int l = idx & 3, c = (idx >> 2) & 1, sl = (idx >> 3) % 6, p = idx / 48;
        const uint4 v = *reinterpret_cast<const uint4*>(ds + size_t(p) * MX_DSTRIDE + ((sl * 2 + c) * 4 + l) * 16);
        if (rbase + l < rcap && j0 + c * 16 < Jpad) {
          int8_t* dst = ZS + ((((size_t(sl) * P + p) * n_rblk + rblk) * nkch + kch) * 16 + g) * 256 + (c * 8 + r8 + l) * 16;
          *reinterpret_cast<uint4*>(dst) = v;
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// Synthesis: for pulsar p and its knot subset K_p (sorted rows of A),
//   G[r][g_off[p] + i] = sum_j A[K_p[i]][j] * Zm[p][r][j].
// D = Z * A^T: mma A-operand = Z (row-major, K contiguous), B-operand = rows of A ("col": K contiguous per
// n).  CTA tile 128 realizations x 64 knots, BK = 16, 8 warps as 4 (r) x 2 (n), each a 32 x 32 warp tile =
// 4 x 4 DMMA tiles; operands staged with 16-byte cp.async through a 3-stage ring; rows padded to 20 doubles
// so the 8x4 fragment loads are conflict free.  The host lists the (pulsar, knot-block) tiles heaviest
// first (a lower-triangular A makes k run only to the tile's last knot).
constexpr int DM_BC = 128, DM_BN = 64, DM_BK = 16, DM_S = DM_BK + 4, DM_STAGES = 3;
constexpr size_t DM_SMEM = sizeof(double) * DM_STAGES * (DM_BC + DM_BN) * DM_S;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const int bytes = valid ? 16 : 0;  // src-size 0 => zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(bytes) : "memory");
}

__global__ void __launch_bounds__(256, 2) gwb_synth_dmma_kernel(double* __restrict__ G, int64_t g_ld, int64_t g_ldr,
                                                                 const double* __restrict__ A, int64_t lda,
                                                                 const double* __restrict__ Z, int J, int64_t nreal,
                                                                 const int32_t* __restrict__ tile_list,
                                                                 const int32_t* __restrict__ knots, int lower_tri) {
  extern __shared__ __align__(16) double dm_smem[];
  double* Zs = dm_smem;                                     // [STAGES][128][20]
  double* As = dm_smem + size_t(DM_STAGES) * DM_BC * DM_S;  // [STAGES][64][20]
  __shared__ int s_rows[DM_BN];                              // row of A for each knot of the tile (-1: none)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int32_t* tl = tile_list + size_t(blockIdx.x) * 4;   // {pulsar, first knot (index into knots[]), count, kend}
  const int p = tl[0], kn0 = tl[1], kcnt = tl[2];
  const int kend = lower_tri ? min(J, tl[3]) : J;
  const int64_t r0 = int64_t(blockIdx.y) * DM_BC;
  const int nk = (kend + DM_BK - 1) / DM_BK;
  if (tid < DM_BN) s_rows[tid] = tid < kcnt ? knots[kn0 + tid] : -1;
  __syncthreads();
  const int wc = (warp & 3) * 32, wn = (warp >> 2) * 32;
  const int fr = lane >> 2, fk = lane & 3;
  const double* Zp = Z + size_t(p) * nreal * J;

  auto load_stage = [&](int kt, int st) {
    const int k0 = kt * DM_BK;
#pragma unroll
    for (int i = 0; i < 4; ++i) {  // Z: 128 rows x 8 chunks of 2 doubles
      const int ch = tid + i * 256;
      const int row = ch >> 3, kc = (ch & 7) * 2;
      const int64_t r = r0 + row;
      const bool ok = (r < nreal) && (k0 + kc < J);
      cp_async16(Zs + (size_t(st) * DM_BC + row) * DM_S + kc, Zp + (ok ? size_t(r) * J + k0 + kc : 0), ok);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {  // A: 64 gathered rows x 8 chunks
      const int ch = tid + i * 256;
      const int row = ch >> 3, kc = (ch & 7) * 2;
      const int ar = s_rows[row];
      const bool ok = (ar >= 0) && (k0 + kc < J);
      cp_async16(As + (size_t(st) * DM_BN + row) * DM_S + kc, A + (ok ? size_t(ar) * lda + k0 + kc : 0), ok);
    }
  };

  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int m = 0; m < 4; ++m) acc[i][m][0] = acc[i][m][1] = 0.0;

#pragma unroll
  for (int s = 0; s < DM_STAGES - 1; ++s) {
    if (s < nk) load_stage(s, s);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  for (int kt = 0; kt < nk; ++kt) {
    asm volatile("cp.async.wait_group %0;" ::"n"(DM_STAGES - 2) : "memory");
    __syncthreads();
    {  // prefetch tile kt + STAGES - 1 into the slot freed in the previous iteration
      const int nxt = kt + DM_STAGES - 1;
      if (nxt < nk) load_stage(nxt, nxt % DM_STAGES);
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
    const int st = kt % DM_STAGES;
    const double* zs = Zs + size_t(st) * DM_BC * DM_S;
    const double* as = As + size_t(st) * DM_BN * DM_S;
#pragma unroll
    for (int kk = 0; kk < DM_BK; kk += 4) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = zs[(wc + i * 8 + fr) * DM_S + kk + fk];
#pragma unroll
      for (int m = 0; m < 4; ++m) b[m] = as[(wn + m * 8 + fr) * DM_S + kk + fk];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int m = 0; m < 4; ++m) PTAR_DMMA(acc[i][m][0], acc[i][m][1], a[i], b[m]);
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  // the compact grid shares its column index with knots[] and is column-major: G[kn0 + n][r]; pulsar blocks are padded
  // to even length (pad knots = -1 -> zero rows)
  const int kpad = (kcnt + 1) & ~1;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t r = r0 + wc + i * 8 + fr;
    if (r >= nreal) continue;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int n = wn + m * 8 + 2 * fk;
      if (n < kpad) {
        G[size_t(kn0 + n) * g_ldr + r] = acc[i][m][0];
        G[size_t(kn0 + n + 1) * g_ldr + r] = acc[i][m][1];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// Lower Cholesky, one CTA per matrix, left-looking; every inner product is a warp-shuffle
// reduction (north_star: "warp-shuffle reductions for the small dense Cholesky").
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(256) cholesky_kernel(double* __restrict__ Lall, const double* __restrict__ Aall,
                                                        int n, int* __restrict__ info) {
  double* L = Lall + size_t(blockIdx.x) * n * n;
  const double* A = Aall + size_t(blockIdx.x) * n * n;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  __shared__ double s_diag;
  __shared__ int s_bad;
  if (tid == 0) s_bad = 0;
  for (int idx = tid; idx < n * n; idx += blockDim.x) {
    const int i = idx / n, j = idx % n;
    L[idx] = (j <= i) ? A[idx] : 0.0;
  }
  __syncthreads();
  for (int j = 0; j < n; ++j) {
    if (warp == 0) {
      double s = 0.0;
      for (int k = lane; k < j; k += 32) s = fma(L[size_t(j) * n + k], L[size_t(j) * n + k], s);
      s = warp_sum(s);
      if (lane == 0) {
        const double d = L[size_t(j) * n + j] - s;
        if (!(d > 0.0)) {
          s_bad = j + 1;
          s_diag = 1.0;
        } else {
          s_diag = sqrt(d);
        }
      }
    }
    __syncthreads();
    if (s_bad) break;
    const double ljj = s_diag;
    for (int i = j + 1 + warp; i < n; i += nwarps) {
      double s = 0.0;
      for (int k = lane; k < j; k += 32) s = fma(L[size_t(i) * n + k], L[size_t(j) * n + k], s);
      s = warp_sum(s);
      if (lane == 0) L[size_t(i) * n + j] = (L[size_t(i) * n + j] - s) / ljj;
    }
    if (tid == 0) L[size_t(j) * n + j] = ljj;
    __syncthreads();
  }
  if (tid == 0 && info) info[blockIdx.x] = s_bad;
}

}  // namespace ptar

// GWB synthesis on the Hopper tensor cores (wgmma, int8), throughput mode.
//
//   G[r][q] = sum_j A[knot(q)][j] * Zm[p(q)][r][j]            (red_noise.py:269-285 as one linear map, see ptar_gwb.cuh)
//
// fp64 has no wgmma kind, so the product is evaluated EXACTLY in integers (Ozaki-style error-free splitting):
// both operands are written as fixed-point numbers with six signed radix-256 digits,
//   A[n][j]  = sA[n] * sum_t a_t[n][j] 2^(-8(t+1)),     Zm[p][r][j] = sZ[p] * sum_s z_s[p][r][j] 2^(-8(s+1)),
// (a_t, z_s int8; sA, sZ powers of two chosen so that |value / scale| <= 1/4, i.e. 46-48 significant bits relative
// to the row maximum), every digit-slice product is an int8 x int8 -> int32 GEMM on wgmma.mma_async .s32.s8.s8 --
// exact -- and slice pairs of equal weight s + t = d accumulate into the same int32 registers.  Diagonals d = 0..6
// are kept (26 of the 36 slice pairs; the dropped ones weigh <= 2^-56 of full scale).  The epilogue combines the
// seven int32 accumulators in fp64 (sum_d D_d 2^(-8 d)) and applies the two scales.  Checked against the fp64 DMMA
// kernel on the same input: tests/test_gpu_gwb_i8.py.
//
// Operand staging: the producers write both operands in the tensor core's K-major no-swizzle layout (8 rows x 16
// bytes core matrices), tile by tile, so that one k-chunk of one operand is a single contiguous bulk-async (TMA) copy:
//   ZS  [slice s][pulsar p][r-block of 128][k-chunk of 32 j][16 row groups][2 x 16-byte k][8 rows][16 bytes]   (4 KB per tile)
//   AS  [tile][k-chunk of 32 j][slice t][BN / 8 row groups][2][8][16]                                         (9 KB per copy)
// A CTA copies the contiguous 2 KB half of a Z tile that holds its 64 realizations (row groups 0-7 or 8-15).  One
// m64nBNk32 instruction per slice pair multiplies Z slice s (64 realizations x 32 j) with A slice t (BN knots x 32 j)
// into the BN / 2 accumulator registers of diagonal s + t.  (Stacking the A slices along N into one wide instruction
// per Z slice makes the accumulator ranges of the instructions overlap at different offsets; ptxas then serializes the
// wgmma pipeline.)
//
// CTA = one tile of BN = 48 knots x 64 realizations, 256 threads = two warpgroups that read the same stage and split
// the diagonals: warpgroup 0 owns d = 0, 1, 3, 5 and warpgroup 1 owns d = 2, 4, 6, 13 slice pairs each (4 x 24 and
// 3 x 24 int32 accumulators per thread), so the kernel fits 128 registers and two CTAs share an SM: one CTA's
// prologue and epilogue run under the other's k-loop.  Per 64 x 32 outputs a k-chunk moves 75 KB through shared memory
// (operand reads + the stage), against 93 KB for a 128 x 32 tile whose two warpgroups hold all seven diagonals.  Thread 0
// issues the bulk copies into a 4-stage mbarrier ring (21 KB per stage); a stage is refilled once both warpgroups'
// wgmma groups that read it have retired (one wgmma group stays in flight behind the one being issued).  The epilogue
// swaps half of the accumulators between the warpgroups through the drained ring, so that one thread holds all seven
// diagonals of each output it folds.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ptar {

constexpr int I8_SLICES = 6;          // digits per operand
constexpr int I8_DIAGS = 7;           // kept weights d = s + t = 0 .. 6
constexpr int I8_BM = 128;            // realizations per r-block of ZS (the row tile of the slice producers)
constexpr int I8_CM = 64;             // realizations per CTA: one half of an r-block, the M of one wgmma
constexpr int I8_BN = 48;             // knots per CTA
constexpr int I8_BK = 32;             // j per pipeline stage (bytes, int8) = the K of one wgmma
constexpr int I8_STAGES = 4;          // 84 KB of ring: two CTAs per SM still fit
constexpr int I8_ZT_BYTES = I8_BM * I8_BK;                // one Z-slice tile of ZS: 4 KB
constexpr int I8_A_BYTES = I8_CM * I8_BK;                 // one Z slice of one stage: 2 KB
constexpr int I8_B_BYTES = I8_SLICES * I8_BN * I8_BK;     // all A slices of one stage: 9 KB
constexpr int I8_STAGE_BYTES = I8_SLICES * I8_A_BYTES + I8_B_BYTES;   // 21 KB
constexpr int I8_NACC = I8_BN / 2;                        // int32 accumulators per diagonal and thread (m64nBN fragment)
constexpr int I8_NC = I8_BN / 8;                          // 8-column groups of the fragment (4 registers each)
constexpr int I8_THREADS = 256;
constexpr size_t I8_SMEM = size_t(I8_STAGES) * I8_STAGE_BYTES + 128;   // + barriers
// epilogue exchange: each warpgroup hands over its diagonals of the other warpgroup's half of the column groups
constexpr int I8_XWORDS = I8_DIAGS * (I8_NC / 2) * 4;    // int32 per thread pair
static_assert(I8_NC % 2 == 0, "the epilogue splits the column groups in halves");
static_assert(size_t(I8_XWORDS) * 128 * 4 <= size_t(I8_STAGES) * I8_STAGE_BYTES, "exchange must fit the ring");

// Warpgroup w's accumulator slot of diagonal d, or -1 when the other warpgroup owns d.
__host__ __device__ constexpr int i8_slot(int w, int d) {
  return w == 0 ? (d == 0 ? 0 : d == 1 ? 1 : d == 3 ? 2 : d == 5 ? 3 : -1) : (d == 2 ? 0 : d == 4 ? 1 : d == 6 ? 2 : -1);
}
__host__ __device__ constexpr int i8_ndiag(int w) { return w == 0 ? 4 : 3; }

__device__ __forceinline__ uint32_t i8_smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void i8_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(i8_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void i8_mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(i8_smem_u32(bar)), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void i8_mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(i8_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void i8_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(i8_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void i8_bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(i8_smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(i8_smem_u32(bar))
               : "memory");
}

// wgmma shared-memory descriptor, K-major, no swizzle: core matrix = 8 rows x 16 bytes stored contiguously (128 B).
// lbo = byte distance between the two core matrices that are adjacent in K, sbo = byte distance between consecutive
// groups of 8 rows (M / N direction).  Bits: [0,14) address >> 4, [16,30) lbo >> 4, [32,46) sbo >> 4, [62,64) layout
// = 0 (no swizzle).
__device__ __forceinline__ uint64_t i8_smem_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  return uint64_t((smem_addr >> 4) & 0x3FFF) | (uint64_t((lbo >> 4) & 0x3FFF) << 16) | (uint64_t((sbo >> 4) & 0x3FFF) << 32);
}

// D[64 x 48] += A[64 x 32] * B[48 x 32]^T, D = the accumulator registers d[OFF .. OFF + 24) (six column groups of 8,
// four registers each: rows lane/4 and lane/4 + 8 of the warp's 16, columns 2 (lane % 4) + {0, 1}).
#define I8_R8(o)                                                                                                          \
  "+r"(d[OFF + (o)]), "+r"(d[OFF + (o) + 1]), "+r"(d[OFF + (o) + 2]), "+r"(d[OFF + (o) + 3]), "+r"(d[OFF + (o) + 4]),     \
      "+r"(d[OFF + (o) + 5]), "+r"(d[OFF + (o) + 6]), "+r"(d[OFF + (o) + 7])
template <int OFF, int NA>
__device__ __forceinline__ void wg_i8_n48(int32_t (&d)[NA], uint64_t a, uint64_t b) {
  static_assert(I8_BN == 48 && OFF + 24 <= NA, "m64n48 fragment");
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n48k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, "
               "%14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p;\n\t}"
               : I8_R8(0), I8_R8(8), I8_R8(16)
               : "l"(a), "l"(b), "r"(1));
}
#undef I8_R8

template <int NA>
__device__ __forceinline__ void i8_wg_fence_acc(int32_t (&d)[NA]) {
#pragma unroll
  for (int i = 0; i < NA; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// ---------------------------------------------------------------------------------------------------------------
// Zm (fp64, [p][r][J]) -> six int8 digit slices in the tile layout described above.  zinv[p] = 2^48 / sZ[p].
// One thread = one row x 16 consecutive j (one 16-byte k-piece of every slice).  Consecutive threads take consecutive
// rows of an 8-row core matrix, so a warp writes 4 x 128 contiguous bytes per slice.
__global__ void __launch_bounds__(256) gwb_slice_kernel(int8_t* __restrict__ ZS, const double* __restrict__ Zm,
                                                         const double* __restrict__ zinv, int P, int J, int Jpad, int64_t nreal,
                                                         int64_t rcap) {
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int npiece = Jpad / 16;
  const int64_t rows8 = (nreal + 7) / 8;                   // groups of 8 rows that hold at least one realization
  const int64_t per_p = rows8 * npiece * 8;
  if (idx >= per_p * P) return;
  const int p = static_cast<int>(idx / per_p);
  int64_t rem = idx % per_p;
  const int r8 = static_cast<int>(rem & 7);
  rem >>= 3;
  const int piece = static_cast<int>(rem % npiece);        // 16-byte piece along j
  const int64_t g8 = rem / npiece;                         // 8-row group
  const int64_t r = g8 * 8 + r8;
  __align__(16) int8_t dig[I8_SLICES][16];
  const double sc = zinv[p];
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int j = piece * 16 + k;
    double v = 0.0;
    if (r < nreal && j < J) v = Zm[(size_t(p) * nreal + r) * J + j];
    long long X = __double2ll_rn(v * sc);
#pragma unroll
    for (int s = I8_SLICES - 1; s >= 0; --s) {           // balanced digits, least significant first
      const int d = static_cast<int>(static_cast<int8_t>(X & 0xFF));
      dig[s][k] = static_cast<int8_t>(d);
      X = (X - d) >> 8;
    }
  }
  const int64_t rblk = r / I8_BM;
  const int g = static_cast<int>((r % I8_BM) / 8);
  const int kch = piece / 2, c = piece % 2;
  const int64_t nkch = Jpad / I8_BK;
  const int64_t n_rblk = rcap / I8_BM;
  const size_t tile_off = ((((rblk * nkch + kch) * 16 + g) * 2 + c) * 8 + r8) * 16;
#pragma unroll
  for (int s = 0; s < I8_SLICES; ++s) {
    int8_t* dst = ZS + ((size_t(s) * P + p) * n_rblk) * (nkch * I8_ZT_BYTES) + tile_off;
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(dig[s]);
  }
}


// Diagnostics (ptar_debug_i8_timestamps): when set, the CTAs of the first 64 realizations record clock64() at the
// phase boundaries of thread 0, 8 slots per tile: start, setup done, loads issued, first stage landed, wgmmas issued,
// accumulators complete, epilogue done, k-chunks.
__device__ long long* g_i8_dbg = nullptr;

// Both warpgroups of a CTA meet here (a named barrier: the two warpgroups run different code paths).
__device__ __forceinline__ void i8_cta_barrier() { asm volatile("barrier.sync 1, %0;" ::"r"(I8_THREADS) : "memory"); }

// Warpgroup W's k-loop over the stage ring and its half of the epilogue.  Thread 0 (warpgroup 0) is also the producer:
// load_stage(kc) fills the ring slot of k-chunk kc.
template <int W, class LoadStage>
__device__ __forceinline__ void i8_synth_warpgroup(const LoadStage& load_stage, unsigned char* stage_base, uint64_t* full,
                                                   uint64_t* empty, int nk, long long* dbg, double* __restrict__ G,
                                                   int64_t g_ldr, const double* s_colscale, int kn0, int kpad, int64_t nreal) {
  constexpr int ND = i8_ndiag(W);
  const int tid = threadIdx.x, lt = tid & 127, warp = lt >> 5, lane = tid & 31;
  int32_t acc[ND * I8_NACC];
#pragma unroll
  for (int i = 0; i < ND * I8_NACC; ++i) acc[i] = 0;
  for (int kc = 0; kc < nk; ++kc) {
    const int st = kc % I8_STAGES;
    i8_mbar_wait(full + st, (kc / I8_STAGES) & 1);
    if (W == 0 && dbg && tid == 0 && kc == 0) dbg[3] = clock64();
    const uint32_t sa = i8_smem_u32(stage_base + size_t(st) * I8_STAGE_BYTES);
    const uint32_t sb = sa + I8_SLICES * I8_A_BYTES;
    // stage layout of one operand: [row group][2 k-pieces of 16 B][8 rows][16 B]: lbo = 128, sbo = 256.  Slice pair
    // (s, t) accumulates into registers I8_NACC * i8_slot(W, s + t) ..
    i8_wg_fence_acc(acc);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int s = 0; s < I8_SLICES; ++s) {
      const uint64_t adesc = i8_smem_desc(sa + s * I8_A_BYTES, 128, 256);
#pragma unroll
      for (int t = 0; t < I8_SLICES; ++t) {
        if (s + t >= I8_DIAGS) break;
        const uint64_t bdesc = i8_smem_desc(sb + t * (I8_BN * I8_BK), 128, 256);
        switch (i8_slot(W, s + t)) {
          case 0: wg_i8_n48<0>(acc, adesc, bdesc); break;
          case 1: wg_i8_n48<I8_NACC>(acc, adesc, bdesc); break;
          case 2: wg_i8_n48<2 * I8_NACC>(acc, adesc, bdesc); break;
          case 3:
            if constexpr (ND > 3) wg_i8_n48<3 * I8_NACC>(acc, adesc, bdesc);
            break;
          default: break;                                  // the other warpgroup's diagonal
        }
      }
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    // the group of k-chunk kc - 1 has retired: its stage is free
    asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
    i8_wg_fence_acc(acc);
    if (kc > 0) {
      const int pst = (kc - 1) % I8_STAGES;
      if (lt == 0) i8_mbar_arrive(empty + pst);
      if (W == 0 && tid == 0 && kc - 1 + I8_STAGES < nk) {
        i8_mbar_wait(empty + pst, ((kc - 1) / I8_STAGES) & 1);
        load_stage(kc - 1 + I8_STAGES);
      }
    }
  }
  if (W == 0 && dbg && tid == 0) dbg[2] = dbg[4] = clock64();
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
  i8_wg_fence_acc(acc);
  if (W == 0 && dbg && tid == 0) dbg[5] = clock64();

  // ---- epilogue.  Register 4 c + k of a diagonal holds knot 8 c + 2 (lane % 4) + (k & 1), realization
  // 16 warp + lane / 4 + 8 (k >> 1) -- the same output in both warpgroups.  Warpgroup 0 folds column groups
  // 0 .. NC/2 - 1, warpgroup 1 the rest; each first hands its diagonals of the other half to the other warpgroup through
  // the ring: word ((d NC/2 + c') 4 + k) 128 + lt.  Every issued bulk copy has landed (each was waited on) and both
  // warpgroups' wgmmas have retired once both pass the first barrier, so the ring is free.
  constexpr int H = I8_NC / 2;
  constexpr int c_own = W == 0 ? 0 : H, c_give = W == 0 ? H : 0;
  int32_t* xbuf = reinterpret_cast<int32_t*>(stage_base);
  i8_cta_barrier();
#pragma unroll
  for (int d = 0; d < I8_DIAGS; ++d) {
    if (i8_slot(W, d) < 0) continue;
#pragma unroll
    for (int i = 0; i < 4 * H; ++i) xbuf[(d * 4 * H + i) * 128 + lt] = acc[i8_slot(W, d) * I8_NACC + 4 * c_give + i];
  }
  i8_cta_barrier();
  // fold the seven diagonals in fp64 (int32 -> double without the conversion pipe: 2^52 + 2^31 + x sits exactly in the
  // mantissa of {0x43300000, x ^ 2^31}), scale, store
  const int64_t rrow = int64_t(blockIdx.x) * I8_CM + warp * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 4 * H; ++i) {
    const int c = c_own + i / 4, k = i & 3;
    double v = 0.0, w = 1.0;
#pragma unroll
    for (int d = 0; d < I8_DIAGS; ++d) {
      const int32_t xi = i8_slot(W, d) >= 0 ? acc[i8_slot(W, d) * I8_NACC + 4 * c + k] : xbuf[(d * 4 * H + i) * 128 + lt];
      const uint32_t vi = static_cast<uint32_t>(xi);
      const double x = __hiloint2double(0x43300000, static_cast<int>(vi ^ 0x80000000u)) - 4503601774854144.0;
      v = fma(x, w, v);
      w *= 0.00390625;                                     // 2^-8 per diagonal
    }
    const int n = 8 * c + 2 * (lane & 3) + (k & 1);
    const int64_t r = rrow + 8 * (k >> 1);
    // column-major grid G[kn0 + n][r]: a warp's store covers 8 consecutive realizations (64 B) of 4 knots
    if (r < nreal && n < kpad) G[size_t(kn0 + n) * g_ldr + r] = v * s_colscale[n];
  }
  if (W == 0 && dbg && tid == 0) dbg[6] = clock64();
}

// ---------------------------------------------------------------------------------------------------------------
// grid = (64-realization blocks, tiles); the realization index is fastest so the CTAs that share a tile's A slices run
// together.  Realization block b is half b % 2 of ZS r-block b / 2.  tile_list[tile] = {pulsar, first compact column,
// columns (<= BN), k extent}; AS tile index = blockIdx.y (the host builds AS in tile_list order).
// colscale[q] = sA[knot(q)] * 2^-16; zscale[p] = sZ[p].
__global__ void __launch_bounds__(I8_THREADS, 2)
gwb_synth_i8_kernel(double* __restrict__ G, int64_t g_ld, int64_t g_ldr, const int8_t* __restrict__ AS, const double* __restrict__ colscale,
                    const int8_t* __restrict__ ZS, const double* __restrict__ zscale, int P, int J, int Jpad, int64_t nreal,
                    int64_t rcap, const int32_t* __restrict__ tile_list) {
  extern __shared__ __align__(128) unsigned char i8_smem[];
  unsigned char* stage_base = i8_smem;
  uint64_t* full = reinterpret_cast<uint64_t*>(i8_smem + size_t(I8_STAGES) * I8_STAGE_BYTES);
  uint64_t* empty = full + I8_STAGES;

  const int tid = threadIdx.x;
  const int32_t* tl = tile_list + size_t(blockIdx.y) * 4;
  const int p = tl[0], kn0 = tl[1], kcnt = tl[2];
  const int kend = min(J, tl[3]);
  const int nk = (kend + I8_BK - 1) / I8_BK;               // k-chunks of 32 with a non-zero A column
  const int64_t nkch = Jpad / I8_BK;
  const int64_t n_rblk = rcap / I8_BM;

  long long* dbg = (g_i8_dbg != nullptr && blockIdx.x == 0) ? g_i8_dbg + size_t(blockIdx.y) * 8 : nullptr;
  if (dbg && tid == 0) {
    dbg[0] = clock64();
    dbg[7] = nk;
  }
  // this CTA's half of Z-slice tile (s, k-chunk kc) is at zsrc + s * zslice + kc * I8_ZT_BYTES
  const int8_t* zsrc = ZS + ((size_t(p) * n_rblk + (blockIdx.x >> 1)) * nkch) * I8_ZT_BYTES + (blockIdx.x & 1) * I8_A_BYTES;
  const size_t zslice = size_t(P) * n_rblk * nkch * I8_ZT_BYTES;
  const int8_t* asrc = AS + size_t(blockIdx.y) * nkch * I8_B_BYTES;
  auto load_stage = [&](int kc) {          // one thread: 6 Z-slice halves + the stacked A-slice tile of k-chunk kc
    const int st = kc % I8_STAGES;
    unsigned char* sb = stage_base + size_t(st) * I8_STAGE_BYTES;
    i8_mbar_expect_tx(full + st, I8_STAGE_BYTES);
#pragma unroll
    for (int s = 0; s < I8_SLICES; ++s)
      i8_bulk_load(sb + s * I8_A_BYTES, zsrc + s * zslice + size_t(kc) * I8_ZT_BYTES, I8_A_BYTES, full + st);
    i8_bulk_load(sb + I8_SLICES * I8_A_BYTES, asrc + size_t(kc) * I8_B_BYTES, I8_B_BYTES, full + st);
  };
  __shared__ double s_colscale[I8_BN];
  if (tid >= 64 && tid < 64 + I8_BN) {       // scales of this tile's columns (read by the epilogue from shared memory)
    const int n = tid - 64;
    s_colscale[n] = (n < kcnt) ? colscale[kn0 + n] * zscale[p] : 0.0;
  }
  if (tid == 0) {
    for (int s = 0; s < I8_STAGES; ++s) {
      i8_mbar_init(full + s, 1);
      i8_mbar_init(empty + s, 2);            // one arrival per warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    for (int kc = 0; kc < nk && kc < I8_STAGES; ++kc) load_stage(kc);
  }
  __syncthreads();
  if (dbg && tid == 0) dbg[1] = clock64();

  const int kpad = (kcnt + 1) & ~1;
  if (tid < 128)
    i8_synth_warpgroup<0>(load_stage, stage_base, full, empty, nk, dbg, G, g_ldr, s_colscale, kn0, kpad, nreal);
  else
    i8_synth_warpgroup<1>(load_stage, stage_base, full, empty, nk, dbg, G, g_ldr, s_colscale, kn0, kpad, nreal);
}

}  // namespace ptar

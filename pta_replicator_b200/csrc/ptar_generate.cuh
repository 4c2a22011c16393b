// Fused residual generator for sm_90a (H100).
//
//   out[r][i] = w1_i z1 + w2_i z2                      white_noise.py:105-109
//             + ecorr_e z_{bucket(e)}                  white_noise.py:182
//             + sum_j F(t_i)_j sqrt(prior_j) z_j       red_noise.py:126-128
//             + lerp(G[r][psr], t_i)                   red_noise.py:286-287
//             + det_i                                  deterministic.py:160-165
//             + sum_s w_s(i) sum_j F(t_i)_j sqrt(prior_s,j) z_j    chromatic slots (DM, scattering; CHROM builds)
//
// One CTA = one tile (<=1024 time-sorted TOAs of one pulsar, <=64 kernel-epochs) x RC
// realizations.  Everything that is smooth inside an epoch is evaluated once per
// (epoch, realization) in an "epoch stage" and kept in shared memory as a quadratic in
// dt = t - t_ref(epoch):
//   * the Fourier projection F_e . a_r -- a [64 x J] x [J x 3RC] fp64 GEMM on the FMA pipe whose
//     three right-hand sides are the coefficient vector and its first two time derivatives, so
//     TOAs inside an epoch (sub-band TOAs < 1 s apart) are reached by a 2nd-order Taylor step whose
//     remainder is below fp64 rounding of the direct sum (the host picks the window and nd per tile
//     from the amplitude-weighted moments of omega, engine._taylor_moments; single-TOA epochs are
//     exact, nd = 1);
//   * the GWB grid interpolation (epochs never straddle a grid knot, so it is exactly linear in dt);
//   * the ECORR draw of the epoch's bucket.
// The basis tile F [J][64] arrives by one bulk-async (TMA) copy that overlaps the Philox generation
// of the coefficients.  The "TOA stage" then streams the realizations: one thread owns a TOA and
// four consecutive realizations (= the four outputs of one Philox counter), so per 4 outputs it
// spends two Philox calls, four Box-Muller pairs, six 128-bit shared loads, a Horner step and four
// coalesced 8-byte stores -- the only HBM traffic that scales with R x N_toa.
// The two stages can also run as two kernels (STAGE template parameter, ptar_generate_stage).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/ptar.h"
#include "ptar_rng.cuh"

namespace ptar {

// A CTA has 16 threads per realization of its chunk: RC = 16 -> 256 threads (4 CTAs/SM),
// RC = 32 -> 512 threads (2 CTAs/SM; the epoch stage is amortised over twice the outputs).
__host__ __device__ constexpr int gen_threads(int RC) { return 16 * RC; }
constexpr int EP = PTAR_TILE_EPOCHS;  // 64
#ifndef GEN_UNROLL
#define GEN_UNROLL 2  // two realization groups in flight per thread: +1.4 % measured (4: same)
#endif
constexpr int kGenUnroll = GEN_UNROLL;

__host__ __device__ constexpr int gen_css(int RC) { return 3 * RC + 2; }  // even (16-B rows), 4e-word bank skew

__host__ __device__ inline size_t gen_smem_bytes(int J, int RC) {
  // mbarrier (16 B) + max(Fs[J][64] + As[3][J][RC], Cs[64][css])  (Cs aliases the GEMM operands)
  const size_t ops = size_t(J) * EP + size_t(3) * J * RC;
  const size_t cs = size_t(EP) * gen_css(RC);
  return 16 + sizeof(double) * (ops > cs ? ops : cs);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- pieces of the epoch stage shared by the fused kernel (gen_body) and the standalone epoch kernel: one copy of
// the arithmetic, so the two schedules agree bit for bit by construction.

// Fourier-process coefficients a = sqrt(prior) * z of RB realizations and their first two time derivatives (1/2 folded
// into the 2nd): As = [3][J][RB].  One work item = one (even, odd) column pair x 4 realizations (red_noise.py:126-127).
// zrow(r) = the injected draws of local realization r (parity mode); Philox index blk0 + column on stream ``kind``.
template <int RB, bool INJECT, int NTHREADS, class ZRow>
__device__ __forceinline__ void fourier_coefficients(const double* scale, const double* om, double sgn_even, ZRow zrow,
                                                     uint32_t kind, uint32_t blk0, const PhiloxKeys& K, uint32_t psr, int J,
                                                     int nr, uint64_t rgroup0, double* As, int tid) {
  constexpr int RG = RB / 4;
  double* A0 = As;
  double* A1 = As + size_t(J) * RB;
  double* A2 = As + size_t(2) * J * RB;
  for (int idx = tid; idx < (J / 2) * RG; idx += NTHREADS) {
    const int k = idx / RG, rg = idx % RG;
    const int je = 2 * k, jo = 2 * k + 1;
    double ye[4], yo[4];
    if (INJECT) {
#pragma unroll
      for (int l = 0; l < 4; ++l) {
        const int r = rg * 4 + l;
        const bool ok = r < nr;
        const double* z = zrow(ok ? r : 0);
        ye[l] = ok ? z[je] : 0.0;
        yo[l] = ok ? z[jo] : 0.0;
      }
    } else {
      float n[4];
      normals4(n, blk0 + je, kind, psr, rgroup0 + rg, K);
#pragma unroll
      for (int l = 0; l < 4; ++l) ye[l] = static_cast<double>(n[l]);
      normals4(n, blk0 + jo, kind, psr, rgroup0 + rg, K);
#pragma unroll
      for (int l = 0; l < 4; ++l) yo[l] = static_cast<double>(n[l]);
    }
    const double se = scale[je], so = scale[jo], w = om[k];
    const double h = -0.5 * w * w;
    double ae[4], ao[4];
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      ae[l] = se * ye[l];
      ao[l] = so * yo[l];
    }
    auto put = [&](double* row, double v0, double v1, double v2, double v3) {
      double2* q = reinterpret_cast<double2*>(row + rg * 4);
      q[0] = make_double2(v0, v1);
      q[1] = make_double2(v2, v3);
    };
    put(A0 + je * RB, ae[0], ae[1], ae[2], ae[3]);
    put(A0 + jo * RB, ao[0], ao[1], ao[2], ao[3]);
    const double s1 = sgn_even * w, s2 = -sgn_even * w;
    put(A1 + je * RB, s1 * ao[0], s1 * ao[1], s1 * ao[2], s1 * ao[3]);
    put(A1 + jo * RB, s2 * ae[0], s2 * ae[1], s2 * ae[2], s2 * ae[3]);
    put(A2 + je * RB, h * ae[0], h * ae[1], h * ae[2], h * ae[3]);
    put(A2 + jo * RB, h * ao[0], h * ao[1], h * ao[2], h * ao[3]);
  }
}

// Red-noise coefficients of RB realizations (first local realization r0).
template <int RB, bool INJECT, int NTHREADS>
__device__ __forceinline__ void rn_coefficients(const ptar_gen_params& P, const PhiloxKeys& K, uint32_t psr, int J, int r0,
                                                int nr, uint64_t rgroup0, double* As, int tid) {
  auto zrow = [&](int r) { return P.zrn + (size_t(r0 + r) * P.n_psr + psr) * J; };
  fourier_coefficients<RB, INJECT, NTHREADS>(P.rn_scale + size_t(psr) * J, P.rn_omega + size_t(psr) * (J / 2),
                                             P.rn_convention ? 1.0 : -1.0, zrow, PTAR_K_RED, 0u, K, psr, J, nr, rgroup0, As,
                                             tid);
}

// Coefficients of chromatic slot s (basis (sin, cos) on absolute time, as rn_convention = 0); zoff = first column of
// the slot in the injected zchr rows.
template <int RB, bool INJECT, int NTHREADS>
__device__ __forceinline__ void chrom_coefficients(const ptar_gen_params& P, const ptar_chrom_model& CM, const PhiloxKeys& K,
                                                   int s, int zoff, int zld, uint32_t psr, int r0, int nr, uint64_t rgroup0,
                                                   double* As, int tid) {
  const int J = CM.J[s];
  auto zrow = [&](int r) { return CM.zchr + (size_t(r0 + r) * P.n_psr + psr) * zld + zoff; };
  fourier_coefficients<RB, INJECT, NTHREADS>(CM.scale[s] + size_t(psr) * J, CM.omega[s] + size_t(psr) * (J / 2), -1.0, zrow,
                                             PTAR_K_CHROM, uint32_t(s) << 16, K, psr, J, nr, rgroup0, As, tid);
}

// One bulk-async copy global -> shared completing on mbarrier ``bar``, and the wait for phase ``parity`` of ``bar``.
__device__ __forceinline__ void bulk_to_smem(uint64_t* bar, double* dst, const double* src, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}

__device__ __forceinline__ void mbar_init(uint64_t* bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar)));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// Shared memory of the chromatic builds: the operands of the widest GEMM (Jo columns) or the red-noise block Cs[64][css]
// that aliases them, then the chromatic block Cx[64][3 RC n_slot + 2] of the slots' sums.  The TOA-only kernel (STAGE 2)
// holds one unified block [64][3 RC (1 + n_slot) + 2].
__host__ __device__ inline size_t gen_chrom_xoff(int Jo, int RC) {
  const size_t ops = size_t(Jo) * EP + size_t(3) * Jo * RC;
  const size_t cs = size_t(EP) * gen_css(RC);
  return ops > cs ? ops : cs;
}
__host__ __device__ inline size_t gen_chrom_smem_bytes(int Jo, int RC, int n_slot, int stage) {
  if (stage == 2) return 16 + sizeof(double) * EP * (gen_css(RC) + 3 * RC * n_slot);
  return 16 + sizeof(double) * (gen_chrom_xoff(Jo, RC) + size_t(EP) * (3 * RC * n_slot + 2));
}

// GWB grid values of 4 consecutive realizations (first local row rl) at knot column j and j + 1: the grid is
// column-major, so each is one 32-byte sector.
__device__ __forceinline__ void load_grid4(const ptar_gen_params& P, int j, int r_first, double g0[4], double g1[4]) {
  const double2* Gc = reinterpret_cast<const double2*>(P.G + size_t(j) * P.g_ldr + r_first);
  const double2* Gn = reinterpret_cast<const double2*>(P.G + size_t(j + 1) * P.g_ldr + r_first);
  const double2 a01 = __ldg(Gc), a23 = __ldg(Gc + 1), b01 = __ldg(Gn), b23 = __ldg(Gn + 1);
  g0[0] = a01.x; g0[1] = a01.y; g0[2] = a23.x; g0[3] = a23.y;
  g1[0] = b01.x; g1[1] = b01.y; g1[2] = b23.x; g1[3] = b23.y;
}

// Additive terms of one (epoch, 4 realizations): GWB interpolation at the epoch reference time and its slope
// (red_noise.py:286-287; exactly linear inside an epoch), plus the ECORR draw of the epoch's bucket (white_noise.py:182).
// nv = how many of the 4 realizations exist; r_first = row of the first one in the injected arrays.
template <bool INJECT>
__device__ __forceinline__ void epoch_addends4(const ptar_gen_params& P, const PhiloxKeys& K, int ge, uint32_t psr, uint64_t rfield,
                                               int r_first, int nv, bool has_gwb, bool has_ecorr, const double g0[4],
                                               const double g1[4], double add0[4], double add1[4]) {
#pragma unroll
  for (int l = 0; l < 4; ++l) add0[l] = add1[l] = 0.0;
  if (has_gwb) {
    const double gwt = P.ep_gw[ge], ginv = P.ep_ginv[ge];
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      if (l < nv) {
        const double dg = g1[l] - g0[l];
        add0[l] = fma(gwt, dg, g0[l]);
        add1[l] = dg * ginv;
      }
    }
  }
  if (has_ecorr) {
    const double ec = P.ep_ecorr[ge];
    if (INJECT) {
      const size_t zo = P.psr_bucket_off[psr] + P.ep_bucket[ge];
#pragma unroll
      for (int l = 0; l < 4; ++l)
        if (l < nv) add0[l] += ec * P.zb[size_t(r_first + l) * P.n_bucket_total + zo];
    } else {
      float n[4];
      normals4(n, P.ep_bucket[ge], PTAR_K_ECORR, psr, rfield, K);
#pragma unroll
      for (int l = 0; l < 4; ++l) add0[l] += ec * static_cast<double>(n[l]);
    }
  }
}

// The quadratic of 4 realizations at dt: c = 12 doubles (c0, c1, c2) x 4 of one Cs row, nd Taylor terms.
__device__ __forceinline__ void quad4(const double* c, double dt, int nd, double v[4]) {
  const double2* c2 = reinterpret_cast<const double2*>(c);
  const double2 q0 = c2[0], q1 = c2[1], q2 = c2[2], q3 = c2[3], q4 = c2[4], q5 = c2[5];
  // (c0,c1,c2) x 4 realizations = q0.x q0.y q1.x | q1.y q2.x q2.y | q3.x q3.y q4.x | q4.y q5.x q5.y
  if (nd > 2) {
    v[0] = fma(dt, fma(dt, q1.x, q0.y), q0.x);
    v[1] = fma(dt, fma(dt, q2.y, q2.x), q1.y);
    v[2] = fma(dt, fma(dt, q4.x, q3.y), q3.x);
    v[3] = fma(dt, fma(dt, q5.y, q5.x), q4.y);
  } else if (nd > 1) {  // (c0, c1) only
    v[0] = fma(dt, q0.y, q0.x);
    v[1] = fma(dt, q2.x, q1.y);
    v[2] = fma(dt, q3.y, q3.x);
    v[3] = fma(dt, q5.x, q4.y);
  } else {
    v[0] = q0.x; v[1] = q1.y; v[2] = q3.x; v[3] = q4.y;
  }
}

// C[e][r][d] += sum_{j in [jlo, jhi)} F[j][e] * A[d][j][r] for epochs e0..e0+3 and realization rr of the fused epoch stage
// (F = Fs[J][64], A = As[3][J][RC]); one instantiation per Taylor order, so no predicated-off FMAs in the loop.
template <int RC>
__device__ __forceinline__ void epoch_gemm(const double* Fs, const double* As, int J, int jlo, int jhi, int e0, int rr, int nd,
                                           double acc[4][3]) {
  auto gemm = [&](auto ND) {
    constexpr int kNd = decltype(ND)::value;
    for (int j = jlo; j < jhi; ++j) {
      const double2 f01 = *reinterpret_cast<const double2*>(Fs + j * EP + e0);
      const double2 f23 = *reinterpret_cast<const double2*>(Fs + j * EP + e0 + 2);
      const double f[4] = {f01.x, f01.y, f23.x, f23.y};
#pragma unroll
      for (int d = 0; d < kNd; ++d) {
        const double a = As[(d * J + j) * RC + rr];
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i][d] = fma(f[i], a, acc[i][d]);
      }
    }
  };
  if (nd >= 3) gemm(std::integral_constant<int, 3>{});
  else if (nd == 2) gemm(std::integral_constant<int, 2>{});
  else gemm(std::integral_constant<int, 1>{});
}

// WHITE / DET: -1 = decided at run time from P.flags (generic build, used by the parity mode);
// WHITE 0/1/2 = no white noise / one merged draw / two draws, DET 0/1 = no / with deterministic term
// (specialised builds of the throughput mode: the flag tests disappear from the inner loop).
// STAGE 0: fused (epoch stage + TOA stage in one CTA); STAGE 1: epoch stage only, the per-(tile, chunk) block
// Cs[n_ep][CSS] goes to P.Cbuf; STAGE 2: TOA stage only, the block comes back with one bulk-async copy.
// Splitting costs ~20 % extra HBM traffic but the TOA-stage warps no longer share their SM with warps that
// sit in the epoch stage's barriers and load latencies.
// CHROM = 1: the chromatic slots of *CM (ptar_generate_chrom) -- their GEMMs run first, into Cx, so that the red-noise
// block Cs can still alias the GEMM operands; CHROM = 0 builds never touch CM.
template <int RC, bool INJECT, int WHITE, int DET, int STAGE, int CHROM = 0>
__device__ __forceinline__ void gen_body(const ptar_gen_params& P, const PhiloxKeys& K, const int tile_idx,
                                         const int chunk_idx, unsigned char* smem_raw, const ptar_chrom_model* CM) {
  constexpr int GEN_THREADS = 16 * RC;
  uint64_t* mbar = reinterpret_cast<uint64_t*>(smem_raw);
  double* Fs = reinterpret_cast<double*>(smem_raw + 16);
  const int J = P.J;
  double* As = Fs + size_t(J) * EP;
  double* Cs = Fs;  // written only after the GEMM has consumed Fs / As
  constexpr int CSS = gen_css(RC);
  constexpr int RG = RC / 4;

  const int tid = threadIdx.x;
  const ptar_tile tile = P.tiles[tile_idx];
  const int r0 = chunk_idx * RC;  // first realization (local to this call)
  const int nr = min(RC, P.nreal - r0);
  const uint32_t flags = P.flags;
  const bool has_red = (flags & PTAR_F_RED) && J > 0;
  const bool has_ecorr = (flags & PTAR_F_ECORR) != 0;
  const bool has_gwb = (flags & PTAR_F_GWB) && P.npts > 0;
  const bool has_epoch = has_red || has_ecorr || has_gwb || CHROM > 0;
  const int nd = tile.nd;
  const uint32_t psr = static_cast<uint32_t>(tile.psr);
  const uint64_t rgroup0 = static_cast<uint64_t>(P.real0 + r0) >> 2;
  // chromatic builds: Cbuf rows are [red 3 RC | slot 0 3 RC | slot 1 3 RC | 2 pad] (css_u doubles); in shared memory the
  // TOA-only kernel keeps that row, the epoch stage keeps the slots apart in Cx[64][cssx]
  const int n_slot = CHROM ? CM->n_slot : 0;
  const int css_u = CSS + 3 * RC * n_slot;
  const int rowp = STAGE == 2 ? css_u : CSS;
  int Jo = J;
  if (CHROM) {
#pragma unroll
    for (int s = 0; s < PTAR_CHROM_SLOTS; ++s) Jo = s < n_slot ? max(Jo, CM->J[s]) : Jo;
  }
  double* Cx = CHROM ? (STAGE == 2 ? Cs + 3 * RC : Fs + gen_chrom_xoff(Jo, RC)) : nullptr;
  const int cssx = STAGE == 2 ? css_u : 3 * RC * n_slot + 2;
  const bool on0 = CHROM && CM->on[0][psr], on1 = CHROM && n_slot > 1 && CM->on[1][psr];

  const int n_chunks = (P.nreal + RC - 1) / RC;
  double* cblock = (STAGE != 0 && P.Cbuf)
                       ? P.Cbuf + (size_t(tile.reserved) * n_chunks + size_t(chunk_idx) * tile.n_ep) * css_u
                       : nullptr;
  if (STAGE == 2) {
    if (has_epoch) {  // fetch the block the epoch kernel left for this (tile, chunk)
      if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(mbar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      }
      __syncthreads();
      if (tid == 0) {
        const uint32_t bytes = static_cast<uint32_t>(sizeof(double) * tile.n_ep * css_u);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mbar)), "r"(bytes)
                     : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                smem_u32(Cs)),
            "l"(cblock), "r"(bytes), "r"(smem_u32(mbar))
            : "memory");
      }
      uint32_t done = 0;
      while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(mbar))
            : "memory");
      }
    }
  } else {
  // ---- epoch stage -------------------------------------------------------------------
  // GEMM ownership: thread -> realization rr, epochs e0..e0+3, slice ks of the J columns.  Tiles with
  // few epochs split the column range 2- or 4-way so that all 8 warps work (split-K, reduced through
  // shared memory below).
  static_assert(RC == 16 || RC == 32, "RC must be 16 or 32");
  const int nsplit = tile.n_ep <= 16 ? 4 : (tile.n_ep <= 32 ? 2 : 1);
  const int eper = EP / nsplit;                 // epochs covered per split group
  const int gthreads = GEN_THREADS / nsplit;    // threads per split group
  const int ks = tid / gthreads, tg = tid % gthreads;
  const int rr = tg & (RC - 1);
  const int e0 = (tg / RC) * 4;
  double acc[4][3];
#pragma unroll
  for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = acc[i][2] = 0.0;

  if (CHROM) {  // chromatic slots: the same GEMM over each slot's basis tile, sums to Cx
    uint64_t* cbar = mbar + 1;
    uint32_t phase = 0;
    if (tid == 0) mbar_init(cbar);
    const int zld = CM->J[0] + (n_slot > 1 ? CM->J[1] : 0);
#pragma unroll
    for (int s = 0; s < PTAR_CHROM_SLOTS; ++s) {
      if (s >= n_slot) break;
      const int zoff = s ? CM->J[0] : 0;
      if (!(s == 0 ? on0 : on1)) continue;  // uniform per CTA
      const int Js = CM->J[s];
      double* Asx = Fs + size_t(Js) * EP;
      __syncthreads();  // the previous slot's operands are consumed; cbar's init is visible
      if (tid == 0)
        bulk_to_smem(cbar, Fs, CM->Ftile[s] + size_t(tile_idx) * Js * EP, static_cast<uint32_t>(sizeof(double) * Js * EP));
      chrom_coefficients<RC, INJECT, GEN_THREADS>(P, *CM, K, s, zoff, zld, psr, r0, nr, rgroup0, Asx, tid);
      __syncthreads();
      mbar_wait(cbar, phase);
      phase ^= 1;
      double cacc[4][3];
#pragma unroll
      for (int i = 0; i < 4; ++i) cacc[i][0] = cacc[i][1] = cacc[i][2] = 0.0;
      if (e0 < tile.n_ep) epoch_gemm<RC>(Fs, Asx, Js, (Js * ks) / nsplit, (Js * (ks + 1)) / nsplit, e0, rr, nd, cacc);
      __syncthreads();  // operands consumed
      double* cx = Cx + 3 * RC * s;
      if (nsplit > 1) {
        if (ks > 0) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            double* c = cx + (ks * eper + e0 + i) * cssx + rr * 3;
            c[0] = cacc[i][0]; c[1] = cacc[i][1]; c[2] = cacc[i][2];
          }
        }
        __syncthreads();
        if (ks == 0) {
          for (int g = 1; g < nsplit; ++g) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const double* c = cx + (g * eper + e0 + i) * cssx + rr * 3;
              cacc[i][0] += c[0]; cacc[i][1] += c[1]; cacc[i][2] += c[2];
            }
          }
        }
        __syncthreads();
      }
      if (ks == 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          double* c = cx + (e0 + i) * cssx + rr * 3;
          c[0] = cacc[i][0]; c[1] = cacc[i][1]; c[2] = cacc[i][2];
        }
      }
    }
    __syncthreads();  // Fs is free for the red-noise tile
  }

  if (has_red) {
    if (tid == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(mbar)));
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
      const uint32_t bytes = static_cast<uint32_t>(sizeof(double) * J * EP);
      const double* src = P.Ftile + size_t(tile_idx) * J * EP;
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mbar)), "r"(bytes)
                   : "memory");
      asm volatile(
          "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
              smem_u32(Fs)),
          "l"(src), "r"(bytes), "r"(smem_u32(mbar))
          : "memory");
    }
    // coefficients and their first two time derivatives: overlaps the bulk copy
    rn_coefficients<RC, INJECT, GEN_THREADS>(P, K, psr, J, r0, nr, rgroup0, As, tid);
    __syncthreads();
    {  // wait for the basis tile
      uint32_t done = 0;
      while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(mbar))
            : "memory");
      }
    }
    // C[e][r][d] = sum_j F[j][e] * A[d][j][r]   (this thread: columns [jlo, jhi))
    if (e0 < tile.n_ep) epoch_gemm<RC>(Fs, As, J, (J * ks) / nsplit, (J * (ks + 1)) / nsplit, e0, rr, nd, acc);
    __syncthreads();  // everyone is done reading Fs / As: Cs may overwrite them
    if (nsplit > 1) {  // split-K reduction: groups ks >= 1 park their partial sums in rows ks*eper + e
      if (ks > 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          double* c = Cs + (ks * eper + e0 + i) * CSS + rr * 3;
          c[0] = acc[i][0]; c[1] = acc[i][1]; c[2] = acc[i][2];
        }
      }
      __syncthreads();
      if (ks == 0) {
        for (int g = 1; g < nsplit; ++g) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const double* c = Cs + (g * eper + e0 + i) * CSS + rr * 3;
            acc[i][0] += c[0]; acc[i][1] += c[1]; acc[i][2] += c[2];
          }
        }
      }
      __syncthreads();
    }
  }
  if (has_epoch && ks == 0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      double* c = Cs + (e0 + i) * CSS + rr * 3;
      c[0] = acc[i][0];
      c[1] = acc[i][1];
      c[2] = acc[i][2];
    }
  }
  if (has_epoch && (has_ecorr || has_gwb)) {
    __syncthreads();
    // one pass over (epoch, 4 realizations): ECORR draw of the epoch's bucket, and the GWB grid
    // interpolation at the epoch reference time with its slope (exactly linear inside the epoch)
    for (int idx = tid; idx < tile.n_ep * RG; idx += GEN_THREADS) {
      const int e = idx / RG, rg = idx % RG;
      const int ge = tile.ep_start + e;
      double g0[4] = {0.0, 0.0, 0.0, 0.0}, g1[4] = {0.0, 0.0, 0.0, 0.0}, add0[4], add1[4];
      const int nv = nr - rg * 4;                       // realizations of this group that exist (may be <= 0)
      if (has_gwb && nv > 0) load_grid4(P, P.ep_gidx[ge], r0 + rg * 4, g0, g1);
      epoch_addends4<INJECT>(P, K, ge, psr, rgroup0 + rg, r0 + rg * 4, nv, has_gwb, has_ecorr, g0, g1, add0, add1);
#pragma unroll
      for (int l = 0; l < 4; ++l) {
        double* c = Cs + e * CSS + (rg * 4 + l) * 3;
        c[0] += add0[l];
        c[1] += add1[l];
      }
    }
  }
  if (has_epoch) __syncthreads();

    if (STAGE == 1) {
      if (CHROM) {  // red rows and slot rows merge into the Cbuf row
        const int n = tile.n_ep * css_u;
        for (int idx = tid; idx < n; idx += GEN_THREADS) {
          const int e = idx / css_u, c = idx - e * css_u;
          const double v = c < 3 * RC ? Cs[e * CSS + c] : (c < css_u - 2 ? Cx[e * cssx + c - 3 * RC] : 0.0);
          __stcg(cblock + idx, v);
        }
      } else if (has_epoch) {
        const int n = tile.n_ep * CSS;
        for (int idx = tid; idx < n; idx += GEN_THREADS) __stcg(cblock + idx, Cs[idx]);
      }
      return;
    }
  }
  // ---- TOA stage ---------------------------------------------------------------------
  const bool has_white = WHITE >= 0 ? (WHITE > 0) : ((flags & PTAR_F_WHITE) != 0);
  const bool two_draws = WHITE >= 0 ? (WHITE == 2) : (has_white && !(flags & PTAR_F_WHITE1));
  const bool has_det = DET >= 0 ? (DET > 0) : ((flags & PTAR_F_DET) != 0);
  const size_t ld = static_cast<size_t>(P.ld_out);
  for (int tt = tid; tt < tile.n_toa; tt += GEN_THREADS) {
    const size_t gi = size_t(tile.toa_start) + tt;
    // statics of this TOA (their latency is covered by the first Philox evaluation below)
    const double w1 = has_white ? P.w1[gi] : 0.0;
    const double w2 = two_draws ? P.w2[gi] : 0.0;
    const double det = has_det ? P.det[gi] : 0.0;
    const double dt = (has_epoch && nd > 1) ? P.dtau[gi] : 0.0;
    const int el = has_epoch ? static_cast<int>(P.eloc[gi]) : 0;
    const double wc0 = on0 ? CM->weight[0][gi] : 0.0, wc1 = on1 ? CM->weight[1][gi] : 0.0;
    const uint32_t wblock = static_cast<uint32_t>(tile.toa_local0 + tt);
    double* orow = P.out + size_t(r0) * ld + gi;
#pragma unroll kGenUnroll
    for (int rg = 0; rg * 4 < nr; ++rg, orow += 4 * ld) {
      float n1[4], n2[4];
      if (INJECT) {
        n1[0] = n1[1] = n1[2] = n1[3] = n2[0] = n2[1] = n2[2] = n2[3] = 0.f;
      }
      if (!INJECT && has_white) {
        normals4(n1, wblock, PTAR_K_WHITE1, psr, rgroup0 + rg, K);
        if (two_draws) normals4(n2, wblock, PTAR_K_WHITE2, psr, rgroup0 + rg, K);
      }
      double v[4] = {0.0, 0.0, 0.0, 0.0};
      if (has_epoch) {
        quad4(Cs + el * rowp + rg * 12, dt, nd, v);
        if (CHROM) {  // + w_s(TOA) * quadratic of slot s
          double q[4];
          if (on0) {
            quad4(Cx + el * cssx + rg * 12, dt, nd, q);
#pragma unroll
            for (int l = 0; l < 4; ++l) v[l] = fma(wc0, q[l], v[l]);
          }
          if (on1) {
            quad4(Cx + el * cssx + 3 * RC + rg * 12, dt, nd, q);
#pragma unroll
            for (int l = 0; l < 4; ++l) v[l] = fma(wc1, q[l], v[l]);
          }
        }
      }
      if (has_det) {
        v[0] += det; v[1] += det; v[2] += det; v[3] += det;
      }
      if (has_white) {
        if (INJECT) {
#pragma unroll
          for (int l = 0; l < 4; ++l) {
            if (rg * 4 + l < nr) {
              const size_t zi = size_t(r0 + rg * 4 + l) * ld + gi;
              v[l] = fma(w1, P.z1[zi], v[l]);
              if (two_draws) v[l] = fma(w2, P.z2[zi], v[l]);
            }
          }
        } else {
#ifdef GEN_WHITE_FP32
          const float w1f = static_cast<float>(w1), w2f = static_cast<float>(w2);
#pragma unroll
          for (int l = 0; l < 4; ++l) {
            const float x = two_draws ? fmaf(w2f, n2[l], w1f * n1[l]) : w1f * n1[l];
            v[l] += static_cast<double>(x);
          }
#else
#pragma unroll
          for (int l = 0; l < 4; ++l) v[l] = fma(w1, static_cast<double>(n1[l]), v[l]);
          if (two_draws) {
#pragma unroll
            for (int l = 0; l < 4; ++l) v[l] = fma(w2, static_cast<double>(n2[l]), v[l]);
          }
#endif
        }
      }
      if (rg * 4 + 4 <= nr) {  // streaming stores: the output is never re-read by this kernel
        __stcs(orow, v[0]);
        __stcs(orow + ld, v[1]);
        __stcs(orow + 2 * ld, v[2]);
        __stcs(orow + 3 * ld, v[3]);
      } else {
#pragma unroll
        for (int l = 0; l < 4; ++l)
          if (rg * 4 + l < nr) __stcs(orow + l * ld, v[l]);
      }
    }
  }
  // alignment slots after a pulsar's last TOA are written as zeros
  const int n_pad = ((tile.n_toa + 3) & ~3) - tile.n_toa;
  if (tid < n_pad) {
    for (int r = 0; r < nr; ++r) P.out[size_t(r0 + r) * ld + tile.toa_start + tile.n_toa + tid] = 0.0;
  }
}

// grid = (realization chunks, tiles); the chunk index is fastest so the CTAs that share a tile's statics and
// basis run together and hit L2.
template <int RC, bool INJECT, int WHITE, int DET, int STAGE>
__global__ void __launch_bounds__(16 * RC, 1024 / (16 * RC)) gen_kernel(const ptar_gen_params P, const PhiloxKeys K) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  gen_body<RC, INJECT, WHITE, DET, STAGE>(P, K, blockIdx.y, blockIdx.x, smem_raw, nullptr);
}

// The same with chromatic slots.  Their Cx block leaves room for two CTAs per SM at most (RC = 16, J = 60: 79-104 KB).
template <int RC, bool INJECT, int WHITE, int DET, int STAGE>
__global__ void __launch_bounds__(16 * RC, 512 / (16 * RC)) gen_chrom_kernel(const ptar_gen_params P, const PhiloxKeys K,
                                                                           const ptar_chrom_model CM) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  gen_body<RC, INJECT, WHITE, DET, STAGE, 1>(P, K, blockIdx.y, blockIdx.x, smem_raw, &CM);
}

// ---- standalone epoch kernel (two-kernel schedule) ------------------------------------------------------
// Same arithmetic as the epoch stage of gen_body (same summation order, so the two schedules agree bit for bit),
// blocked for the FP64 pipe instead of for co-residency with the TOA stage: one CTA = one tile x 32
// realizations (two 16-realization blocks of P.Cbuf); a thread accumulates 4 epochs x 2 realizations x 3 Taylor
// orders (24 DFMA per five 128-bit shared loads) and writes its 6 coefficients per epoch straight to Cbuf.
// The ECORR draw and the GWB grid interpolation (scattered reads of G, the long-latency part) are fetched
// first, into their own shared array, so their latency hides behind the coefficient generation and the GEMM.
// 16 + 8 (160 J + 4096) bytes of shared memory: 109.6 KB at J = 60 -> 2 CTAs per SM.
constexpr int EPK_RB = 32;
constexpr int EPK_THREADS = 256;
constexpr int EPK_CSS = gen_css(16);  // row pitch of a Cbuf block (must match the TOA kernel's RC = 16 build)

__host__ __device__ inline size_t epoch_smem_bytes(int J) {
  size_t ops = size_t(J) * EP + size_t(3) * J * EPK_RB;  // Fs[J][64] + As[3][J][32]
  const size_t scratch = size_t(3) * 24 * 64;             // split-K partial sums alias the operands
  if (ops < scratch) ops = scratch;
  return 16 + sizeof(double) * (ops + size_t(EP) * EPK_RB * 2);  // + Add[64][32][2]
}

// acc[i][l][d] += sum_{j in [jlo, jhi)} F[j][e0 + i] * A[d][j][2 rp + l] (epoch kernel: 4 epochs x 2 realizations x nd)
__device__ __forceinline__ void epk_gemm(const double* Fs, const double* As, int J, int jlo, int jhi, int e0, int rp, int nd,
                                         double acc[4][2][3]) {
  auto gemm = [&](auto ND) {
    constexpr int kNd = decltype(ND)::value;
#pragma unroll 2
    for (int j = jlo; j < jhi; ++j) {
      const double2 f01 = *reinterpret_cast<const double2*>(Fs + j * EP + e0);
      const double2 f23 = *reinterpret_cast<const double2*>(Fs + j * EP + e0 + 2);
      const double f[4] = {f01.x, f01.y, f23.x, f23.y};
#pragma unroll
      for (int d = 0; d < kNd; ++d) {
        const double2 a = *reinterpret_cast<const double2*>(As + (d * J + j) * EPK_RB + 2 * rp);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          acc[i][0][d] = fma(f[i], a.x, acc[i][0][d]);
          acc[i][1][d] = fma(f[i], a.y, acc[i][1][d]);
        }
      }
    }
  };
  if (nd >= 3) gemm(std::integral_constant<int, 3>{});
  else if (nd == 2) gemm(std::integral_constant<int, 2>{});
  else gemm(std::integral_constant<int, 1>{});
}

// split-K of the epoch kernel: groups ks >= 1 park their 24 partial sums in scratch[ks-1][q][tg] (over the dead operands
// at Fs), group 0 adds them in group order
__device__ __forceinline__ void epk_split_k(double* Fs, int ks, int nsplit, int gthreads, int tg, double acc[4][2][3]) {
  __syncthreads();
  double* scratch = Fs;
  if (ks > 0) {
    double* s = scratch + size_t(ks - 1) * 24 * gthreads + tg;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int l = 0; l < 2; ++l)
#pragma unroll
        for (int d = 0; d < 3; ++d) s[((i * 2 + l) * 3 + d) * gthreads] = acc[i][l][d];
  }
  __syncthreads();
  if (ks == 0) {
    for (int g = 1; g < nsplit; ++g) {
      const double* s = scratch + size_t(g - 1) * 24 * gthreads + tg;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int l = 0; l < 2; ++l)
#pragma unroll
          for (int d = 0; d < 3; ++d) acc[i][l][d] += s[((i * 2 + l) * 3 + d) * gthreads];
    }
  }
}

// Its chromatic build (CHROM = 1) sizes the operand region for the widest basis (Jo columns: epoch_smem_bytes(Jo)), then
// runs one more GEMM per slot after the red-noise one, into the slot's columns of the Cbuf row (50 + 48 n_slot doubles).

template <bool INJECT, int CHROM>
__device__ __forceinline__ void epoch_body(const ptar_gen_params& P, const PhiloxKeys& K, unsigned char* smem_raw,
                                           const ptar_chrom_model* CM) {
  uint64_t* mbar = reinterpret_cast<uint64_t*>(smem_raw);
  double* Fs = reinterpret_cast<double*>(smem_raw + 16);
  const int J = P.J;
  constexpr int RB = EPK_RB, CSS = EPK_CSS, RG = RB / 4;
  const int n_slot = CHROM ? CM->n_slot : 0;
  const int css_u = CSS + 48 * n_slot;
  int Jo = J;
  if (CHROM) {
#pragma unroll
    for (int s = 0; s < PTAR_CHROM_SLOTS; ++s) Jo = s < n_slot ? max(Jo, CM->J[s]) : Jo;
  }
  double* As = Fs + size_t(J) * EP;
  const size_t ops = size_t(Jo) * EP + size_t(3) * Jo * RB;
  double* Add = Fs + (ops < size_t(3) * 24 * 64 ? size_t(3) * 24 * 64 : ops);  // [epoch][realization][c0 add, c1 add]

  const int tid = threadIdx.x;
  const int tile_idx = blockIdx.y;
  const ptar_tile tile = P.tiles[tile_idx];
  const int r0 = blockIdx.x * RB;
  const int nr = min(RB, P.nreal - r0);
  const uint32_t flags = P.flags;
  const bool has_red = (flags & PTAR_F_RED) && J > 0;
  const bool has_ecorr = (flags & PTAR_F_ECORR) != 0;
  const bool has_gwb = (flags & PTAR_F_GWB) && P.npts > 0;
  const bool has_add = has_ecorr || has_gwb;
  const int nd = tile.nd;
  const uint32_t psr = static_cast<uint32_t>(tile.psr);
  const uint64_t rgroup0 = static_cast<uint64_t>(P.real0 + r0) >> 2;
  const int n_chunks = (P.nreal + 15) / 16;

  if (has_red) {
    if (tid == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(mbar)));
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      const uint32_t bytes = static_cast<uint32_t>(sizeof(double) * J * EP);
      const double* src = P.Ftile + size_t(tile_idx) * J * EP;
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mbar)), "r"(bytes)
                   : "memory");
      asm volatile(
          "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
              smem_u32(Fs)),
          "l"(src), "r"(bytes), "r"(smem_u32(mbar))
          : "memory");
    }
  }
  // ---- additive terms per (epoch, realization): GWB grid interpolation at the epoch reference time and its
  // slope, plus the ECORR draw of the epoch's bucket.  One work item = (epoch, 4 realizations), at most two per
  // thread.  The scattered grid loads are issued here and consumed after the coefficient generation below.
  constexpr int ADD_ITEMS = EP * RG / EPK_THREADS;  // 2
  double g0[ADD_ITEMS][4], g1[ADD_ITEMS][4];
#pragma unroll
  for (int m = 0; m < ADD_ITEMS; ++m) {
#pragma unroll
    for (int l = 0; l < 4; ++l) g0[m][l] = g1[m][l] = 0.0;
    const int idx = tid + m * EPK_THREADS;
    if (has_gwb && idx < tile.n_ep * RG) {
      const int e = idx / RG, rg = idx % RG;
      if (rg * 4 < nr) load_grid4(P, P.ep_gidx[tile.ep_start + e], r0 + rg * 4, g0[m], g1[m]);
    }
  }
  auto finish_add = [&]() {
#pragma unroll
    for (int m = 0; m < ADD_ITEMS; ++m) {
      const int idx = tid + m * EPK_THREADS;
      if (idx < tile.n_ep * RG) {
        const int e = idx / RG, rg = idx % RG;
        double add0[4], add1[4];
        epoch_addends4<INJECT>(P, K, tile.ep_start + e, psr, rgroup0 + rg, r0 + rg * 4, nr - rg * 4, has_gwb, has_ecorr, g0[m],
                               g1[m], add0, add1);
        double2* q = reinterpret_cast<double2*>(Add + (size_t(e) * RB + rg * 4) * 2);
#pragma unroll
        for (int l = 0; l < 4; ++l) q[l] = make_double2(add0[l], add1[l]);
      }
    }
  };

  // GEMM ownership (same split-K rule as gen_body): realization pair rp, epochs e0..e0+3, column slice ks
  const int nsplit = tile.n_ep <= 16 ? 4 : (tile.n_ep <= 32 ? 2 : 1);
  const int gthreads = EPK_THREADS / nsplit;
  const int ks = tid / gthreads, tg = tid % gthreads;
  const int rp = tg & 15;
  const int e0 = (tg >> 4) * 4;
  double acc[4][2][3];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int l = 0; l < 2; ++l) acc[i][l][0] = acc[i][l][1] = acc[i][l][2] = 0.0;

  if (has_red) {
    // coefficients and their first two time derivatives for 32 realizations (overlaps the bulk copy)
    rn_coefficients<RB, INJECT, EPK_THREADS>(P, K, psr, J, r0, nr, rgroup0, As, tid);
    if (has_add) finish_add();
    __syncthreads();  // As (and Add, and thread 0's mbarrier init) visible
    {
      uint32_t done = 0;
      while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(mbar))
            : "memory");
      }
    }
    if (e0 < tile.n_ep) epk_gemm(Fs, As, J, (J * ks) / nsplit, (J * (ks + 1)) / nsplit, e0, rp, nd, acc);
    if (nsplit > 1) epk_split_k(Fs, ks, nsplit, gthreads, tg, acc);
  } else if (has_add) {
    finish_add();
    __syncthreads();  // Add visible
  }
  // ---- out: 6 coefficients per epoch (2 realizations x 3 orders) = 48 contiguous bytes of the Cbuf row the TOA
  // kernel fetches with one bulk copy; the eight pair-threads of a 16-realization block cover 384 B of it.
  const int chunk = 2 * blockIdx.x + (rp >> 3);
  if (ks == 0 && chunk < n_chunks) {
    const int rl = (2 * rp) & 15;
    double* blockp = P.Cbuf + (size_t(tile.reserved) * n_chunks + size_t(chunk) * tile.n_ep) * css_u;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = e0 + i;
      if (e < tile.n_ep) {
        double a00 = 0.0, a01 = 0.0, a10 = 0.0, a11 = 0.0;
        if (has_add) {
          const double2* q = reinterpret_cast<const double2*>(Add + (size_t(e) * RB + 2 * rp) * 2);
          const double2 t0 = q[0], t1 = q[1];
          a00 = t0.x; a01 = t0.y; a10 = t1.x; a11 = t1.y;
        }
        double2* o = reinterpret_cast<double2*>(blockp + size_t(e) * css_u + rl * 3);
        __stcg(o, make_double2(acc[i][0][0] + a00, acc[i][0][1] + a01));
        __stcg(o + 1, make_double2(acc[i][0][2], acc[i][1][0] + a10));
        __stcg(o + 2, make_double2(acc[i][1][1] + a11, acc[i][1][2]));
        if (rl == 14) {  // row padding (the row's last two doubles)
          if (CHROM) __stcg(reinterpret_cast<double2*>(blockp + size_t(e) * css_u + css_u - 2), make_double2(0.0, 0.0));
          else __stcg(o + 3, make_double2(0.0, 0.0));
        }
      }
    }
  }
  if (CHROM) {  // one more GEMM per chromatic slot, same ownership and split-K as the red noise (same sums as gen_body)
    uint64_t* cbar = mbar + 1;
    uint32_t phase = 0;
    if (tid == 0) mbar_init(cbar);
    const int zld = CM->J[0] + (n_slot > 1 ? CM->J[1] : 0);
#pragma unroll
    for (int s = 0; s < PTAR_CHROM_SLOTS; ++s) {
      if (s >= n_slot) break;
      const int zoff = s ? CM->J[0] : 0;
      if (!CM->on[s][psr]) continue;  // uniform per CTA
      const int Js = CM->J[s];
      double* Asx = Fs + size_t(Js) * EP;
      __syncthreads();  // Fs and the split-K scratch are free; cbar's init is visible
      if (tid == 0)
        bulk_to_smem(cbar, Fs, CM->Ftile[s] + size_t(tile_idx) * Js * EP, static_cast<uint32_t>(sizeof(double) * Js * EP));
      chrom_coefficients<RB, INJECT, EPK_THREADS>(P, *CM, K, s, zoff, zld, psr, r0, nr, rgroup0, Asx, tid);
      __syncthreads();
      mbar_wait(cbar, phase);
      phase ^= 1;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int l = 0; l < 2; ++l) acc[i][l][0] = acc[i][l][1] = acc[i][l][2] = 0.0;
      if (e0 < tile.n_ep) epk_gemm(Fs, Asx, Js, (Js * ks) / nsplit, (Js * (ks + 1)) / nsplit, e0, rp, nd, acc);
      if (nsplit > 1) epk_split_k(Fs, ks, nsplit, gthreads, tg, acc);
      if (ks == 0 && chunk < n_chunks) {
        const int rl = (2 * rp) & 15;
        double* blockp = P.Cbuf + (size_t(tile.reserved) * n_chunks + size_t(chunk) * tile.n_ep) * css_u;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int e = e0 + i;
          if (e < tile.n_ep) {
            double2* o = reinterpret_cast<double2*>(blockp + size_t(e) * css_u + 48 * (1 + s) + rl * 3);
            __stcg(o, make_double2(acc[i][0][0], acc[i][0][1]));
            __stcg(o + 1, make_double2(acc[i][0][2], acc[i][1][0]));
            __stcg(o + 2, make_double2(acc[i][1][1], acc[i][1][2]));
          }
        }
      }
    }
  }
}

template <bool INJECT>
__global__ void __launch_bounds__(EPK_THREADS, 2) epoch_kernel(const ptar_gen_params P, const PhiloxKeys K) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  epoch_body<INJECT, 0>(P, K, smem_raw, nullptr);
}

template <bool INJECT>
__global__ void __launch_bounds__(EPK_THREADS, 2) epoch_chrom_kernel(const ptar_gen_params P, const PhiloxKeys K,
                                                                     const ptar_chrom_model CM) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  epoch_body<INJECT, 1>(P, K, smem_raw, &CM);
}

}  // namespace ptar

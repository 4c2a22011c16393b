// libptar_b200.so -- C ABI (include/ptar.h) over the sm_90a (H100) kernels.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -shared -Xcompiler -fPIC
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "../../include/ptar.h"
#include "ptar_burst.cuh"
#include "ptar_bwm.cuh"
#include "ptar_cpop.cuh"
#include "ptar_curn.cuh"
#include "ptar_cwpop.cuh"
#include "ptar_generate.cuh"
#include "ptar_gwb.cuh"
#include "ptar_gwb_i8.cuh"
#include "ptar_hd.cuh"
#include "ptar_fe.cuh"
#include "ptar_fp.cuh"
#include "ptar_fs.cuh"
#include "ptar_fs_refit.cuh"
#include "ptar_os.cuh"
#include "ptar_os_aniso.cuh"
#include "ptar_os_null.cuh"
#include "ptar_os_pf.cuh"
#include "ptar_rn.cuh"
#include "ptar_rng.cuh"
#include "ptar_timing.cuh"
#include "ptar_tpop.cuh"

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, const char* detail = "") {
  snprintf(g_err, sizeof(g_err), fmt, detail);
  return code;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE attribute of a kernel: remember, per kernel and
// device, that the opt-in has been made (one process may drive several GPUs).
constexpr int kMaxDevices = 64;
struct SmemOptIn {
  bool done[kMaxDevices] = {};
};
template <class Kernel>
int opt_in_smem(Kernel k, SmemOptIn& state, size_t bytes, const char* what) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = -1;
  if (dev >= 0 && state.done[dev]) return 0;
  const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
  if (e != cudaSuccess) {
    snprintf(g_err, sizeof(g_err), "%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e));
    return -100;
  }
  if (dev >= 0) state.done[dev] = true;
  return 0;
}

int check_launch(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
    return -100;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------
// red_noise.py:92-101 -- operation order kept: (2*pi * t) * f, then sin / cos.
__global__ void fourier_basis_kernel(double* __restrict__ out, const int64_t* __restrict__ row_off,
                                     int64_t col_stride, const double* __restrict__ tprime,
                                     const int32_t* __restrict__ row_psr, const double* __restrict__ freqs,
                                     const double* __restrict__ phase, int K, int convention, int64_t nrows) {
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= nrows * K) return;
  const int64_t row = idx / K;
  const int k = static_cast<int>(idx % K);
  const double f = freqs[size_t(row_psr[row]) * K + k];
  double arg = __dmul_rn(__dmul_rn(6.283185307179586, tprime[row]), f);
  if (phase) arg = __dadd_rn(arg, phase[size_t(row_psr[row]) * K + k]);   // pshift (red_noise.py:83-84)
  double s, c;
  sincos(arg, &s, &c);
  double* o = out + row_off[row];
  o[int64_t(2 * k) * col_stride] = convention ? c : s;
  o[int64_t(2 * k + 1) * col_stride] = convention ? s : c;
}

// deterministic.py:98-163.  src = {w0, fac1, fac2, fac3, phase0(orbital), w053, incfac1,
// incfac2, cos2psi, sin2psi}; psr_par[p] = {fplus, fcross, cosMu, pd_seconds}.
__global__ void cgw_kernel(double* __restrict__ out, const double* __restrict__ t, const int32_t* __restrict__ psr_of_toa,
                           const double* __restrict__ psr_par, const double* __restrict__ src, int mode, int psr_term,
                           int accumulate, int64_t n) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double w0 = src[0], fac1 = src[1], fac2 = src[2], fac3 = src[3], phase0 = src[4], w053 = src[5];
  const double inc1 = src[6], inc2 = src[7], c2p = src[8], s2p = src[9];
  const double* pp = psr_par + size_t(psr_of_toa[i]) * 4;
  const double fplus = pp[0], fcross = pp[1], cosMu = pp[2], pd = pp[3];
  const double toa = t[i];
  const double tp = toa - pd * (1 - cosMu);
  double omega, omega_p, phase, phase_p;
  if (mode == 0) {
    omega = w0 * pow(1 - fac1 * toa, -3.0 / 8);
    omega_p = w0 * pow(1 - fac1 * tp, -3.0 / 8);
    phase = phase0 + fac2 * (w053 - pow(omega, -5.0 / 3));
    phase_p = phase0 + fac2 * (w053 - pow(omega_p, -5.0 / 3));
  } else if (mode == 1) {
    omega = w0;
    omega_p = w0 * pow(1 + fac1 * pd * (1 - cosMu), -3.0 / 8);
    phase = phase0 + omega * toa;
    phase_p = phase0 + fac2 * (w053 - pow(omega_p, -5.0 / 3)) + omega_p * toa;
  } else {
    omega = w0;
    omega_p = omega;
    phase = phase0 + omega * toa;
    phase_p = phase0 + omega * tp;
  }
  const double At = sin(2 * phase) * inc1, Bt = cos(2 * phase) * inc2;
  const double Atp = sin(2 * phase_p) * inc1, Btp = cos(2 * phase_p) * inc2;
  const double alpha = fac3 / cbrt(omega), alpha_p = fac3 / cbrt(omega_p);
  const double rplus = alpha * (At * c2p + Bt * s2p), rcross = alpha * (-At * s2p + Bt * c2p);
  const double rplus_p = alpha_p * (Atp * c2p + Btp * s2p), rcross_p = alpha_p * (-Atp * s2p + Btp * c2p);
  const double res = psr_term ? fplus * (rplus_p - rplus) + fcross * (rcross_p - rcross)
                              : -fplus * rplus - fcross * rcross;
  out[i] = accumulate ? out[i] + res : res;
}

// ---------------------------------------------------------------------------------------
// Catalog of continuous-wave sources (deterministic.py:188-561; the reference's numba loops).
// cw_prefactor_kernel: the per-source scalars of :340-376 for one pulsar direction ->
//   pre[s][16] = {w0, fac1, fac2, fac3, phase0/2, w0^-5/3, incfac1, incfac2, cos2psi, sin2psi, fplus, fcross,
//                 cosMu, pd_sec, -, -}
// cw_catalog_kernel: thread = one TOA, CTA = 128 TOAs x one slice of the catalog staged through shared memory;
// NaN contributions (a binary that has already merged, :433-438) are dropped; slices are summed in a fixed order
// by cw_reduce_kernel so the result is deterministic.
__global__ void cw_prefactor_kernel(double* __restrict__ pre, const double* __restrict__ cat, int64_t n_src,
                                    double px, double py, double pz, double pdist_kpc, double pphase, int use_pphase) {
  const int64_t s = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (s >= n_src) return;
  const double gwtheta = cat[s], gwphi = cat[n_src + s];
  const double mc = cat[2 * n_src + s] * 4.925838061995516e-06;     // SOLAR2S (constants.py:6)
  const double dist = cat[3 * n_src + s] * 102927125054338.98;      // MPC2S   (constants.py:8)
  const double fgw = cat[4 * n_src + s], phase0 = cat[5 * n_src + s] / 2, psi = cat[6 * n_src + s], inc = cat[7 * n_src + s];
  const double w0 = 3.141592653589793 * fgw;
  const double cgt = cos(gwtheta), cgp = cos(gwphi), sgt = sin(gwtheta), sgp = sin(gwphi);
  const double mx = sgp, my = -cgp;
  const double nx = -cgt * cgp, ny = -cgt * sgp, nz = sgt;
  const double ox = -sgt * cgp, oy = -sgt * sgp, oz = -cgt;
  const double mc53 = pow(mc, 5.0 / 3);
  const double mdp = mx * px + my * py + 0.0 * pz, ndp = nx * px + ny * py + nz * pz, odp = ox * px + oy * py + oz * pz;
  const double cosMu = -odp;
  double pd = use_pphase ? pphase / (2 * 3.141592653589793 * fgw * (1 - cosMu)) / 102927125054.33899 : pdist_kpc;
  pd *= 102927125054.33899;                                          // KPC2S (constants.py:7)
  double* o = pre + s * 16;
  o[0] = w0;
  o[1] = 256.0 / 5 * mc53 * pow(w0, 8.0 / 3);
  o[2] = 1.0 / 32 / mc53;
  o[3] = mc53 / dist;
  o[4] = phase0;
  o[5] = pow(w0, -5.0 / 3);
  o[6] = 0.5 * (3 + cos(2 * inc));
  o[7] = 2 * cos(inc);
  o[8] = cos(2 * psi);
  o[9] = sin(2 * psi);
  o[10] = 0.5 * (mdp * mdp - ndp * ndp) / (1 + odp);
  o[11] = (mdp * ndp) / (1 + odp);
  o[12] = cosMu;
  o[13] = pd;
  o[14] = o[15] = 0.0;
}

constexpr int CW_TOAS = 128, CW_STAGE = 32;

__global__ void __launch_bounds__(CW_TOAS) cw_catalog_kernel(double* __restrict__ partial, const double* __restrict__ t,
                                                             int64_t n_toa, const double* __restrict__ pre, int64_t n_src,
                                                             int64_t src_per_slice, int mode, int psr_term) {
  __shared__ double sp[CW_STAGE][16];
  const int64_t i = int64_t(blockIdx.x) * CW_TOAS + threadIdx.x;
  const int64_t s_begin = int64_t(blockIdx.y) * src_per_slice;
  const int64_t s_end = min(n_src, s_begin + src_per_slice);
  const double toa = i < n_toa ? t[i] : 0.0;
  double acc = 0.0;
  for (int64_t s0 = s_begin; s0 < s_end; s0 += CW_STAGE) {
    const int64_t rem = s_end - s0;
    const int cnt = rem < CW_STAGE ? static_cast<int>(rem) : CW_STAGE;
    __syncthreads();
    for (int k = threadIdx.x; k < cnt * 16; k += CW_TOAS) sp[k >> 4][k & 15] = pre[(s0 + (k >> 4)) * 16 + (k & 15)];
    __syncthreads();
    for (int k = 0; k < cnt; ++k) {
      const double* q = sp[k];
      const double w0 = q[0], fac1 = q[1], fac2 = q[2], fac3 = q[3], phase0 = q[4], w053 = q[5];
      const double tp = toa - q[13] * (1 - q[12]);
      double omega, omega_p, phase, phase_p;
      if (mode == 0) {
        omega = w0 * pow(1 - fac1 * toa, -3.0 / 8);
        omega_p = w0 * pow(1 - fac1 * tp, -3.0 / 8);
        phase = phase0 + fac2 * (w053 - pow(omega, -5.0 / 3));
        phase_p = phase0 + fac2 * (w053 - pow(omega_p, -5.0 / 3));
      } else if (mode == 1) {
        omega = w0;
        omega_p = w0 * pow(1 + fac1 * q[13] * (1 - q[12]), -3.0 / 8);
        phase = phase0 + omega * toa;
        phase_p = phase0 + fac2 * (w053 - pow(omega_p, -5.0 / 3)) + omega_p * toa;
      } else {
        omega = w0;
        omega_p = omega;
        phase = phase0 + omega * toa;
        phase_p = phase0 + omega * tp;
      }
      double s2, c2, s2p, c2p;
      sincos(2 * phase, &s2, &c2);
      sincos(2 * phase_p, &s2p, &c2p);
      const double At = s2 * q[6], Bt = c2 * q[7], Atp = s2p * q[6], Btp = c2p * q[7];
      const double alpha = fac3 / cbrt(omega), alpha_p = fac3 / cbrt(omega_p);
      const double rplus = alpha * (At * q[8] + Bt * q[9]), rcross = alpha * (-At * q[9] + Bt * q[8]);
      const double rplus_p = alpha_p * (Atp * q[8] + Btp * q[9]), rcross_p = alpha_p * (-Atp * q[9] + Btp * q[8]);
      const double r = psr_term ? q[10] * (rplus_p - rplus) + q[11] * (rcross_p - rcross) : -q[10] * rplus - q[11] * rcross;
      acc += isnan(r) ? 0.0 : r;
    }
  }
  if (i < n_toa) partial[int64_t(blockIdx.y) * n_toa + i] = acc;
}

__global__ void cw_reduce_kernel(double* __restrict__ out, const double* __restrict__ partial, int64_t n_toa, int n_slices,
                                 int accumulate) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_toa) return;
  double a = 0.0;
  for (int k = 0; k < n_slices; ++k) a += partial[int64_t(k) * n_toa + i];
  out[i] = accumulate ? out[i] + a : a;
}

// deterministic.py:771-780: elliptically polarised burst from the two waveform samples of each TOA.  The products are
// rounded one by one (no FMA contraction) so the result is the reference's bit for bit.
__global__ void burst_kernel(double* __restrict__ out, const double* __restrict__ hplus, const double* __restrict__ hcross,
                             double fplus, double fcross, double c2, double s2, int accumulate, int64_t n) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double hp = hplus[i], hx = hcross[i];
  const double rplus = __dsub_rn(__dmul_rn(hp, c2), __dmul_rn(hx, s2));
  const double rcross = __dadd_rn(__dmul_rn(hp, s2), __dmul_rn(hx, c2));
  const double res = __dsub_rn(__dmul_rn(-fplus, rplus), __dmul_rn(fcross, rcross));
  out[i] = accumulate ? out[i] + res : res;
}

// deterministic.py:868-872: burst with memory, a ramp after the burst epoch.
__global__ void memory_kernel(double* __restrict__ out, const double* __restrict__ t, double amp, double t0, int accumulate,
                              int64_t n) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double res = t[i] < t0 ? 0.0 : __dmul_rn(amp, __dsub_rn(t[i], t0));
  out[i] = accumulate ? out[i] + res : res;
}

__global__ void philox_normals_kernel(float* __restrict__ out, int kind, int psr, int64_t realization, int64_t idx0,
                                      int64_t n, uint64_t seed) {
  const int64_t k = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (k >= n) return;
  float z[4];
  ptar::normals4(z, static_cast<uint32_t>(idx0 + k), kind, psr, static_cast<uint64_t>(realization) >> 2, ptar::philox_keys(seed));
  out[k] = z[realization & 3];
}

// Widest GEMM operand of a chromatic build: red noise or any slot.
int chrom_jo(const ptar_gen_params& p, const ptar_chrom_model* cm) {
  int jo = (p.flags & PTAR_F_RED) ? p.J : 0;
  for (int s = 0; s < cm->n_slot; ++s) jo = std::max(jo, int(cm->J[s]));
  return jo;
}

template <int RC, bool INJECT, int WHITE, int DET, int STAGE, int CHROM = 0>
int launch_stage(const ptar_gen_params& p, cudaStream_t st, const ptar_chrom_model* cm = nullptr) {
  // STAGE 2 only needs the Cs block; STAGE 0/1 need the GEMM operands
  size_t smem = ptar::gen_smem_bytes(p.J, RC);
  if (STAGE == 2) smem = 16 + sizeof(double) * ptar::EP * ptar::gen_css(RC);
  if (CHROM) smem = ptar::gen_chrom_smem_bytes(chrom_jo(p, cm), RC, cm->n_slot, STAGE);
  if (smem > 227 * 1024)
    return fail(-3, CHROM ? "ptar_generate_chrom: red-noise and chromatic bases too wide for shared memory at this rc%s"
                          : "ptar_generate: J too large for shared memory%s");
  static SmemOptIn optin;  // per instantiation
  if constexpr (CHROM) {
    if (int rc = opt_in_smem(ptar::gen_chrom_kernel<RC, INJECT, WHITE, DET, STAGE>, optin, 227 * 1024, "ptar_generate_chrom"))
      return rc;
  } else {
    if (int rc = opt_in_smem(ptar::gen_kernel<RC, INJECT, WHITE, DET, STAGE>, optin, 227 * 1024, "ptar_generate")) return rc;
  }
  const dim3 grid((p.nreal + RC - 1) / RC, p.n_tiles);
  if (grid.y > 65535) return fail(-3, "ptar_generate: more than 65535 tiles%s");
  if (STAGE != 0 && p.Cbuf) {  // the Cs blocks of this build must fit the scratch the caller gave
    const int64_t need = p.c_rows * int64_t(grid.x) * (ptar::gen_css(RC) + (CHROM ? 3 * RC * cm->n_slot : 0));
    if (p.c_rows <= 0 || p.cbuf_len < need) return fail(-2, "ptar_generate: Cbuf too small for this rc (need c_rows * ceil(nreal/rc) * (3 rc + 2) doubles)%s");
  }
  if constexpr (CHROM) {
    ptar::gen_chrom_kernel<RC, INJECT, WHITE, DET, STAGE><<<grid, ptar::gen_threads(RC), smem, st>>>(p, ptar::philox_keys(p.seed), *cm);
    return check_launch("ptar_generate_chrom");
  } else {
    ptar::gen_kernel<RC, INJECT, WHITE, DET, STAGE><<<grid, ptar::gen_threads(RC), smem, st>>>(p, ptar::philox_keys(p.seed));
    return check_launch("ptar_generate");
  }
}

// Epoch kernel of the two-kernel schedule (RC = 16 blocks of Cbuf, two per CTA).
template <bool INJECT, int CHROM = 0>
int launch_epoch(const ptar_gen_params& p, cudaStream_t st, const ptar_chrom_model* cm = nullptr) {
  const size_t smem = ptar::epoch_smem_bytes(CHROM ? chrom_jo(p, cm) : p.J);
  if (smem > 227 * 1024)
    return fail(-3, CHROM ? "ptar_generate_chrom: red-noise and chromatic bases too wide for the epoch kernel%s"
                          : "ptar_generate: J too large for shared memory%s");
  static SmemOptIn optin;
  const dim3 grid((p.nreal + ptar::EPK_RB - 1) / ptar::EPK_RB, p.n_tiles);
  if (grid.y > 65535) return fail(-3, "ptar_generate: more than 65535 tiles%s");
  {
    const int64_t need = p.c_rows * int64_t((p.nreal + 15) / 16) * (ptar::EPK_CSS + (CHROM ? 48 * cm->n_slot : 0));
    if (p.c_rows <= 0 || p.cbuf_len < need) return fail(-2, "ptar_generate: Cbuf too small (need c_rows * ceil(nreal/16) * 50 doubles)%s");
  }
  if constexpr (CHROM) {
    if (int rc = opt_in_smem(ptar::epoch_chrom_kernel<INJECT>, optin, 227 * 1024, "ptar_generate_chrom (epoch kernel)")) return rc;
    ptar::epoch_chrom_kernel<INJECT><<<grid, ptar::EPK_THREADS, smem, st>>>(p, ptar::philox_keys(p.seed), *cm);
    return check_launch("ptar_generate_chrom (epoch kernel)");
  } else {
    if (int rc = opt_in_smem(ptar::epoch_kernel<INJECT>, optin, 227 * 1024, "ptar_generate (epoch kernel)")) return rc;
    ptar::epoch_kernel<INJECT><<<grid, ptar::EPK_THREADS, smem, st>>>(p, ptar::philox_keys(p.seed));
    return check_launch("ptar_generate (epoch kernel)");
  }
}

thread_local int g_only_stage = 0;  // set by ptar_generate_stage: 1 = epoch kernel only, 2 = TOA kernel only

template <int RC, bool INJECT, int WHITE, int DET, int CHROM = 0>
int launch_gen(const ptar_gen_params& p, cudaStream_t st, const ptar_chrom_model* cm = nullptr) {
  const bool has_epoch = CHROM || (p.flags & (PTAR_F_RED | PTAR_F_ECORR | PTAR_F_GWB)) != 0;
  if (p.Cbuf && has_epoch) {  // two-kernel schedule
    if (g_only_stage != 2) {
      // the epoch kernel does not depend on WHITE / DET
      const int rc = RC == 16 ? launch_epoch<INJECT, CHROM>(p, st, cm) : launch_stage<RC, INJECT, -1, -1, 1, CHROM>(p, st, cm);
      if (rc || g_only_stage == 1) return rc;
    }
    return launch_stage<RC, INJECT, WHITE, DET, 2, CHROM>(p, st, cm);
  }
  if (g_only_stage == 1) return 0;   // nothing to do: no epoch terms (or fused schedule)
  return launch_stage<RC, INJECT, WHITE, DET, 0, CHROM>(p, st, cm);
}

// The build for (parity mode | rc, white draws, deterministic term).
template <int CHROM>
int dispatch_gen(const ptar_gen_params& p, cudaStream_t st, const ptar_chrom_model* cm, bool inject, int rc, int white, bool det) {
  if (inject) return launch_gen<16, true, -1, -1, CHROM>(p, st, cm);
  if (rc == 32) {
    switch (white * 2 + (det ? 1 : 0)) {
      case 0: return launch_gen<32, false, 0, 0, CHROM>(p, st, cm);
      case 1: return launch_gen<32, false, 0, 1, CHROM>(p, st, cm);
      case 2: return launch_gen<32, false, 1, 0, CHROM>(p, st, cm);
      case 3: return launch_gen<32, false, 1, 1, CHROM>(p, st, cm);
      case 4: return launch_gen<32, false, 2, 0, CHROM>(p, st, cm);
      default: return launch_gen<32, false, 2, 1, CHROM>(p, st, cm);
    }
  }
  switch (white * 2 + (det ? 1 : 0)) {
    case 0: return launch_gen<16, false, 0, 0, CHROM>(p, st, cm);
    case 1: return launch_gen<16, false, 0, 1, CHROM>(p, st, cm);
    case 2: return launch_gen<16, false, 1, 0, CHROM>(p, st, cm);
    case 3: return launch_gen<16, false, 1, 1, CHROM>(p, st, cm);
    case 4: return launch_gen<16, false, 2, 0, CHROM>(p, st, cm);
    default: return launch_gen<16, false, 2, 1, CHROM>(p, st, cm);
  }
}

template <bool INJECT, bool SLICE>
int launch_mix(double* Zm, const double* M, const double* zin, int n_psr, int J, int64_t nreal, uint64_t seed, int64_t real0,
               int8_t* ZS, const double* zinv, int Jpad, int64_t rcap, cudaStream_t st, const char* what) {
  const int KP = (n_psr + 3) & ~3, NP = (n_psr + 7) & ~7;
  // draws [KP][132] + M [NP][KP + 4] doubles: 113 KB at 67 pulsars (2 CTAs per SM), 217 KB at 112 pulsars; 113 pulsars pad
  // to KP = 116, NP = 120 (232 KB) and no longer fit the 227 KB limit (_cabi.MIX_MAX_PSR)
  const size_t smem = sizeof(double) * (size_t(KP) * ptar::MX_ZS + size_t(NP) * (KP + 4));
  if (smem > 227 * 1024) return fail(-3, "ptar_gwb_mix: more than 112 pulsars do not fit the shared-memory tile%s");
  static SmemOptIn optin;   // per instantiation
  if (int rc = opt_in_smem(ptar::gwb_mix_dmma_kernel<INJECT, SLICE>, optin, 227 * 1024, what)) return rc;
  // persistent: as many CTAs as are resident at once, each stages M once and loops over (column block, group) items
  int dev = 0, n_sm = 0, per_sm = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ptar::gwb_mix_dmma_kernel<INJECT, SLICE>, 256, smem);
  if (e != cudaSuccess || per_sm < 1) return fail(-100, "ptar_gwb_mix: resident-CTA query: %s", cudaGetErrorString(e));
  const int64_t items = int64_t((J + ptar::MIX_JT - 1) / ptar::MIX_JT) * ((nreal + 3) / 4);
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(items, int64_t(n_sm) * per_sm));
  ptar::gwb_mix_dmma_kernel<INJECT, SLICE><<<grid, 256, smem, st>>>(Zm, M, zin, n_psr, J, nreal, ptar::philox_keys(seed), real0, ZS,
                                                                     zinv, Jpad, rcap);
  return check_launch(what);
}

template <int KC>
int launch_timing(double* out, int64_t ld, int32_t nreal, const ptar_timing_model& tm, double* scratch, int stage,
                  cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>((nreal + ptar::tm_rb<KC>() - 1) / ptar::tm_rb<KC>()), static_cast<unsigned>(tm.n_tiles));
  if (stage != 2) {
    ptar::timing_reduce_kernel<KC><<<grid, ptar::TM_THREADS, 0, st>>>(out, ld, nreal, tm, scratch);
    if (int rc = check_launch("ptar_timing_project (reduce)")) return rc;
  }
  if (stage != 1) {
    ptar::timing_apply_kernel<KC><<<grid, ptar::TM_THREADS, 0, st>>>(out, ld, nreal, tm, scratch);
    if (int rc = check_launch("ptar_timing_project (apply)")) return rc;
  }
  return 0;
}

// The checks of the sky grid that the Fe and BWM models share: every model array present (``arrays``), n_psr and kp,
// n_sky and n_sb, and the arrays the sky kernels stage 16-byte aligned: ant, linv and BWM's ``sqm`` (nullptr for Fe).
// The caller checks the model's frequency or epoch count.
template <class Model>
int sky_model_check(const Model* m, bool arrays, const double* sqm, const char* what) {
  if (!arrays || !m->ant || !m->linv) return fail(-2, "%s: model arrays missing", what);
  if (m->n_psr < 1 || m->n_psr > PTAR_FE_MAX_PSR || m->kp != ((m->n_psr + 15) & ~15))
    return fail(-2, "%s: need 1 <= n_psr <= 128 and kp = n_psr rounded up to a multiple of 16", what);
  if (m->n_sky < 1 || m->n_sky > PTAR_FE_MAX_SKY || m->n_sb != (m->n_sky + ptar::FE_SB - 1) / ptar::FE_SB)
    return fail(-2, "%s: need 1 <= n_sky <= 12288 and n_sb = ceil(n_sky / 32)", what);
  if ((reinterpret_cast<uintptr_t>(sqm) | reinterpret_cast<uintptr_t>(m->ant) | reinterpret_cast<uintptr_t>(m->linv)) & 15)
    return fail(-2, sqm ? "%s: sqm, ant and linv must be 16-byte aligned" : "%s: ant and linv must be 16-byte aligned", what);
  return 0;
}

// The checks every population entry point shares: the call's arguments (-1) and, with rows, the slot table the add stage
// reads (-2).  Model: ptar_cwpop_model, ptar_cpop_model or ptar_tpop_model.
template <class Model>
int population_check(const double* rows, int64_t ld, int32_t nreal, int64_t real0, const Model* m, const double* scratch,
                     int stage, const char* what) {
  if (!m || !scratch || nreal <= 0 || real0 < 0 || stage < 0 || stage > 2) return fail(-1, "%s: bad argument", what);
  if (rows && (ld <= 0 || !m->slot_t || !m->slot_psr)) return fail(-2, "%s: rows need ld, slot_t and slot_psr", what);
  if (!rows && stage == 2) return fail(-2, "%s: the add stage needs rows", what);
  return 0;
}

// The grid of a population's add stage: `toas` slots by `rb` realizations per CTA (-3 past 65535 realization blocks).
int population_add_grid(int64_t ld, int32_t nreal, int toas, int rb, dim3* grid, const char* what) {
  const int64_t nrb = (int64_t(nreal) + rb - 1) / rb;
  if (nrb > 65535) return fail(-3, "%s: too many realizations per call", what);
  *grid = dim3(static_cast<unsigned>((ld + toas - 1) / toas), static_cast<unsigned>(nrb));
  return 0;
}

}  // namespace

extern "C" {

int ptar_version(void) { return PTAR_VERSION; }
const char* ptar_last_error(void) { return g_err; }

int ptar_cholesky_lower(double* L, const double* A, int n, int batch, int* info, void* stream) {
  if (!L || !A || n <= 0 || n > 1024 || batch <= 0) return fail(-1, "ptar_cholesky_lower: bad argument%s");
  ptar::cholesky_kernel<<<batch, 256, 0, static_cast<cudaStream_t>(stream)>>>(L, A, n, info);
  return check_launch("ptar_cholesky_lower");
}

int ptar_fourier_basis(double* out, const int64_t* row_off, int64_t col_stride, const double* tprime,
                       const int32_t* row_psr, const double* freqs, const double* phase, int K, int convention,
                       int64_t nrows, void* stream) {
  if (!out || !row_off || !tprime || !row_psr || !freqs || K <= 0 || nrows < 0)
    return fail(-1, "ptar_fourier_basis: bad argument%s");
  if (nrows == 0) return 0;
  const int64_t total = nrows * K;
  fourier_basis_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      out, row_off, col_stride, tprime, row_psr, freqs, phase, K, convention, nrows);
  return check_launch("ptar_fourier_basis");
}

int ptar_cgw_delay(double* out, const double* t, const int32_t* psr_of_toa, const double* psr_par, const double* src,
                   int mode, int psr_term, int accumulate, int64_t n, void* stream) {
  if (!out || !t || !psr_of_toa || !psr_par || !src || mode < 0 || mode > 2 || n < 0)
    return fail(-1, "ptar_cgw_delay: bad argument%s");
  if (n == 0) return 0;
  cgw_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      out, t, psr_of_toa, psr_par, src, mode, psr_term, accumulate, n);
  return check_launch("ptar_cgw_delay");
}

int ptar_burst_delay(double* out, const double* hplus, const double* hcross, double fplus, double fcross, double cos2psi,
                     double sin2psi, int accumulate, int64_t n, void* stream) {
  if (!out || !hplus || !hcross || n < 0) return fail(-1, "ptar_burst_delay: bad argument%s");
  if (n == 0) return 0;
  burst_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      out, hplus, hcross, fplus, fcross, cos2psi, sin2psi, accumulate, n);
  return check_launch("ptar_burst_delay");
}

int ptar_memory_delay(double* out, const double* t, double amp, double t0, int accumulate, int64_t n, void* stream) {
  if (!out || !t || n < 0) return fail(-1, "ptar_memory_delay: bad argument%s");
  if (n == 0) return 0;
  memory_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(out, t, amp, t0,
                                                                                                     accumulate, n);
  return check_launch("ptar_memory_delay");
}

int ptar_cw_catalog(double* out, const double* t, int64_t n_toa, const double* phat_host, const double* cat, int64_t n_src,
                    double pdist_kpc, double pphase, int use_pphase, int mode, int psr_term, int accumulate, double* pre,
                    double* partial, int n_slices, void* stream) {
  if (!out || !t || !phat_host || !cat || !pre || !partial || n_toa <= 0 || n_src <= 0 || n_slices <= 0 || mode < 0 || mode > 2)
    return fail(-1, "ptar_cw_catalog: bad argument%s");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cw_prefactor_kernel<<<static_cast<unsigned>((n_src + 255) / 256), 256, 0, st>>>(pre, cat, n_src, phat_host[0], phat_host[1],
                                                                                   phat_host[2], pdist_kpc, pphase, use_pphase);
  if (int rc = check_launch("ptar_cw_catalog (prefactors)")) return rc;
  const int64_t per = (n_src + n_slices - 1) / n_slices;
  const dim3 grid(static_cast<unsigned>((n_toa + CW_TOAS - 1) / CW_TOAS), static_cast<unsigned>(n_slices));
  if (grid.y > 65535) return fail(-3, "ptar_cw_catalog: more than 65535 slices%s");
  cw_catalog_kernel<<<grid, CW_TOAS, 0, st>>>(partial, t, n_toa, pre, n_src, per, mode, psr_term);
  if (int rc = check_launch("ptar_cw_catalog (sources x TOAs)")) return rc;
  cw_reduce_kernel<<<static_cast<unsigned>((n_toa + 255) / 256), 256, 0, st>>>(out, partial, n_toa, n_slices, accumulate);
  return check_launch("ptar_cw_catalog (slice reduction)");
}

int ptar_gwb_mix(double* Zm, const double* M, const double* zin, int n_psr, int J, int64_t nreal, uint64_t seed,
                 int64_t real0, void* stream) {
  if (!Zm || !M || n_psr <= 0 || J <= 0 || nreal <= 0) return fail(-1, "ptar_gwb_mix: bad argument%s");
  if (!zin && (real0 & 3)) return fail(-2, "ptar_gwb_mix: real0 must be a multiple of 4%s");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (zin) return launch_mix<true, false>(Zm, M, zin, n_psr, J, nreal, seed, real0, nullptr, nullptr, 0, 0, st, "ptar_gwb_mix");
  return launch_mix<false, false>(Zm, M, zin, n_psr, J, nreal, seed, real0, nullptr, nullptr, 0, 0, st, "ptar_gwb_mix");
}

int ptar_gwb_mix_i8(int8_t* ZS, const double* M, const double* zinv, int n_psr, int J, int Jpad, int64_t nreal, int64_t rcap,
                    uint64_t seed, int64_t real0, void* stream) {
  if (!ZS || !M || !zinv || n_psr <= 0 || J <= 0 || nreal <= 0) return fail(-1, "ptar_gwb_mix_i8: bad argument%s");
  if (n_psr > 8 * ptar::MX_MAXNT) return fail(-3, "ptar_gwb_mix_i8: more than 72 pulsars (use ptar_gwb_mix + ptar_gwb_slice_i8)%s");
  if (real0 & 3) return fail(-2, "ptar_gwb_mix_i8: real0 must be a multiple of 4%s");
  if (Jpad < J || (Jpad % ptar::I8_BK) || rcap < nreal || (rcap % ptar::I8_BM))
    return fail(-2, "ptar_gwb_mix_i8: need Jpad %% 32 == 0 >= J and rcap %% 128 == 0 >= nreal%s");
  return launch_mix<false, true>(nullptr, M, nullptr, n_psr, J, nreal, seed, real0, ZS, zinv, Jpad, rcap, static_cast<cudaStream_t>(stream),
                                 "ptar_gwb_mix_i8");
}

int ptar_gwb_synth(double* G, int64_t g_ld, int64_t g_ldr, const double* A, int64_t lda, const double* Zm, int J, int64_t nreal,
                   const int32_t* tile_list, int n_tiles, const int32_t* knots, int lower_tri, void* stream) {
  if (!G || !A || !Zm || !tile_list || !knots || J <= 0 || nreal <= 0 || n_tiles <= 0 || g_ld <= 0)
    return fail(-1, "ptar_gwb_synth: bad argument%s");
  if ((J & 3) || (lda & 1) || lda < J || (g_ld & 1) || (g_ldr & 3) || g_ldr < nreal)
    return fail(-2, "ptar_gwb_synth: need J %% 4 == 0, even lda >= J, even g_ld, g_ldr %% 4 == 0 >= nreal%s");
  const int64_t r_blocks = (nreal + ptar::DM_BC - 1) / ptar::DM_BC;
  if (r_blocks > 65535) return fail(-3, "ptar_gwb_synth: too many realizations per call%s");
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::gwb_synth_dmma_kernel, optin, ptar::DM_SMEM, "ptar_gwb_synth")) return rc;
  const dim3 grid(static_cast<unsigned>(n_tiles), static_cast<unsigned>(r_blocks));
  ptar::gwb_synth_dmma_kernel<<<grid, 256, ptar::DM_SMEM, static_cast<cudaStream_t>(stream)>>>(
      G, g_ld, g_ldr, A, lda, Zm, J, nreal, tile_list, knots, lower_tri);
  return check_launch("ptar_gwb_synth");
}

int ptar_gwb_slice_i8(int8_t* ZS, const double* Zm, const double* zinv, int n_psr, int J, int Jpad, int64_t nreal, int64_t rcap,
                      void* stream) {
  if (!ZS || !Zm || !zinv || n_psr <= 0 || J <= 0 || nreal <= 0) return fail(-1, "ptar_gwb_slice_i8: bad argument%s");
  if (Jpad < J || (Jpad % ptar::I8_BK) || rcap < nreal || (rcap % ptar::I8_BM))
    return fail(-2, "ptar_gwb_slice_i8: need Jpad %% 32 == 0 >= J and rcap %% 128 == 0 >= nreal%s");
  const int64_t total = ((nreal + 7) / 8) * (Jpad / 16) * 8 * n_psr;
  ptar::gwb_slice_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      ZS, Zm, zinv, n_psr, J, Jpad, nreal, rcap);
  return check_launch("ptar_gwb_slice_i8");
}

int ptar_gwb_synth_i8(double* G, int64_t g_ld, int64_t g_ldr, const int8_t* AS, const double* colscale, const int8_t* ZS, const double* zscale,
                      int n_psr, int J, int Jpad, int64_t nreal, int64_t rcap, const int32_t* tile_list, int n_tiles,
                      void* stream) {
  if (!G || !AS || !colscale || !ZS || !zscale || !tile_list || n_psr <= 0 || J <= 0 || nreal <= 0 || n_tiles <= 0 || g_ld <= 0)
    return fail(-1, "ptar_gwb_synth_i8: bad argument%s");
  if (Jpad < J || (Jpad % ptar::I8_BK) || rcap < nreal || (rcap % ptar::I8_BM) || (g_ld & 1) || (g_ldr & 3) || g_ldr < nreal)
    return fail(-2, "ptar_gwb_synth_i8: need Jpad %% 32 == 0 >= J, rcap %% 128 == 0 >= nreal, even g_ld, g_ldr %% 4 == 0 >= nreal%s");
  if ((reinterpret_cast<uintptr_t>(AS) | reinterpret_cast<uintptr_t>(ZS)) & 15)
    return fail(-2, "ptar_gwb_synth_i8: AS / ZS must be 16-byte aligned%s");
  if (n_tiles > 65535) return fail(-3, "ptar_gwb_synth_i8: more than 65535 tiles%s");
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::gwb_synth_i8_kernel, optin, ptar::I8_SMEM, "ptar_gwb_synth_i8")) return rc;
  const dim3 grid(static_cast<unsigned>((nreal + ptar::I8_CM - 1) / ptar::I8_CM), static_cast<unsigned>(n_tiles));
  ptar::gwb_synth_i8_kernel<<<grid, ptar::I8_THREADS, ptar::I8_SMEM, static_cast<cudaStream_t>(stream)>>>(
      G, g_ld, g_ldr, AS, colscale, ZS, zscale, n_psr, J, Jpad, nreal, rcap, tile_list);
  return check_launch("ptar_gwb_synth_i8");
}

int ptar_debug_i8_timestamps(void* buf) {
  const cudaError_t e = cudaMemcpyToSymbol(ptar::g_i8_dbg, &buf, sizeof(buf));
  if (e != cudaSuccess) return fail(-100, "ptar_debug_i8_timestamps: %s", cudaGetErrorString(e));
  return 0;
}

int ptar_generate(const ptar_gen_params* pp, void* stream) { return ptar_generate_chrom(pp, nullptr, stream); }

int ptar_generate_chrom(const ptar_gen_params* pp, const ptar_chrom_model* cm, void* stream) {
  if (!pp) return fail(-1, "ptar_generate: null params%s");
  const ptar_gen_params& p = *pp;
  if (!p.out || !p.tiles || p.n_tiles <= 0 || p.nreal <= 0 || p.n_psr <= 0)
    return fail(-1, "ptar_generate: bad geometry%s");
  if ((p.ld_out & 3) || (reinterpret_cast<uintptr_t>(p.out) & 31)) return fail(-2, "ptar_generate: out must be 32-byte aligned, ld_out %% 4 == 0%s");
  if ((p.flags & PTAR_F_RED) && (p.J <= 0 || (p.J & 1) || !p.Ftile || !p.rn_scale || !p.rn_omega))
    return fail(-2, "ptar_generate: red noise needs even J, Ftile, rn_scale, rn_omega%s");
  if ((p.flags & PTAR_F_WHITE) && (!p.w1 || (!(p.flags & PTAR_F_WHITE1) && !p.w2)))
    return fail(-2, "ptar_generate: white noise needs w1/w2%s");
  if ((p.flags & PTAR_F_ECORR) && (!p.ep_ecorr || !p.ep_bucket)) return fail(-2, "ptar_generate: ECORR needs ep_ecorr/ep_bucket%s");
  if ((p.flags & (PTAR_F_ECORR | PTAR_F_RED)) && (!p.eloc || !p.dtau)) return fail(-2, "ptar_generate: epoch terms need eloc/dtau%s");
  if ((p.flags & PTAR_F_GWB) && (!p.G || p.npts <= 1 || p.g_ld <= 0 || !p.ep_gidx || !p.ep_gw || !p.ep_ginv || !p.eloc || !p.dtau))
    return fail(-2, "ptar_generate: GWB needs G, g_ld, ep_gidx, ep_gw, ep_ginv, eloc, dtau%s");
  if ((p.flags & PTAR_F_GWB) && ((p.g_ldr & 3) || p.g_ldr < ((p.nreal + 3) & ~3) || (reinterpret_cast<uintptr_t>(p.G) & 31)))
    return fail(-2, "ptar_generate: G must be 32-byte aligned, column-major with g_ldr %% 4 == 0 >= nreal rounded up to 4%s");
  if ((p.flags & PTAR_F_DET) && !p.det) return fail(-2, "ptar_generate: DET needs det%s");
  const bool inject = p.z1 || p.z2 || p.zb || p.zrn || (cm && cm->zchr);
  if (inject) {
    if ((p.flags & PTAR_F_WHITE) && (!p.z1 || (!(p.flags & PTAR_F_WHITE1) && !p.z2))) return fail(-2, "ptar_generate: injected white draws missing%s");
    if ((p.flags & PTAR_F_ECORR) && (!p.zb || !p.psr_bucket_off)) return fail(-2, "ptar_generate: injected ECORR draws missing%s");
    if ((p.flags & PTAR_F_RED) && !p.zrn) return fail(-2, "ptar_generate: injected red-noise draws missing%s");
  } else if (p.real0 & 3) {
    return fail(-2, "ptar_generate: real0 must be a multiple of 4%s");
  }
  if (p.Cbuf && p.cbuf_len <= 0) return fail(-2, "ptar_generate: Cbuf given without cbuf_len%s");
  if (cm) {
    if (cm->n_slot < 1 || cm->n_slot > PTAR_CHROM_SLOTS) return fail(-2, "ptar_generate_chrom: n_slot must be 1 or 2%s");
    for (int s = 0; s < cm->n_slot; ++s) {
      if (cm->J[s] <= 0 || (cm->J[s] & 1) || !cm->Ftile[s] || !cm->scale[s] || !cm->omega[s] || !cm->weight[s] || !cm->on[s])
        return fail(-2, "ptar_generate_chrom: every slot needs even J > 0, Ftile, scale, omega, weight and on%s");
    }
    if (!p.eloc || !p.dtau) return fail(-2, "ptar_generate_chrom: chromatic terms need eloc/dtau%s");
    if (inject && !cm->zchr) return fail(-2, "ptar_generate_chrom: injected chromatic draws missing%s");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rc = p.rc ? p.rc : 16;
  if (rc != 16 && rc != 32) return fail(-2, "ptar_generate: rc must be 16 or 32%s");
  const int white = !(p.flags & PTAR_F_WHITE) ? 0 : ((p.flags & PTAR_F_WHITE1) ? 1 : 2);
  const bool det = (p.flags & PTAR_F_DET) != 0;
  if (cm) return dispatch_gen<1>(p, st, cm, inject, rc, white, det);
  return dispatch_gen<0>(p, st, nullptr, inject, rc, white, det);
}

int ptar_generate_stage(const ptar_gen_params* pp, int stage, void* stream) {
  return ptar_generate_stage_chrom(pp, nullptr, stage, stream);
}

int ptar_generate_stage_chrom(const ptar_gen_params* pp, const ptar_chrom_model* cm, int stage, void* stream) {
  if (stage < 1 || stage > 2) return fail(-1, "ptar_generate_stage: stage must be 1 (epoch kernel) or 2 (TOA kernel)%s");
  if (!pp || !pp->Cbuf) return fail(-2, "ptar_generate_stage: needs the two-kernel schedule (Cbuf)%s");
  g_only_stage = stage;
  const int rc = ptar_generate_chrom(pp, cm, stream);
  g_only_stage = 0;
  return rc;
}

int ptar_philox_normals(float* out, int kind, int psr, int64_t realization, int64_t idx0, int64_t n, uint64_t seed,
                        void* stream) {
  if (!out || n < 0) return fail(-1, "ptar_philox_normals: bad argument%s");
  if (n == 0) return 0;
  philox_normals_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      out, kind, psr, realization, idx0, n, seed);
  return check_launch("ptar_philox_normals");
}

int ptar_peer_export(const void* dev_ptr, void* handle_host, int64_t* offset) {
  if (!dev_ptr || !handle_host || !offset) return fail(-1, "ptar_peer_export: bad argument%s");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle is 64 bytes");
  cudaPointerAttributes attr;
  cudaError_t e = cudaPointerGetAttributes(&attr, dev_ptr);
  if (e != cudaSuccess || attr.type != cudaMemoryTypeDevice) return fail(-2, "ptar_peer_export: not a device pointer%s");
  // the handle describes the whole allocation: find its base with the driver's range query (through the runtime's
  // driver entry point, so that libcuda need not be linked)
  typedef int (*range_fn)(unsigned long long*, size_t*, unsigned long long);
  static range_fn get_range = nullptr;
  if (!get_range) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    e = cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &qr);
    if (e != cudaSuccess || !fn) return fail(-100, "ptar_peer_export: cuMemGetAddressRange unavailable%s");
    get_range = reinterpret_cast<range_fn>(fn);
  }
  unsigned long long base = 0;
  size_t size = 0;
  if (get_range(&base, &size, reinterpret_cast<unsigned long long>(dev_ptr)) != 0)
    return fail(-100, "ptar_peer_export: cuMemGetAddressRange failed%s");
  e = cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle_host), reinterpret_cast<void*>(base));
  if (e != cudaSuccess) return fail(-100, "ptar_peer_export: cudaIpcGetMemHandle: %s", cudaGetErrorString(e));
  *offset = static_cast<int64_t>(reinterpret_cast<unsigned long long>(dev_ptr) - base);
  return 0;
}

int ptar_peer_open(const void* handle_host, void** base_out) {
  if (!handle_host || !base_out) return fail(-1, "ptar_peer_open: bad argument%s");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle_host, sizeof(h));
  const cudaError_t e = cudaIpcOpenMemHandle(base_out, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return fail(-100, "ptar_peer_open: cudaIpcOpenMemHandle: %s", cudaGetErrorString(e));
  return 0;
}

int ptar_peer_close(void* base) {
  if (!base) return 0;
  const cudaError_t e = cudaIpcCloseMemHandle(base);
  if (e != cudaSuccess) return fail(-100, "ptar_peer_close: %s", cudaGetErrorString(e));
  return 0;
}

int ptar_peer_copy(void* dst, const void* src, int64_t bytes, void* stream) {
  if (!dst || !src || bytes < 0) return fail(-1, "ptar_peer_copy: bad argument%s");
  if (bytes == 0) return 0;
  const cudaError_t e = cudaMemcpyAsync(dst, src, static_cast<size_t>(bytes), cudaMemcpyDefault, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(-100, "ptar_peer_copy: %s", cudaGetErrorString(e));
  return 0;
}

int ptar_timing_project_stage(double* out, int64_t ld_out, int32_t nreal, const ptar_timing_model* tm, double* scratch,
                              int64_t scratch_len, int stage, void* stream) {
  if (!out || !tm || nreal <= 0 || ld_out <= 0 || stage < 0 || stage > 2) return fail(-1, "ptar_timing_project: bad argument%s");
  if (tm->n_tiles <= 0) return 0;   // no pulsar has a model
  if (!tm->tiles || !tm->seg_len || !tm->k || !tm->q_off || !tm->tile0 || !tm->n_tile || !tm->Q || !tm->sqrtw || !scratch)
    return fail(-2, "ptar_timing_project: model arrays / scratch missing%s");
  if (tm->kmax <= 0 || tm->kmax > PTAR_TM_KMAX) return fail(-2, "ptar_timing_project: kmax must be in 1..32%s");
  if (tm->n_tiles > 65535) return fail(-3, "ptar_timing_project: more than 65535 tiles%s");
  if (scratch_len < int64_t(tm->n_tiles) * nreal * tm->kmax)
    return fail(-2, "ptar_timing_project: scratch too small (need n_tiles * nreal * kmax doubles)%s");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (tm->kmax <= 4) return launch_timing<4>(out, ld_out, nreal, *tm, scratch, stage, st);
  if (tm->kmax <= 8) return launch_timing<8>(out, ld_out, nreal, *tm, scratch, stage, st);
  if (tm->kmax <= 16) return launch_timing<16>(out, ld_out, nreal, *tm, scratch, stage, st);
  return launch_timing<32>(out, ld_out, nreal, *tm, scratch, stage, st);
}

int ptar_timing_project(double* out, int64_t ld_out, int32_t nreal, const ptar_timing_model* tm, double* scratch,
                        int64_t scratch_len, void* stream) {
  return ptar_timing_project_stage(out, ld_out, nreal, tm, scratch, scratch_len, 0, stream);
}

// The basis width of the projection X [nreal][n_psr][ncp] (0 < nc <= max, ncp = nc rounded up to a multiple of 8) and
// the (log10 A, gamma) grid of the CURN, HD and red-noise likelihoods (2 <= n_amp <= 256, 1 <= n_gamma <= 256).
static inline bool nc_ok(int32_t nc, int32_t ncp, int32_t max = PTAR_OS_MAX_NC) { return nc > 0 && nc <= max && ncp == ((nc + 7) & ~7); }
static inline bool grid_ok(int32_t na, int32_t ng) { return na >= 2 && na <= PTAR_CURN_MAX_NA && ng >= 1 && ng <= PTAR_CURN_MAX_NG; }

int ptar_os_project_stage(const double* rows, int64_t ld, int32_t nreal, const ptar_os_model* os, double* partial,
                          int64_t partial_len, double* X, int stage, void* stream) {
  if (!rows || !os || !partial || !X || nreal <= 0 || ld <= 0 || stage < 0 || stage > 2)
    return fail(-1, "ptar_os_project: bad argument%s");
  if (!os->tiles || !os->tile0 || !os->n_tile || !os->C || os->n_tiles <= 0 || os->n_psr <= 0)
    return fail(-2, "ptar_os_project: model arrays missing%s");
  if (!nc_ok(os->nc, os->ncp, PTAR_RN_MAX_NC))   // the projection alone goes to 64
    return fail(-2, "ptar_os_project: need 0 < nc <= 64 and ncp = nc rounded up to a multiple of 8%s");
  if ((ld & 3) || (reinterpret_cast<uintptr_t>(rows) & 31))
    return fail(-2, "ptar_os_project: rows must be 32-byte aligned with ld %% 4 == 0%s");
  if (os->n_tiles > 65535) return fail(-3, "ptar_os_project: more than 65535 tiles%s");
  if (partial_len < int64_t(os->n_tiles) * nreal * os->ncp)
    return fail(-2, "ptar_os_project: partial too small (need n_tiles * nreal * ncp doubles)%s");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (stage != 2) {
    const dim3 grid(static_cast<unsigned>((nreal + ptar::OS_RB - 1) / ptar::OS_RB), static_cast<unsigned>(os->n_tiles));
    const int nt = os->ncp / 8;
    static SmemOptIn optin[8];
    switch (nt) {
#define PTAR_OS_LAUNCH(NT)                                                                                          \
  case NT:                                                                                                          \
    if (int rc = opt_in_smem(ptar::os_project_kernel<NT>, optin[NT - 1], ptar::os_project_smem(NT), "ptar_os_project")) \
      return rc;                                                                                                    \
    ptar::os_project_kernel<NT><<<grid, ptar::OS_THREADS, ptar::os_project_smem(NT), st>>>(rows, ld, nreal, *os, partial); \
    break;
      PTAR_OS_LAUNCH(1)
      PTAR_OS_LAUNCH(2)
      PTAR_OS_LAUNCH(3)
      PTAR_OS_LAUNCH(4)
      PTAR_OS_LAUNCH(5)
      PTAR_OS_LAUNCH(6)
      PTAR_OS_LAUNCH(7)
      PTAR_OS_LAUNCH(8)
#undef PTAR_OS_LAUNCH
    }
    if (int rc = check_launch("ptar_os_project (tile GEMM)")) return rc;
  }
  if (stage != 1) {
    const int64_t total = int64_t(nreal) * os->n_psr * os->ncp;
    ptar::os_sum_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(partial, nreal, *os, X);
    if (int rc = check_launch("ptar_os_project (tile sums)")) return rc;
  }
  return 0;
}

int ptar_os_project(const double* rows, int64_t ld, int32_t nreal, const ptar_os_model* os, double* partial,
                    int64_t partial_len, double* X, void* stream) {
  return ptar_os_project_stage(rows, ld, nreal, os, partial, partial_len, X, 0, stream);
}

int ptar_os_pairs(const double* X, int32_t nreal, const ptar_os_model* os, double* rho, double* a2, double* snr,
                  double* a2_mc, void* stream) {
  if (!X || !os || !a2 || !snr || !a2_mc || nreal <= 0) return fail(-1, "ptar_os_pairs: bad argument%s");
  if (!os->sqrt_phi || !os->pairs || !os->t_ab || !os->orf || !os->dnorm || !os->dsqrt || !os->finv)
    return fail(-2, "ptar_os_pairs: model arrays missing%s");
  if (os->n_psr < 2 || os->n_psr > PTAR_OS_MAX_PSR) return fail(-3, "ptar_os_pairs: need 2..256 pulsars%s");
  if (os->n_orf <= 0 || os->n_orf > PTAR_OS_MAX_ORF || os->n_pairs <= 0)
    return fail(-2, "ptar_os_pairs: need 1..4 templates and at least one pair%s");
  if (!nc_ok(os->nc, os->ncp))
    return fail(-2, "ptar_os_pairs: need 0 < nc <= 32 and ncp = nc rounded up to a multiple of 8%s");
  const size_t smem = sizeof(double) * (size_t(os->n_psr) * os->ncp + size_t(PTAR_OS_MAX_ORF) * ptar::OS_PAIR_THREADS);
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::os_pairs_kernel, optin, sizeof(double) * (size_t(PTAR_OS_MAX_PSR) * PTAR_OS_MAX_NC +
                                                                           size_t(PTAR_OS_MAX_ORF) * ptar::OS_PAIR_THREADS),
                           "ptar_os_pairs"))
    return rc;
  ptar::os_pairs_kernel<<<static_cast<unsigned>(nreal), ptar::OS_PAIR_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      X, nreal, *os, rho, a2, snr, a2_mc);
  return check_launch("ptar_os_pairs");
}

int ptar_os_pf(const double* X, int32_t nreal, const ptar_os_model* os, const ptar_os_pf_model* pf, double* rho,
               double* phi, double* snr, double* phi_mc, void* stream) {
  if (!X || !os || !pf || !phi || !snr || !phi_mc || nreal <= 0) return fail(-1, "ptar_os_pf: bad argument%s");
  if (!os->pairs || !os->orf || !pf->t || !pf->dnorm || !pf->dsqrt || !pf->finv)
    return fail(-2, "ptar_os_pf: model arrays missing%s");
  if (os->n_psr < 2 || os->n_psr > PTAR_OS_MAX_PSR) return fail(-3, "ptar_os_pf: need 2..256 pulsars%s");
  if (os->n_orf <= 0 || os->n_orf > PTAR_OS_MAX_ORF || os->n_pairs <= 0)
    return fail(-2, "ptar_os_pf: need 1..4 templates and at least one pair%s");
  if (!nc_ok(os->nc, os->ncp) || (os->nc & 1))
    return fail(-2, "ptar_os_pf: need an even 0 < nc <= 32 and ncp = nc rounded up to a multiple of 8%s");
  const size_t smem = sizeof(double) * size_t(os->n_psr) * os->nc;
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::os_pf_kernel, optin, sizeof(double) * size_t(PTAR_OS_MAX_PSR) * PTAR_OS_MAX_NC, "ptar_os_pf"))
    return rc;
  ptar::os_pf_kernel<<<static_cast<unsigned>(nreal), ptar::PF_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      X, *os, *pf, rho, phi, snr, phi_mc);
  return check_launch("ptar_os_pf");
}

// Stages 1 and 2 (0: both) of ptar_os_null and ptar_os_aniso: the pair products U of X (os_null_prepare_kernel), then
// out = U V / dsqrt over the column set of nl (os_null_gemm_kernel).  Errors name the entry point ``what`` and the stage.
static int os_pair_gemm(const double* X, int32_t nreal, const ptar_os_model& os, const ptar_os_null_model& nl, double* U,
                        double* out, int stage, cudaStream_t st, const char* what) {
  char msg[64];
  if (stage == 0 || stage == 1) {
    snprintf(msg, sizeof(msg), "%s (prepare)", what);
    static SmemOptIn optin;
    if (int rc = opt_in_smem(ptar::os_null_prepare_kernel, optin, sizeof(double) * PTAR_OS_MAX_PSR * PTAR_OS_MAX_NC, msg)) return rc;
    const size_t smem = sizeof(double) * size_t(os.n_psr) * os.ncp;
    ptar::os_null_prepare_kernel<<<static_cast<unsigned>(nreal), ptar::NL_THREADS, smem, st>>>(X, os, nl, U);
    if (int rc = check_launch(msg)) return rc;
  }
  if (stage == 0 || stage == 2) {
    snprintf(msg, sizeof(msg), "%s (GEMM)", what);
    static SmemOptIn optin;
    if (int rc = opt_in_smem(ptar::os_null_gemm_kernel, optin, ptar::NL_SMEM, msg)) return rc;
    const dim3 grid(static_cast<unsigned>(nl.n_colp / ptar::NL_BN), static_cast<unsigned>((nreal + ptar::NL_BM - 1) / ptar::NL_BM));
    ptar::os_null_gemm_kernel<<<grid, ptar::NL_THREADS, ptar::NL_SMEM, st>>>(U, nreal, nl, out);
    if (int rc = check_launch(msg)) return rc;
  }
  return 0;
}

int ptar_os_null_stage(const double* X, int32_t nreal, const ptar_os_model* os, const ptar_os_null_model* nl, double* U,
                       double* snr, int64_t* exceed, double* fap, int stage, void* stream) {
  if (!X || !os || !nl || !U || !snr || !exceed || !fap || nreal <= 0 || stage < 0 || stage > 3)
    return fail(-1, "ptar_os_null: bad argument%s");
  if (!os->sqrt_phi || !os->pairs || !nl->V || !nl->dsqrt) return fail(-2, "ptar_os_null: model arrays missing%s");
  if (os->n_psr < 2 || os->n_psr > PTAR_OS_MAX_PSR || os->n_pairs != os->n_psr * (os->n_psr - 1) / 2)
    return fail(-3, "ptar_os_null: need 2..256 pulsars and every pair%s");
  if (!nc_ok(os->nc, os->ncp) || (os->nc & 1))
    return fail(-2, "ptar_os_null: need an even 0 < nc <= 32 and ncp = nc rounded up to a multiple of 8%s");
  if (nl->method != PTAR_OS_NULL_PHASE_SHIFT && nl->method != PTAR_OS_NULL_SKY_SCRAMBLE)
    return fail(-2, "ptar_os_null: unknown method%s");
  if (nl->n_col < 2 || nl->n_col > PTAR_OS_MAX_NULL + 1 || nl->n_colp != ((nl->n_col + ptar::NL_BN - 1) & ~(ptar::NL_BN - 1)))
    return fail(-2, "ptar_os_null: need 2 <= n_col <= 65537 and n_colp = n_col rounded up to a multiple of 64%s");
  const int64_t kd = nl->method == PTAR_OS_NULL_PHASE_SHIFT ? int64_t(os->n_pairs) * os->nc : int64_t(os->n_pairs);
  if (nl->kd != kd || nl->kdp != ((kd + ptar::NL_BK - 1) & ~int64_t(ptar::NL_BK - 1)))
    return fail(-2, "ptar_os_null: kd must be 2 K n_pairs (phase shift) or n_pairs (sky scramble), kdp kd rounded up to 32%s");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = os_pair_gemm(X, nreal, *os, *nl, U, snr, stage, st, "ptar_os_null")) return rc;
  if (stage == 0 || stage == 3) {
    ptar::os_null_count_kernel<<<static_cast<unsigned>(nreal), ptar::NL_THREADS, 0, st>>>(snr, nl->n_col, exceed, fap);
    if (int rc = check_launch("ptar_os_null (count)")) return rc;
  }
  return 0;
}

int ptar_os_null(const double* X, int32_t nreal, const ptar_os_model* os, const ptar_os_null_model* nl, double* U,
                 double* snr, int64_t* exceed, double* fap, void* stream) {
  return ptar_os_null_stage(X, nreal, os, nl, U, snr, exceed, fap, 0, stream);
}

int ptar_os_aniso_stage(const double* X, int32_t nreal, const ptar_os_model* os, const ptar_os_aniso_model* am, double* U,
                        double* map, double* clm, double* z, double* chi2, double* snr_max, int64_t* argmax,
                        double* radio_map, int stage, void* stream) {
  if (!X || !os || !am || !U || !map || nreal <= 0 || stage < 0 || stage > 3) return fail(-1, "ptar_os_aniso: bad argument%s");
  if (!os->sqrt_phi || !os->pairs || !am->V || !am->dsqrt) return fail(-2, "ptar_os_aniso: model arrays missing%s");
  if (os->n_psr < 2 || os->n_psr > PTAR_OS_MAX_PSR || os->n_pairs != os->n_psr * (os->n_psr - 1) / 2)
    return fail(-3, "ptar_os_aniso: need 2..256 pulsars and every pair%s");
  if (!nc_ok(os->nc, os->ncp))
    return fail(-2, "ptar_os_aniso: need 0 < nc <= 32 and ncp = nc rounded up to a multiple of 8%s");
  if (am->n_lm < 0 || am->n_lm > PTAR_OS_ANISO_MAX_LM || am->n_z != std::max(am->n_lm - 1, 0) || am->n_sky < 0 ||
      am->n_sky > PTAR_OS_ANISO_MAX_SKY || am->n_lm + am->n_sky < 1)
    return fail(-2, "ptar_os_aniso: need 0 <= n_lm <= 64, n_z = max(n_lm - 1, 0), 0 <= n_sky <= 12288 and a basis%s");
  if (am->n_col != am->n_lm + am->n_z + am->n_sky || am->n_colp != ((am->n_col + ptar::NL_BN - 1) & ~(ptar::NL_BN - 1)))
    return fail(-2, "ptar_os_aniso: need n_col = n_lm + n_z + n_sky and n_colp = n_col rounded up to a multiple of 64%s");
  if (am->kd != os->n_pairs || am->kdp != ((am->kd + ptar::NL_BK - 1) & ~int64_t(ptar::NL_BK - 1)))
    return fail(-2, "ptar_os_aniso: kd must be n_pairs and kdp kd rounded up to 32%s");
  if ((am->n_lm > 0 && (!clm || !chi2 || (am->n_z > 0 && !z))) || (am->n_sky > 0 && (!snr_max || !argmax)))
    return fail(-1, "ptar_os_aniso: an output of a registered basis is NULL%s");
  // the sky-scramble operands of ptar_os_null: U[r][q] = x_a . x_b, V^T rows = the columns of the anisotropy map
  const ptar_os_null_model nl{PTAR_OS_NULL_SKY_SCRAMBLE, am->n_col, am->n_colp, 0, am->kd, am->kdp, am->V, am->dsqrt};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = os_pair_gemm(X, nreal, *os, nl, U, map, stage, st, "ptar_os_aniso")) return rc;
  if (stage == 0 || stage == 3) {
    ptar::os_aniso_reduce_kernel<<<static_cast<unsigned>(nreal), ptar::AN_THREADS, 0, st>>>(map, *am, clm, z, chi2, snr_max,
                                                                                          argmax, radio_map);
    if (int rc = check_launch("ptar_os_aniso (reduce)")) return rc;
  }
  return 0;
}

int ptar_os_aniso(const double* X, int32_t nreal, const ptar_os_model* os, const ptar_os_aniso_model* am, double* U,
                  double* map, double* clm, double* z, double* chi2, double* snr_max, int64_t* argmax, double* radio_map,
                  void* stream) {
  return ptar_os_aniso_stage(X, nreal, os, am, U, map, clm, z, chi2, snr_max, argmax, radio_map, 0, stream);
}

static int fp_model_check(const ptar_fp_model* fp, const char* what) {
  if (!fp->Ct || !fp->psr_order || !fp->seg_off || !fp->seg_len || fp->n_psr <= 0 || fp->ld <= 0)
    return fail(-2, "%s: model arrays missing", what);
  if (fp->n_freq <= 0 || fp->n_freq > PTAR_FP_MAX_FREQ || fp->n_cb != (2 * fp->n_freq + ptar::FP_BN - 1) / ptar::FP_BN)
    return fail(-2, "%s: need 1 <= n_freq <= 256 and n_cb = ceil(2 n_freq / 64)", what);
  return 0;
}

int ptar_fp_project(const double* rows, int64_t ld, int32_t nreal, const ptar_fp_model* fp, double* amps, void* stream) {
  if (!rows || !fp || !amps || nreal <= 0 || ld <= 0) return fail(-1, "ptar_fp_project: bad argument%s");
  if (int rc = fp_model_check(fp, "ptar_fp_project")) return rc;
  if ((ld & 3) || (reinterpret_cast<uintptr_t>(rows) & 31) || (reinterpret_cast<uintptr_t>(fp->Ct) & 15))
    return fail(-2, "ptar_fp_project: rows must be 32-byte aligned with ld %% 4 == 0, Ct 16-byte aligned%s");
  const int64_t blocks = int64_t(fp->n_psr) * ((nreal + ptar::OS_RB - 1) / ptar::OS_RB) * fp->n_cb;
  if (blocks > 0x7fffffff) return fail(-3, "ptar_fp_project: grid too large%s");
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::fp_project_kernel, optin, ptar::FP_SMEM, "ptar_fp_project")) return rc;
  ptar::fp_project_kernel<<<static_cast<unsigned>(blocks), ptar::FP_THREADS, ptar::FP_SMEM, static_cast<cudaStream_t>(stream)>>>(
      rows, ld, nreal, *fp, amps);
  return check_launch("ptar_fp_project");
}

int ptar_fp_reduce_fap(const double* amps, int32_t nreal, const ptar_fp_model* fp, double* Fp, double* Fp_max,
                       int64_t* Fp_argmax, double* fap, void* stream) {
  if (!amps || !fp || !Fp || !Fp_max || !Fp_argmax || nreal <= 0) return fail(-1, "ptar_fp_reduce: bad argument%s");
  if (int rc = fp_model_check(fp, "ptar_fp_reduce")) return rc;
  if (reinterpret_cast<uintptr_t>(amps) & 15) return fail(-2, "ptar_fp_reduce: amps must be 16-byte aligned%s");
  ptar::fp_reduce_kernel<<<static_cast<unsigned>(nreal), ptar::FP_REDUCE_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      amps, nreal, *fp, Fp, Fp_max, Fp_argmax, fap);
  return check_launch("ptar_fp_reduce");
}

int ptar_fp_reduce(const double* amps, int32_t nreal, const ptar_fp_model* fp, double* Fp, double* Fp_max,
                   int64_t* Fp_argmax, void* stream) {
  return ptar_fp_reduce_fap(amps, nreal, fp, Fp, Fp_max, Fp_argmax, nullptr, stream);
}

int ptar_fe_sky(const double* amps, int32_t nreal, const ptar_fe_model* fe, double* fmax, int64_t* fargmax, double* maps,
                void* stream) {
  if (!amps || !fe || !fmax || !fargmax || nreal <= 0) return fail(-1, "ptar_fe_sky: bad argument%s");
  if (int rc = sky_model_check(fe, fe->Lf, nullptr, "ptar_fe_sky")) return rc;
  if (fe->n_freq < 1 || fe->n_freq > PTAR_FP_MAX_FREQ) return fail(-2, "ptar_fe_sky: need 1 <= n_freq <= 256%s");
  if (reinterpret_cast<uintptr_t>(amps) & 15) return fail(-2, "ptar_fe_sky: amps must be 16-byte aligned%s");
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::fe_sky_kernel, optin, ptar::fe_smem_bytes(PTAR_FE_MAX_PSR), "ptar_fe_sky")) return rc;
  const dim3 grid(static_cast<unsigned>((nreal + ptar::FE_RB - 1) / ptar::FE_RB), static_cast<unsigned>(fe->n_freq));
  ptar::fe_sky_kernel<<<grid, ptar::FE_THREADS, ptar::fe_smem_bytes(fe->kp), static_cast<cudaStream_t>(stream)>>>(
      amps, nreal, *fe, fmax, fargmax, maps);
  return check_launch("ptar_fe_sky");
}

int ptar_fe_combine(const double* fmax, const int64_t* fargmax, int32_t nreal, const ptar_fe_model* fe, double* fe_max,
                    int64_t* argmax_f, int64_t* argmax_sky, void* stream) {
  if (!fmax || !fargmax || !fe || !fe_max || !argmax_f || !argmax_sky || nreal <= 0)
    return fail(-1, "ptar_fe_combine: bad argument%s");
  if (int rc = sky_model_check(fe, fe->Lf, nullptr, "ptar_fe_combine")) return rc;
  if (fe->n_freq < 1 || fe->n_freq > PTAR_FP_MAX_FREQ) return fail(-2, "ptar_fe_combine: need 1 <= n_freq <= 256%s");
  const unsigned blocks = static_cast<unsigned>((nreal + ptar::FE_COMBINE_THREADS - 1) / ptar::FE_COMBINE_THREADS);
  ptar::fe_combine_kernel<<<blocks, ptar::FE_COMBINE_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      fmax, fargmax, nreal, fe->n_freq, fe_max, argmax_f, argmax_sky);
  return check_launch("ptar_fe_combine");
}

int ptar_bwm_sky(const double* amps, int32_t nreal, const ptar_bwm_model* bw, double* t0max, int64_t* t0argmax,
                 double* maps, void* stream) {
  if (!amps || !bw || !t0max || !t0argmax || nreal <= 0) return fail(-1, "ptar_bwm_sky: bad argument%s");
  if (int rc = sky_model_check(bw, bw->sqm && bw->seen && bw->antenna, bw->sqm, "ptar_bwm_sky")) return rc;
  if (bw->n_t0 < 1 || bw->n_t0 > PTAR_BWM_MAX_EPOCH) return fail(-2, "ptar_bwm_sky: need 1 <= n_t0 <= 512%s");
  if (reinterpret_cast<uintptr_t>(amps) & 15) return fail(-2, "ptar_bwm_sky: amps must be 16-byte aligned%s");
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::bwm_sky_kernel, optin, ptar::sky_smem_bytes(PTAR_FE_MAX_PSR, ptar::BWM_LINV),
                           "ptar_bwm_sky"))
    return rc;
  const dim3 grid(static_cast<unsigned>((nreal + ptar::FE_RB - 1) / ptar::FE_RB), static_cast<unsigned>((bw->n_t0 + 1) / 2));
  ptar::bwm_sky_kernel<<<grid, ptar::FE_THREADS, ptar::sky_smem_bytes(bw->kp, ptar::BWM_LINV),
                         static_cast<cudaStream_t>(stream)>>>(amps, nreal, *bw, t0max, t0argmax, maps);
  return check_launch("ptar_bwm_sky");
}

int ptar_bwm_combine(const double* amps, const double* t0max, const int64_t* t0argmax, int32_t nreal,
                     const ptar_bwm_model* bw, double* bwm_max, int64_t* argmax_t0, int64_t* argmax_sky, double* strain,
                     double* pol, double* fap, double* psr_max, int64_t* psr_argmax_t0, double* psr_slope,
                     double* psr_fap, void* stream) {
  if (!amps || !t0max || !t0argmax || !bw || !bwm_max || !argmax_t0 || !argmax_sky || !strain || !pol || !fap ||
      !psr_max || !psr_argmax_t0 || !psr_slope || !psr_fap || nreal <= 0)
    return fail(-1, "ptar_bwm_combine: bad argument%s");
  if (int rc = sky_model_check(bw, bw->sqm && bw->seen && bw->antenna, bw->sqm, "ptar_bwm_combine")) return rc;
  if (bw->n_t0 < 1 || bw->n_t0 > PTAR_BWM_MAX_EPOCH) return fail(-2, "ptar_bwm_combine: need 1 <= n_t0 <= 512%s");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int T = ptar::BWM_COMBINE_THREADS;
  ptar::bwm_combine_kernel<<<static_cast<unsigned>((nreal + T - 1) / T), T, 0, st>>>(
      amps, t0max, t0argmax, nreal, *bw, bwm_max, argmax_t0, argmax_sky, strain, pol, fap);
  if (int rc = check_launch("ptar_bwm_combine")) return rc;
  const int64_t n = int64_t(nreal) * bw->n_psr;
  ptar::bwm_psr_kernel<<<static_cast<unsigned>((n + T - 1) / T), T, 0, st>>>(amps, nreal, *bw, psr_max, psr_argmax_t0,
                                                                            psr_slope, psr_fap);
  return check_launch("ptar_bwm_combine (pulsar term)");
}

static int burst_model_check(const ptar_burst_model* bm, const char* what) {
  if (!bm->t || !bm->dinv || !bm->run_start || !bm->run_len || !bm->run_coef || !bm->toa_run || !bm->tmpl || !bm->win || !bm->blk || !bm->H ||
      !bm->wl || !bm->Lf || !bm->linv || !bm->antenna || !bm->seen || !bm->psr_order || !bm->seg_off)
    return fail(-2, "%s: model arrays missing", what);
  if (bm->n_psr < 2 || bm->n_psr > PTAR_FE_MAX_PSR || bm->n_tmpl < 1 || bm->n_tmpl > PTAR_BURST_MAX_TEMPLATE ||
      bm->n_zc < 2 || (bm->n_zc & 1) || bm->n_run < 1)
    return fail(-2, "%s: need 2 <= n_psr <= 128, 1 <= n_tmpl <= 4096, an even n_zc >= 2 and n_run >= 1", what);
  if (bm->n_sky < 1 || bm->n_sky > PTAR_FE_MAX_SKY || bm->n_sb != (bm->n_sky + ptar::FE_SB - 1) / ptar::FE_SB)
    return fail(-2, "%s: need 1 <= n_sky <= 12288 and n_sb = ceil(n_sky / 32)", what);
  if ((reinterpret_cast<uintptr_t>(bm->win) | reinterpret_cast<uintptr_t>(bm->blk)) & 7)
    return fail(-2, "%s: win and blk must be 8-byte aligned", what);
  return 0;
}

int ptar_burst_ninv(const double* rows, int64_t ld, int32_t nreal, const ptar_burst_model* bm, double* y, void* stream) {
  if (!rows || !bm || !y || nreal <= 0 || ld <= 0) return fail(-1, "ptar_burst_ninv: bad argument%s");
  if (int rc = burst_model_check(bm, "ptar_burst_ninv")) return rc;
  const dim3 grid(static_cast<unsigned>((ld + ptar::BU_NINV_THREADS - 1) / ptar::BU_NINV_THREADS),
                  static_cast<unsigned>(std::min(nreal, 65535)));
  ptar::burst_ninv_kernel<<<grid, ptar::BU_NINV_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(rows, ld, nreal, *bm, y);
  return check_launch("ptar_burst_ninv");
}

int ptar_burst_project(const double* y, int64_t ld, int32_t nreal, const double* z, const ptar_burst_model* bm, int32_t group,
                       double* amps, void* stream) {
  if (!y || !z || !bm || !amps || nreal <= 0 || ld <= 0) return fail(-1, "ptar_burst_project: bad argument%s");
  if (int rc = burst_model_check(bm, "ptar_burst_project")) return rc;
  if (group < 0 || group * PTAR_BURST_GROUP >= bm->n_tmpl) return fail(-2, "ptar_burst_project: group out of range%s");
  if ((ld & 3) || (reinterpret_cast<uintptr_t>(y) & 31) || (reinterpret_cast<uintptr_t>(amps) & 15))
    return fail(-2, "ptar_burst_project: y must be 32-byte aligned with ld %% 4 == 0, amps 16-byte aligned%s");
  const int jg = std::min(PTAR_BURST_GROUP, bm->n_tmpl - group * PTAR_BURST_GROUP);
  const int64_t blocks =
      int64_t(bm->n_psr) * ((nreal + ptar::OS_RB - 1) / ptar::OS_RB) * ((jg + ptar::BU_TB - 1) / ptar::BU_TB);
  if (blocks > 0x7fffffff) return fail(-3, "ptar_burst_project: grid too large%s");
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::burst_project_kernel, optin, ptar::BU_SMEM, "ptar_burst_project")) return rc;
  ptar::burst_project_kernel<<<static_cast<unsigned>(blocks), ptar::BU_THREADS, ptar::BU_SMEM,
                               static_cast<cudaStream_t>(stream)>>>(y, ld, nreal, z, *bm, group, amps);
  return check_launch("ptar_burst_project");
}

int ptar_burst_reduce(const double* amps, const double* jmax, const int64_t* jargmax, int32_t nreal, const ptar_burst_model* bm,
                      double* B_tmpl, int64_t* B_tmpl_sky, double* B_max, int64_t* argmax_tmpl, int64_t* argmax_sky,
                      double* fap, double* amp, double* Bt_max, int64_t* argmax_psr, double* fap_psr, double* amp_psr,
                      double* bt_maps, void* stream) {
  if (!amps || !jmax || !jargmax || !bm || !B_tmpl || !B_tmpl_sky || !B_max || !argmax_tmpl || !argmax_sky || !fap || !amp ||
      !Bt_max || !argmax_psr || !fap_psr || nreal <= 0)
    return fail(-1, "ptar_burst_reduce: bad argument%s");
  if (int rc = burst_model_check(bm, "ptar_burst_reduce")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int T = ptar::BU_REDUCE_THREADS;
  ptar::burst_reduce_kernel<<<static_cast<unsigned>((nreal + T - 1) / T), T, 0, st>>>(
      amps, jmax, jargmax, nreal, *bm, B_tmpl, B_tmpl_sky, B_max, argmax_tmpl, argmax_sky, fap, amp);
  if (int rc = check_launch("ptar_burst_reduce")) return rc;
  const int64_t n = int64_t(nreal) * bm->n_psr;
  ptar::burst_psr_kernel<<<static_cast<unsigned>((n + T - 1) / T), T, 0, st>>>(amps, nreal, *bm, Bt_max, argmax_psr, fap_psr,
                                                                             amp_psr, bt_maps);
  return check_launch("ptar_burst_reduce (per pulsar)");
}

static int curn_grid_check(const ptar_curn_model* cm, const char* what) {
  if (!cm->log10_A || !cm->wg || !cm->wx || !cm->prior) return fail(-2, "%s: model arrays missing", what);
  if (!grid_ok(cm->n_amp, cm->n_gamma))
    return fail(-2, "%s: need 2 <= n_amp <= 256 and 1 <= n_gamma <= 256", what);
  if (!(cm->ul > 0.0 && cm->ul < 1.0)) return fail(-2, "%s: need 0 < ul < 1", what);
  return 0;
}

int ptar_curn_grid(const double* X, int32_t nreal, const ptar_curn_model* cm, double* lnL, void* stream) {
  if (!X || !cm || !lnL || nreal <= 0) return fail(-1, "ptar_curn_grid: bad argument%s");
  if (!cm->V || !cm->lam || !cm->a2 || !cm->ldet || cm->n_psr <= 0) return fail(-2, "ptar_curn_grid: model arrays missing%s");
  if (!nc_ok(cm->nc, cm->ncp)) return fail(-2, "ptar_curn_grid: need 0 < nc <= 32 and ncp = nc rounded up to a multiple of 8%s");
  if (int rc = curn_grid_check(cm, "ptar_curn_grid")) return rc;
  if ((reinterpret_cast<uintptr_t>(X) & 31) || (reinterpret_cast<uintptr_t>(cm->V) & 15))
    return fail(-2, "ptar_curn_grid: X must be 32-byte aligned, V 16-byte aligned%s");
  const int64_t nrb = (int64_t(nreal) + ptar::CURN_RB - 1) / ptar::CURN_RB;
  if (nrb > 65535) return fail(-3, "ptar_curn_grid: more than 65535 realization blocks%s");
  const dim3 grid(static_cast<unsigned>((cm->n_amp + ptar::CURN_AB - 1) / ptar::CURN_AB), static_cast<unsigned>(nrb),
                  static_cast<unsigned>(cm->n_gamma));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static SmemOptIn optin[4];
  switch (cm->ncp / 8) {
#define PTAR_CURN_LAUNCH(NT)                                                                                           \
  case NT:                                                                                                             \
    if (int rc = opt_in_smem(ptar::curn_grid_kernel<NT>, optin[NT - 1], ptar::CURN_SMEM, "ptar_curn_grid")) return rc; \
    ptar::curn_grid_kernel<NT><<<grid, ptar::CURN_THREADS, ptar::CURN_SMEM, st>>>(X, nreal, *cm, lnL);                 \
    break;
    PTAR_CURN_LAUNCH(1)
    PTAR_CURN_LAUNCH(2)
    PTAR_CURN_LAUNCH(3)
    PTAR_CURN_LAUNCH(4)
#undef PTAR_CURN_LAUNCH
  }
  return check_launch("ptar_curn_grid");
}

int ptar_curn_reduce(const double* lnL, int32_t nreal, const ptar_curn_model* cm, double* lnL_max, int64_t* ml_gamma,
                     int64_t* ml_amp, double* ln_bayes, double* post_amp, double* post_gamma, double* ul_amp,
                     void* stream) {
  if (!lnL || !cm || !lnL_max || !ml_gamma || !ml_amp || !ln_bayes || !post_amp || !post_gamma || !ul_amp || nreal <= 0)
    return fail(-1, "ptar_curn_reduce: bad argument%s");
  if (int rc = curn_grid_check(cm, "ptar_curn_reduce")) return rc;
  ptar::curn_reduce_kernel<<<static_cast<unsigned>(nreal), ptar::CURN_RED_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      lnL, nreal, *cm, lnL_max, ml_gamma, ml_amp, ln_bayes, post_amp, post_gamma, ul_amp);
  return check_launch("ptar_curn_reduce");
}

int ptar_hd_grid(const double* X, int32_t nreal, const ptar_hd_model* hm, double* lnL, void* stream) {
  if (!X || !hm || !lnL || nreal <= 0) return fail(-1, "ptar_hd_grid: bad argument%s");
  if (!hm->V || !hm->lam || !hm->a2 || !hm->ldet || hm->n_psr <= 0) return fail(-2, "ptar_hd_grid: model arrays missing%s");
  if (!nc_ok(hm->nc, hm->ncp))
    return fail(-2, "ptar_hd_grid: need 0 < nc <= 32 and ncp = nc rounded up to a multiple of 8%s");
  if (int64_t(hm->n) != int64_t(hm->n_psr) * hm->nc || hm->n > PTAR_HD_MAX_N ||
      hm->np != (hm->n + PTAR_HD_JB - 1) / PTAR_HD_JB * PTAR_HD_JB)
    return fail(-2, "ptar_hd_grid: need n = n_psr nc <= 4096 and np = n rounded up to a multiple of 32%s");
  if (!grid_ok(hm->n_amp, hm->n_gamma))
    return fail(-2, "ptar_hd_grid: need 2 <= n_amp <= 256 and 1 <= n_gamma <= 256%s");
  if ((reinterpret_cast<uintptr_t>(X) & 31) || (reinterpret_cast<uintptr_t>(hm->V) & 15))
    return fail(-2, "ptar_hd_grid: X must be 32-byte aligned, V 16-byte aligned%s");
  const int64_t nrb = (int64_t(nreal) + ptar::HD_RB - 1) / ptar::HD_RB;
  const dim3 grid(static_cast<unsigned>(nrb), static_cast<unsigned>(hm->n_gamma));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static SmemOptIn optin[3];
  const int qn = hm->n_amp <= 64 ? 4 : hm->n_amp <= 128 ? 8 : 16;   // 16 QN amplitude columns per CTA
  switch (qn) {
#define PTAR_HD_LAUNCH(QN, I)                                                                                           \
  case QN:                                                                                                              \
    if (int rc = opt_in_smem(ptar::hd_grid_kernel<QN>, optin[I], ptar::hd_smem(QN), "ptar_hd_grid")) return rc;        \
    ptar::hd_grid_kernel<QN><<<grid, ptar::HD_THREADS, ptar::hd_smem(QN), st>>>(X, nreal, *hm, lnL);                    \
    break;
    PTAR_HD_LAUNCH(4, 0)
    PTAR_HD_LAUNCH(8, 1)
    PTAR_HD_LAUNCH(16, 2)
#undef PTAR_HD_LAUNCH
  }
  return check_launch("ptar_hd_grid");
}

int ptar_rn_grid(const double* X, int32_t nreal, const ptar_rn_model* rm, double* lnL, void* stream) {
  if (!X || !rm || !lnL || nreal <= 0) return fail(-1, "ptar_rn_grid: bad argument%s");
  if (!rm->V || !rm->lam || !rm->a2 || !rm->ldet || rm->n_psr <= 0) return fail(-2, "ptar_rn_grid: model arrays missing%s");
  if (!nc_ok(rm->nc, rm->ncp, PTAR_RN_MAX_NC))
    return fail(-2, "ptar_rn_grid: need 0 < nc <= 64 and ncp = nc rounded up to a multiple of 8%s");
  if (!grid_ok(rm->n_amp, rm->n_gamma))
    return fail(-2, "ptar_rn_grid: need 2 <= n_amp <= 256 and 1 <= n_gamma <= 256%s");
  if ((reinterpret_cast<uintptr_t>(X) & 31) || (reinterpret_cast<uintptr_t>(rm->V) & 15))
    return fail(-2, "ptar_rn_grid: X must be 32-byte aligned, V 16-byte aligned%s");
  const int64_t nrb = (int64_t(nreal) + ptar::RN_RB - 1) / ptar::RN_RB;
  const int64_t nz = int64_t(rm->n_psr) * ((rm->n_gamma + ptar::RN_GB - 1) / ptar::RN_GB);
  if (nrb > 65535 || nz > 65535)
    return fail(-3, "ptar_rn_grid: more than 65535 realization blocks or (pulsar, 16-gamma group) pairs%s");
  const dim3 grid(static_cast<unsigned>((rm->n_amp + ptar::RN_AB - 1) / ptar::RN_AB), static_cast<unsigned>(nrb),
                  static_cast<unsigned>(nz));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static SmemOptIn optin[8];
  switch (rm->ncp / 8) {
#define PTAR_RN_LAUNCH(NT)                                                                                       \
  case NT:                                                                                                       \
    if (int rc = opt_in_smem(ptar::rn_grid_kernel<NT>, optin[NT - 1], ptar::RN_SMEM, "ptar_rn_grid")) return rc; \
    ptar::rn_grid_kernel<NT><<<grid, ptar::RN_THREADS, ptar::RN_SMEM, st>>>(X, nreal, *rm, lnL);                 \
    break;
    PTAR_RN_LAUNCH(1)
    PTAR_RN_LAUNCH(2)
    PTAR_RN_LAUNCH(3)
    PTAR_RN_LAUNCH(4)
    PTAR_RN_LAUNCH(5)
    PTAR_RN_LAUNCH(6)
    PTAR_RN_LAUNCH(7)
    PTAR_RN_LAUNCH(8)
#undef PTAR_RN_LAUNCH
  }
  return check_launch("ptar_rn_grid");
}

static int run_job(const ptar_job* job, const ptar_timing_model* tm, const ptar_chrom_model* cm, double* scratch,
                   int64_t scratch_len, int64_t real0, int32_t nreal, double* out, void* stream);

int ptar_run_job_tm(const ptar_job* job, const ptar_timing_model* tm, double* scratch, int64_t scratch_len, int64_t real0,
                    int32_t nreal, double* out, void* stream) {
  return run_job(job, tm, nullptr, scratch, scratch_len, real0, nreal, out, stream);
}

static int run_job(const ptar_job* job, const ptar_timing_model* tm, const ptar_chrom_model* cm, double* scratch,
                   int64_t scratch_len, int64_t real0, int32_t nreal, double* out, void* stream) {
  if (!job || !out || nreal <= 0) return fail(-1, "ptar_run_job: bad argument%s");
  ptar_gen_params g = job->gen;
  g.real0 = real0;
  g.nreal = nreal;
  g.out = out;
  const bool inject = g.z1 || g.z2 || g.zb || g.zrn || job->gwb_zin || (cm && cm->zchr);
  if (g.flags & PTAR_F_GWB) {
    if (!job->M || !job->A || !job->Zm || !job->Gbuf || !job->tile_list || !job->knots)
      return fail(-2, "ptar_run_job: GWB buffers missing%s");
    const bool i8 = job->AS && !inject;
    int rc = 0;
    if (i8 && g.n_psr <= 8 * ptar::MX_MAXNT) {   // mixing emits the digit slices directly
      if (!job->ZS || !job->zinv) return fail(-2, "ptar_run_job: int8 GWB buffers missing%s");
      rc = ptar_gwb_mix_i8(job->ZS, job->M, job->zinv, g.n_psr, job->Jg, job->Jpad, nreal, job->rcap, g.seed, real0, stream);
    } else {
      rc = ptar_gwb_mix(job->Zm, job->M, inject ? job->gwb_zin : nullptr, g.n_psr, job->Jg, nreal, g.seed, real0, stream);
      if (!rc && i8) {
        if (!job->ZS || !job->zinv) return fail(-2, "ptar_run_job: int8 GWB buffers missing%s");
        rc = ptar_gwb_slice_i8(job->ZS, job->Zm, job->zinv, g.n_psr, job->Jg, job->Jpad, nreal, job->rcap, stream);
      }
    }
    if (rc) return rc;
    if (i8) {   // int8 tensor-core path: exact int8 GEMMs on the digit slices, fp64 fix-up
      if (!job->colscale || !job->zscale || !job->tile_list_i8) return fail(-2, "ptar_run_job: int8 GWB buffers missing%s");
      rc = ptar_gwb_synth_i8(job->Gbuf, g.g_ld, g.g_ldr, job->AS, job->colscale, job->ZS, job->zscale, g.n_psr, job->Jg, job->Jpad, nreal,
                             job->rcap, job->tile_list_i8, job->n_syn_tiles_i8, stream);
    } else {
      rc = ptar_gwb_synth(job->Gbuf, g.g_ld, g.g_ldr, job->A, job->lda, job->Zm, job->Jg, nreal, job->tile_list, job->n_syn_tiles,
                          job->knots, job->lower_tri, stream);
    }
    if (rc) return rc;
    g.G = job->Gbuf;
  }
  if (int rc = ptar_generate_chrom(&g, cm, stream)) return rc;
  if (tm) return ptar_timing_project(out, g.ld_out, nreal, tm, scratch, scratch_len, stream);
  return 0;
}

int ptar_run_job(const ptar_job* job, int64_t real0, int32_t nreal, double* out, void* stream) {
  return ptar_run_job_tm(job, nullptr, nullptr, 0, real0, nreal, out, stream);
}

int ptar_run_job_to_host_tm(const ptar_job* job, const ptar_timing_model* tm, double* scratch, int64_t scratch_len,
                            int64_t real0, int64_t nreal, int32_t chunk, double* out_host, double* dev_buf0,
                            double* dev_buf1, void* stream0, void* stream1) {
  return ptar_run_job_to_host_chrom(job, tm, nullptr, scratch, scratch_len, real0, nreal, chunk, out_host, dev_buf0, dev_buf1,
                                    stream0, stream1);
}

int ptar_run_job_to_host_chrom(const ptar_job* job, const ptar_timing_model* tm, const ptar_chrom_model* cm, double* scratch,
                               int64_t scratch_len, int64_t real0, int64_t nreal, int32_t chunk, double* out_host,
                               double* dev_buf0, double* dev_buf1, void* stream0, void* stream1) {
  if (!job || !out_host || !dev_buf0 || !dev_buf1 || chunk <= 0 || (chunk & 3) || nreal <= 0)
    return fail(-1, "ptar_run_job_to_host: bad argument (chunk must be a positive multiple of 4)%s");
  cudaStream_t s0 = static_cast<cudaStream_t>(stream0), s1 = static_cast<cudaStream_t>(stream1);
  cudaEvent_t gen_done[2] = {nullptr, nullptr}, copy_done[2] = {nullptr, nullptr};
  int rc = 0;
  cudaError_t e = cudaSuccess;
  auto ok = [&](cudaError_t r) {  // first runtime error wins; later calls are skipped
    if (e == cudaSuccess && r != cudaSuccess) e = r;
    return e == cudaSuccess;
  };
  for (int i = 0; i < 2; ++i) {
    ok(cudaEventCreateWithFlags(&gen_done[i], cudaEventDisableTiming));
    ok(cudaEventCreateWithFlags(&copy_done[i], cudaEventDisableTiming));
  }
  double* bufs[2] = {dev_buf0, dev_buf1};
  const int64_t ld = job->gen.ld_out;
  int64_t done = 0;
  for (int c = 0; done < nreal && e == cudaSuccess; ++c) {
    const int b = c & 1;
    const int32_t n = static_cast<int32_t>(nreal - done < chunk ? nreal - done : chunk);
    if (c >= 2 && !ok(cudaStreamWaitEvent(s0, copy_done[b], 0))) break;  // buffer free again
    ptar_job j = *job;
    if (j.gen.z1) j.gen.z1 += done * ld;
    if (j.gen.z2) j.gen.z2 += done * ld;
    if (j.gen.zb) j.gen.zb += done * j.gen.n_bucket_total;
    if (j.gen.zrn) j.gen.zrn += done * int64_t(j.gen.n_psr) * j.gen.J;
    if (j.gwb_zin) j.gwb_zin += done * int64_t(j.gen.n_psr) * j.Jg;
    ptar_chrom_model cmc;
    if (cm) {
      cmc = *cm;
      int zld = 0;
      for (int s = 0; s < cmc.n_slot && s < PTAR_CHROM_SLOTS; ++s) zld += cmc.J[s];
      if (cmc.zchr) cmc.zchr += done * int64_t(j.gen.n_psr) * zld;
    }
    rc = run_job(&j, tm, cm ? &cmc : nullptr, scratch, scratch_len, real0 + done, n, bufs[b], s0);
    if (rc) break;
    if (!ok(cudaEventRecord(gen_done[b], s0)) || !ok(cudaStreamWaitEvent(s1, gen_done[b], 0))) break;
    if (!ok(cudaMemcpyAsync(out_host + done * ld, bufs[b], sizeof(double) * size_t(n) * ld, cudaMemcpyDeviceToHost, s1))) break;
    if (!ok(cudaEventRecord(copy_done[b], s1))) break;
    done += n;
  }
  // drain both streams even after an error so no copy is still writing out_host when we return
  const cudaError_t d1 = cudaStreamSynchronize(s1), d0 = cudaStreamSynchronize(s0);
  ok(d1);
  ok(d0);
  for (int i = 0; i < 2; ++i) {
    if (gen_done[i]) cudaEventDestroy(gen_done[i]);
    if (copy_done[i]) cudaEventDestroy(copy_done[i]);
  }
  if (rc) return rc;
  ok(cudaGetLastError());
  if (e != cudaSuccess) return fail(-100, "ptar_run_job_to_host: %s", cudaGetErrorString(e));
  return 0;
}

int ptar_run_job_to_host(const ptar_job* job, int64_t real0, int64_t nreal, int32_t chunk, double* out_host,
                         double* dev_buf0, double* dev_buf1, void* stream0, void* stream1) {
  return ptar_run_job_to_host_tm(job, nullptr, nullptr, 0, real0, nreal, chunk, out_host, dev_buf0, dev_buf1, stream0, stream1);
}

int ptar_fs_grid(const double* X, int32_t nreal, const ptar_fs_model* fm, double* lnL, void* stream) {
  if (!X || !fm || !lnL || nreal <= 0) return fail(-1, "ptar_fs_grid: bad argument%s");
  if (!fm->V || !fm->lam || !fm->a2 || !fm->ldet) return fail(-2, "ptar_fs_grid: model arrays missing%s");
  if (fm->n_psr < 1 || fm->n_psr > PTAR_FS_MAX_PSR || fm->n_bin < 1 || fm->n_bin > PTAR_FS_MAX_BIN ||
      !nc_ok(2 * fm->n_bin, fm->ncp, PTAR_RN_MAX_NC))
    return fail(-2, "ptar_fs_grid: need 1 <= n_psr <= 256, 1 <= n_bin <= 32 and ncp = 2 n_bin rounded up to a multiple of 8%s");
  if (fm->n2p != ((2 * fm->n_psr + 7) & ~7) || fm->np != (2 * fm->n_psr + PTAR_FS_JB - 1) / PTAR_FS_JB * PTAR_FS_JB)
    return fail(-2, "ptar_fs_grid: need n2p = 2 n_psr rounded up to a multiple of 8 and np to a multiple of 32%s");
  if (!grid_ok(fm->n_amp, 1)) return fail(-2, "ptar_fs_grid: need 2 <= n_amp <= 256%s");
  if ((reinterpret_cast<uintptr_t>(X) & 31) || (reinterpret_cast<uintptr_t>(fm->V) & 15))
    return fail(-2, "ptar_fs_grid: X must be 32-byte aligned, V 16-byte aligned%s");
  const int64_t nrb = (int64_t(nreal) + ptar::FS_RB - 1) / ptar::FS_RB;
  if (nrb > 65535) return fail(-3, "ptar_fs_grid: more than 65535 realization blocks%s");
  const dim3 grid(static_cast<unsigned>((fm->n_amp + ptar::FS_AB - 1) / ptar::FS_AB), static_cast<unsigned>(nrb),
                  static_cast<unsigned>(fm->n_bin));
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::fs_grid_kernel, optin, ptar::FS_SMEM, "ptar_fs_grid")) return rc;
  ptar::fs_grid_kernel<<<grid, ptar::FS_THREADS, ptar::FS_SMEM, static_cast<cudaStream_t>(stream)>>>(X, nreal, *fm, lnL);
  return check_launch("ptar_fs_grid");
}

int ptar_fs_y2(const double* X, int32_t nreal, const ptar_fs_model* fm, double* y2, void* stream) {
  if (!X || !fm || !y2 || nreal <= 0) return fail(-1, "ptar_fs_y2: bad argument%s");
  if (!fm->V) return fail(-2, "ptar_fs_y2: model arrays missing%s");
  if (fm->n_psr < 1 || fm->n_psr > PTAR_FS_MAX_PSR || fm->n_bin < 1 || fm->n_bin > PTAR_FS_MAX_BIN ||
      !nc_ok(2 * fm->n_bin, fm->ncp, PTAR_RN_MAX_NC))
    return fail(-2, "ptar_fs_y2: need 1 <= n_psr <= 256, 1 <= n_bin <= 32 and ncp = 2 n_bin rounded up to a multiple of 8%s");
  if (fm->n2p != ((2 * fm->n_psr + 7) & ~7) || fm->np != (2 * fm->n_psr + PTAR_FS_JB - 1) / PTAR_FS_JB * PTAR_FS_JB)
    return fail(-2, "ptar_fs_y2: need n2p = 2 n_psr rounded up to a multiple of 8 and np to a multiple of 32%s");
  if ((reinterpret_cast<uintptr_t>(X) & 31) || (reinterpret_cast<uintptr_t>(fm->V) & 15) ||
      (reinterpret_cast<uintptr_t>(y2) & 15))
    return fail(-2, "ptar_fs_y2: X must be 32-byte aligned, V and y2 16-byte aligned%s");
  const int64_t nrb = (int64_t(nreal) + ptar::FS_RB - 1) / ptar::FS_RB;
  const dim3 grid(static_cast<unsigned>(nrb), static_cast<unsigned>(fm->n_bin));
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::fs_y2_kernel, optin, ptar::FS_Y2_SMEM, "ptar_fs_y2")) return rc;
  ptar::fs_y2_kernel<<<grid, ptar::FS_THREADS, ptar::FS_Y2_SMEM, static_cast<cudaStream_t>(stream)>>>(X, nreal, *fm, y2);
  return check_launch("ptar_fs_y2");
}

int ptar_fs_refit(const double* y2, int32_t nreal, const ptar_fs_refit_model* rm, double* lnL, void* stream) {
  if (!y2 || !rm || !lnL || nreal <= 0) return fail(-1, "ptar_fs_refit: bad argument%s");
  if (!rm->lam || !rm->rho2 || !rm->ldet) return fail(-2, "ptar_fs_refit: model arrays missing%s");
  if (rm->n_bin < 1 || rm->n_bin > PTAR_FS_MAX_BIN || rm->np < PTAR_FS_JB || rm->np > 2 * PTAR_FS_MAX_PSR ||
      rm->np % PTAR_FS_JB || rm->n_tmpl < 1 || rm->n_tmpl > PTAR_FS_MAX_TEMPLATE)
    return fail(-2, "ptar_fs_refit: need 1 <= n_bin <= 32, np a multiple of 32 in 32 .. 512 and 1 <= n_tmpl <= 65536%s");
  if (reinterpret_cast<uintptr_t>(y2) & 15) return fail(-2, "ptar_fs_refit: y2 must be 16-byte aligned%s");
  const int64_t nrb = (int64_t(nreal) + ptar::RF_RB - 1) / ptar::RF_RB;
  if (nrb > 65535) return fail(-3, "ptar_fs_refit: more than 65535 realization blocks%s");
  const dim3 grid(static_cast<unsigned>((rm->n_tmpl + ptar::RF_TB - 1) / ptar::RF_TB), static_cast<unsigned>(nrb));
  static SmemOptIn optin;
  if (int rc = opt_in_smem(ptar::fs_refit_kernel, optin, ptar::RF_SMEM, "ptar_fs_refit")) return rc;
  ptar::fs_refit_kernel<<<grid, ptar::RF_THREADS, ptar::RF_SMEM, static_cast<cudaStream_t>(stream)>>>(y2, nreal, *rm, lnL);
  return check_launch("ptar_fs_refit");
}

int ptar_cw_population_stage(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed, const ptar_cwpop_model* m,
                             double* scratch, int64_t scratch_len, double* params, int stage, void* stream) {
  if (int rc = population_check(rows, ld, nreal, real0, m, scratch, stage, "ptar_cw_population")) return rc;
  if (m->n_psr <= 0 || m->n_src < 1 || m->n_src > PTAR_CWPOP_MAX_SRC || m->mode < 0 || m->mode > 2 || !m->phat)
    return fail(-2, "ptar_cw_population: need n_psr >= 1, 1 <= n_src <= 64, mode 0..2 and phat%s");
  if (!m->pphase && !m->pdist) return fail(-2, "ptar_cw_population: pdist missing (no drawn pulsar phase)%s");
  for (int j = 0; j < PTAR_CWPOP_NPAR; ++j)
    if (m->kind[j] < PTAR_CWPOP_FIXED || m->kind[j] > PTAR_CWPOP_ACOS) return fail(-2, "ptar_cw_population: bad parameter kind%s");
  const int64_t pairs = int64_t(nreal) * m->n_src;
  if (scratch_len < pairs * (ptar::CWP_SRC + int64_t(ptar::CWP_PSR) * m->n_psr))
    return fail(-2, "ptar_cw_population: scratch too small (need nreal * n_src * (16 + 8 n_psr) doubles)%s");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* src = scratch;
  double* psr = scratch + pairs * ptar::CWP_SRC;
  if (stage != 2) {
    double* pph = params && m->pphase ? params + pairs * PTAR_CWPOP_TABLE : nullptr;
    ptar::cwpop_draw_kernel<<<static_cast<unsigned>((pairs + 127) / 128), 128, 0, st>>>(src, psr, params, pph, *m, nreal,
                                                                                        real0, seed);
    if (int rc = check_launch("ptar_cw_population (draw)")) return rc;
  }
  if (!rows || stage == 1) return 0;
  dim3 grid;
  if (int rc = population_add_grid(ld, nreal, ptar::CWP_TOAS, ptar::CWP_RB, &grid, "ptar_cw_population")) return rc;
  if (m->mode == 0)
    ptar::cwpop_add_kernel<0><<<grid, ptar::CWP_TOAS, 0, st>>>(rows, ld, nreal, src, psr, m->slot_t, m->slot_psr, m->n_psr,
                                                               m->n_src, m->psr_term);
  else if (m->mode == 1)
    ptar::cwpop_add_kernel<1><<<grid, ptar::CWP_TOAS, 0, st>>>(rows, ld, nreal, src, psr, m->slot_t, m->slot_psr, m->n_psr,
                                                               m->n_src, m->psr_term);
  else
    ptar::cwpop_add_kernel<2><<<grid, ptar::CWP_TOAS, 0, st>>>(rows, ld, nreal, src, psr, m->slot_t, m->slot_psr, m->n_psr,
                                                               m->n_src, m->psr_term);
  return check_launch("ptar_cw_population (add)");
}

int ptar_cw_population(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed, const ptar_cwpop_model* m,
                       double* scratch, int64_t scratch_len, double* params, void* stream) {
  return ptar_cw_population_stage(rows, ld, nreal, real0, seed, m, scratch, scratch_len, params, 0, stream);
}

int ptar_common_population_stage(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed,
                                 const ptar_cpop_model* m, double* scratch, int64_t scratch_len, double* params, int stage,
                                 void* stream) {
  if (int rc = population_check(rows, ld, nreal, real0, m, scratch, stage, "ptar_common_population")) return rc;
  if (m->n_psr < 1 || m->n_psr > PTAR_CPOP_MAX_PSR || m->K < 1 || m->K > PTAR_CPOP_MAX_K || !m->freqs)
    return fail(-2, "ptar_common_population: need 1 <= n_psr <= 2048, 1 <= K <= 32 and freqs%s");
  if (m->spectrum != PTAR_CPOP_POWERLAW && m->spectrum != PTAR_CPOP_FREE) return fail(-2, "ptar_common_population: bad spectrum%s");
  if (m->spectrum == PTAR_CPOP_POWERLAW && !m->pl_x) return fail(-2, "ptar_common_population: the power law needs pl_x%s");
  for (int j = 0; j < 2; ++j)
    if (m->kind[j] != PTAR_CWPOP_FIXED && m->kind[j] != PTAR_CWPOP_UNIFORM) return fail(-2, "ptar_common_population: bad parameter kind%s");
  const int64_t per_real = int64_t(m->n_psr) * 2 * m->K;
  if (scratch_len < nreal * per_real) return fail(-2, "ptar_common_population: scratch too small (need nreal * n_psr * 2K doubles)%s");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (stage != 2) {
    const int64_t ctas = int64_t(nreal) * m->K;
    if (ctas > INT32_MAX) return fail(-3, "ptar_common_population: too many realizations per call%s");
    ptar::cpop_draw_kernel<<<static_cast<unsigned>(ctas), ptar::CPOP_DRAW_THREADS, 2 * m->n_psr * sizeof(double), st>>>(
        scratch, params, *m, real0, seed);
    if (int rc = check_launch("ptar_common_population (draw)")) return rc;
  }
  if (!rows || stage == 1) return 0;
  dim3 grid;
  if (int rc = population_add_grid(ld, nreal, ptar::CPOP_TOAS, ptar::CPOP_RB, &grid, "ptar_common_population")) return rc;
  if (m->K <= 8)
    ptar::cpop_add_kernel<8><<<grid, ptar::CPOP_TOAS, 0, st>>>(rows, ld, nreal, scratch, m->freqs, m->slot_t, m->slot_psr,
                                                              m->n_psr, m->K);
  else if (m->K <= 16)
    ptar::cpop_add_kernel<16><<<grid, ptar::CPOP_TOAS, 0, st>>>(rows, ld, nreal, scratch, m->freqs, m->slot_t, m->slot_psr,
                                                               m->n_psr, m->K);
  else
    ptar::cpop_add_kernel<32><<<grid, ptar::CPOP_TOAS, 0, st>>>(rows, ld, nreal, scratch, m->freqs, m->slot_t, m->slot_psr,
                                                               m->n_psr, m->K);
  return check_launch("ptar_common_population (add)");
}

int ptar_common_population(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed, const ptar_cpop_model* m,
                           double* scratch, int64_t scratch_len, double* params, void* stream) {
  return ptar_common_population_stage(rows, ld, nreal, real0, seed, m, scratch, scratch_len, params, 0, stream);
}

int ptar_transient_population_stage(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed,
                                    const ptar_tpop_model* m, double* scratch, int64_t scratch_len, double* params, int stage,
                                    void* stream) {
  if (int rc = population_check(rows, ld, nreal, real0, m, scratch, stage, "ptar_transient_population")) return rc;
  if (m->family != PTAR_TPOP_BWM && m->family != PTAR_TPOP_BURST) return fail(-2, "ptar_transient_population: bad family%s");
  if (m->n_psr <= 0 || m->n_src < 1 || m->n_src > PTAR_TPOP_MAX_SRC || !m->phat)
    return fail(-2, "ptar_transient_population: need n_psr >= 1, 1 <= n_src <= 64 and phat%s");
  for (int j = 0; j < PTAR_TPOP_NPAR; ++j)
    if (m->kind[j] < PTAR_CWPOP_FIXED || m->kind[j] > PTAR_CWPOP_ACOS)
      return fail(-2, "ptar_transient_population: bad parameter kind%s");
  const int64_t pairs = int64_t(nreal) * m->n_src;
  if (scratch_len < pairs * (ptar::TP_REC + int64_t(ptar::TP_COEF) * m->n_psr))
    return fail(-2, "ptar_transient_population: scratch too small (need nreal * n_src * (4 + 2 n_psr) doubles)%s");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* rec = scratch;
  double* coef = scratch + pairs * ptar::TP_REC;
  if (stage != 2) {
    ptar::tpop_draw_kernel<<<static_cast<unsigned>((pairs + 127) / 128), 128, 0, st>>>(rec, coef, params, *m, nreal, real0,
                                                                                       seed);
    if (int rc = check_launch("ptar_transient_population (draw)")) return rc;
  }
  if (!rows || stage == 1) return 0;
  dim3 grid;
  if (int rc = population_add_grid(ld, nreal, ptar::TP_TOAS, ptar::TP_RB, &grid, "ptar_transient_population")) return rc;
  if (m->family == PTAR_TPOP_BWM)
    ptar::tpop_add_kernel<PTAR_TPOP_BWM><<<grid, ptar::TP_TOAS, 0, st>>>(rows, ld, nreal, rec, coef, m->slot_t, m->slot_psr,
                                                                         m->n_psr, m->n_src);
  else
    ptar::tpop_add_kernel<PTAR_TPOP_BURST><<<grid, ptar::TP_TOAS, 0, st>>>(rows, ld, nreal, rec, coef, m->slot_t,
                                                                           m->slot_psr, m->n_psr, m->n_src);
  return check_launch("ptar_transient_population (add)");
}

int ptar_transient_population(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed, const ptar_tpop_model* m,
                              double* scratch, int64_t scratch_len, double* params, void* stream) {
  return ptar_transient_population_stage(rows, ld, nreal, real0, seed, m, scratch, scratch_len, params, 0, stream);
}

}  // extern "C"

// Per-realization continuous-wave populations (ptar_cw_population): every realization gets its own n_src sources, drawn
// on the device from the priors of a ptar_cwpop_model and added to its row of residuals.
//
// cwpop_draw_kernel  one thread per (realization, source).  Draws the 8 source parameters from the Philox stream
//                    PTAR_K_CWPOP (counter layout in ptar_rng.cuh), derives the luminosity distance from h0, and writes
//                      src[r][s][16]   = {w0, fac1, fac2, fac3, phase0/2, w0^-5/3, incfac1, incfac2, cos 2psi, sin 2psi,
//                                         alpha = fac3 / cbrt(w0), 0...}   (cw_prefactor_kernel's layout + alpha)
//                      psr[r][s][p][8] = {F+, Fx, cosMu, pd [s], m0, m1, m2, 0}
//                    with the per-pulsar constants of the mode hoisted out of the TOA loop:
//                      mode 1 (phase_approx): m0 = omega_p, m1 = phase0/2 + fac2 (w0^-5/3 - omega_p^-5/3), m2 = fac3 / cbrt(omega_p)
//                      mode 2 (monochromatic): m0 = cos delta, m1 = sin delta, delta = 2 w0 pd (1 - cosMu), so that the
//                                              pulsar term's 2 phase_p = 2 phase - delta is a rotation of the Earth term's
//                    and, on request, the parameter table.  A source within PTAR_CWPOP_POLE_TOL of a pulsar's line of sight
//                    has pattern (0, 0) there (and pd = 0), as antenna_patterns() in engine.py.
// cwpop_add_kernel   rows[r][i] += sum_s cw(r, s, t_i) over the packed TOA axis: a CTA covers CWP_TOAS slots x CWP_RB
//                    realizations; a thread keeps its slot's t and pulsar in registers and walks the realizations with the
//                    (r, s) records staged in shared memory, so each row access is one coalesced read-modify-write.  The
//                    formula is cgw_kernel's (deterministic.py:98-163); a NaN contribution (an evolving binary that has
//                    already merged) is dropped, as cw_catalog_kernel does.  Alignment slots (psr < 0) are never touched.
#pragma once
#include <stdint.h>

#include "ptar_rng.cuh"

namespace ptar {

constexpr int CWP_SRC = 16;       // doubles per (r, s) record
constexpr int CWP_PSR = 8;        // doubles per (r, s, p) record
constexpr int CWP_TAB = 16;       // doubles per (r, s) row of the parameter table
constexpr int CWP_TOAS = 256;     // TOA slots per CTA of the add kernel (one per thread)
constexpr int CWP_RB = 16;        // realizations per CTA of the add kernel
constexpr int CWP_STAGE = 1024;   // doubles of (r, s) records staged in shared memory at once (8 KB)
constexpr uint32_t K_CWPOP = 7;

// The two uniforms of element `elem` of the population stream `kind` (PTAR_K_CWPOP, or a transient population's) for
// pulsar `psr` (0 except for the pulsar-term phases) and global realization `r`.
__device__ __forceinline__ void cwpop_uniforms(double u[2], uint32_t elem, uint32_t psr, uint64_t r, const PhiloxKeys& K,
                                               uint32_t kind = K_CWPOP) {
  const uint4 w = philox4x32_10(make_uint4(elem, kind | (psr << 8), static_cast<uint32_t>(r), static_cast<uint32_t>(r >> 32)), K);
  u[0] = uniform53(w.x, w.y);
  u[1] = uniform53(w.z, w.w);
}

// Parameter j of a source from its uniform: fixed (lo), uniform (lo + width u) or isotropic (acos(lo + width u)).  The
// affine map is rounded operation by operation so the host restatement reproduces it bit for bit.
__device__ __forceinline__ double cwpop_param(int kind, double lo, double width, double u) {
  if (kind == PTAR_CWPOP_FIXED) return lo;
  const double x = __dadd_rn(lo, __dmul_rn(width, u));
  return kind == PTAR_CWPOP_ACOS ? acos(x) : x;
}

__global__ void cwpop_draw_kernel(double* __restrict__ src, double* __restrict__ psr, double* __restrict__ table,
                                  double* __restrict__ table_pph, ptar_cwpop_model m, int32_t nreal, int64_t real0,
                                  uint64_t seed) {
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= int64_t(nreal) * m.n_src) return;
  const int s = static_cast<int>(idx % m.n_src);
  const int64_t r = idx / m.n_src;
  const uint64_t rg = static_cast<uint64_t>(real0 + r);
  const PhiloxKeys K = philox_keys(seed);
  double v[PTAR_CWPOP_NPAR];
#pragma unroll
  for (int j = 0; j < PTAR_CWPOP_NPAR; j += 2) {
    double u[2];
    cwpop_uniforms(u, static_cast<uint32_t>(s * 16 + j / 2), 0, rg, K);
    v[j] = cwpop_param(m.kind[j], m.lo[j], m.width[j], u[0]);
    v[j + 1] = cwpop_param(m.kind[j + 1], m.lo[j + 1], m.width[j + 1], u[1]);
  }
  const double log10_h0 = v[PTAR_CWPOP_LOG10_H0], log10_fgw = v[PTAR_CWPOP_LOG10_FGW], log10_mc = v[PTAR_CWPOP_LOG10_MC];
  const double gwtheta = v[PTAR_CWPOP_GWTHETA], gwphi = v[PTAR_CWPOP_GWPHI], phase0 = v[PTAR_CWPOP_PHASE0];
  const double psi = v[PTAR_CWPOP_PSI], inc = v[PTAR_CWPOP_INC];
  const double h0 = exp10(log10_h0), fgw = exp10(log10_fgw), mc = exp10(log10_mc);
  // the scalars of cgw_inputs (engine.py) for dist_Mpc = 2 Mc^(5/3) (pi fgw)^(2/3) / h0
  const double mc_s = mc * 4.925838061995516e-06;                       // SOLAR2S
  const double w0 = 3.141592653589793 * fgw;
  const double mc53 = pow(mc_s, 5.0 / 3);
  const double dist_s = 2 * mc53 * pow(w0, 2.0 / 3) / h0;
  const double fac1 = 256.0 / 5 * mc53 * pow(w0, 8.0 / 3), fac2 = 1.0 / 32 / mc53, fac3 = mc53 / dist_s;
  const double ph0 = phase0 / 2, w053 = pow(w0, -5.0 / 3);
  const double alpha = fac3 / cbrt(w0);
  double* o = src + idx * CWP_SRC;
  o[0] = w0;
  o[1] = fac1;
  o[2] = fac2;
  o[3] = fac3;
  o[4] = ph0;
  o[5] = w053;
  o[6] = 0.5 * (3 + cos(2 * inc));
  o[7] = 2 * cos(inc);
  o[8] = cos(2 * psi);
  o[9] = sin(2 * psi);
  o[10] = alpha;
#pragma unroll
  for (int k = 11; k < CWP_SRC; ++k) o[k] = 0.0;
  if (table) {
    double* q = table + idx * CWP_TAB;
    q[0] = gwtheta; q[1] = gwphi; q[2] = phase0; q[3] = psi; q[4] = inc;
    q[5] = log10_h0; q[6] = log10_fgw; q[7] = log10_mc; q[8] = dist_s / 102927125054338.98;   // MPC2S
    q[9] = fgw; q[10] = mc; q[11] = h0;
#pragma unroll
    for (int k = 12; k < CWP_TAB; ++k) q[k] = 0.0;
  }
  double cgt, sgt, cgp, sgp;
  sincos(gwtheta, &sgt, &cgt);
  sincos(gwphi, &sgp, &cgp);
  const double mx = sgp, my = -cgp;
  const double nx = -cgt * cgp, ny = -cgt * sgp, nz = sgt;
  const double ox = -sgt * cgp, oy = -sgt * sgp, oz = -cgt;
  double* pr = psr + idx * int64_t(m.n_psr) * CWP_PSR;
  for (int p = 0; p < m.n_psr; ++p) {
    const double px = m.phat[3 * p], py = m.phat[3 * p + 1], pz = m.phat[3 * p + 2];
    const double mdp = mx * px + my * py, ndp = nx * px + ny * py + nz * pz, odp = ox * px + oy * py + oz * pz;
    const double cosMu = -odp;
    // 1 + Omega.p as (m.p^2 + n.p^2) / (1 - Omega.p): keeps its relative accuracy next to the pulsar's line of sight
    const double den = (mdp * mdp + ndp * ndp) / (1 - odp);
    const bool ok = den > PTAR_CWPOP_POLE_TOL;   // false also for NaN (a source antipodal to the pulsar)
    double pd = m.pdist ? m.pdist[p] : 0.0;
    if (m.pphase) {   // uniform on [0, 2 pi): element s * 16 + 4, the pulsar in the kind word
      double u[2];
      cwpop_uniforms(u, static_cast<uint32_t>(s * 16 + PTAR_CWPOP_NPAR / 2), static_cast<uint32_t>(p), rg, K);
      const double pph = __dmul_rn(6.283185307179586, u[0]);
      if (table_pph) table_pph[idx * m.n_psr + p] = pph;
      pd = pph / (2 * 3.141592653589793 * fgw * (1 - cosMu)) / 102927125054.33899;
    }
    pd = ok ? pd * 102927125054.33899 : 0.0;                           // KPC2S; 0 where the pattern is 0
    double* q = pr + int64_t(p) * CWP_PSR;
    q[0] = ok ? 0.5 * (mdp * mdp - ndp * ndp) / den : 0.0;
    q[1] = ok ? (mdp * ndp) / den : 0.0;
    q[2] = cosMu;
    q[3] = pd;
    double m0 = 0.0, m1 = 0.0, m2 = 0.0;
    if (m.mode == 1) {
      const double omega_p = w0 * pow(1 + fac1 * pd * (1 - cosMu), -3.0 / 8);
      m0 = omega_p;
      m1 = ph0 + fac2 * (w053 - pow(omega_p, -5.0 / 3));
      m2 = fac3 / cbrt(omega_p);
    } else if (m.mode == 2) {
      sincos(2 * w0 * (pd * (1 - cosMu)), &m1, &m0);
    }
    q[4] = m0;
    q[5] = m1;
    q[6] = m2;
    q[7] = 0.0;
  }
}

template <int MODE>
__device__ __forceinline__ double cwpop_term(const double* __restrict__ q, const double* __restrict__ pp, double toa,
                                             int psr_term) {
  const double w0 = q[0], fac1 = q[1], fac2 = q[2], phase0 = q[4], w053 = q[5];
  const double inc1 = q[6], inc2 = q[7], c2p = q[8], s2p = q[9];
  const double fplus = pp[0], fcross = pp[1];
  double s2, c2, s2q, c2q, alpha, alpha_p;
  if (MODE == 0) {
    const double fac3 = q[3], cosMu = pp[2], pd = pp[3];
    const double tp = toa - pd * (1 - cosMu);
    const double omega = w0 * pow(1 - fac1 * toa, -3.0 / 8);
    const double omega_p = w0 * pow(1 - fac1 * tp, -3.0 / 8);
    sincos(2 * (phase0 + fac2 * (w053 - pow(omega, -5.0 / 3))), &s2, &c2);
    sincos(2 * (phase0 + fac2 * (w053 - pow(omega_p, -5.0 / 3))), &s2q, &c2q);
    alpha = fac3 / cbrt(omega);
    alpha_p = fac3 / cbrt(omega_p);
  } else if (MODE == 1) {
    sincos(2 * (phase0 + w0 * toa), &s2, &c2);
    sincos(2 * (pp[5] + pp[4] * toa), &s2q, &c2q);
    alpha = q[10];
    alpha_p = pp[6];
  } else {
    sincos(2 * (phase0 + w0 * toa), &s2, &c2);
    const double cd = pp[4], sd = pp[5];   // 2 phase_p = 2 phase - delta
    s2q = s2 * cd - c2 * sd;
    c2q = c2 * cd + s2 * sd;
    alpha = alpha_p = q[10];
  }
  const double At = s2 * inc1, Bt = c2 * inc2, Atp = s2q * inc1, Btp = c2q * inc2;
  const double rplus = alpha * (At * c2p + Bt * s2p), rcross = alpha * (-At * s2p + Bt * c2p);
  if (!psr_term) return -fplus * rplus - fcross * rcross;
  const double rplus_p = alpha_p * (Atp * c2p + Btp * s2p), rcross_p = alpha_p * (-Atp * s2p + Btp * c2p);
  return fplus * (rplus_p - rplus) + fcross * (rcross_p - rcross);
}

template <int MODE>
__global__ void __launch_bounds__(CWP_TOAS) cwpop_add_kernel(double* __restrict__ rows, int64_t ld, int32_t nreal,
                                                             const double* __restrict__ src, const double* __restrict__ psr,
                                                             const double* __restrict__ slot_t,
                                                             const int32_t* __restrict__ slot_psr, int n_psr, int n_src,
                                                             int psr_term) {
  __shared__ double sq[CWP_STAGE];
  const int64_t i = int64_t(blockIdx.x) * CWP_TOAS + threadIdx.x;
  const int p = i < ld ? slot_psr[i] : -1;
  const double toa = p >= 0 ? slot_t[i] : 0.0;
  const int r_begin = blockIdx.y * CWP_RB;
  const int r_end = min(nreal, r_begin + CWP_RB);
  const int per_stage = max(1, CWP_STAGE / (n_src * CWP_SRC));   // realizations whose records fit the stage
  for (int r0 = r_begin; r0 < r_end; r0 += per_stage) {
    const int cnt = min(per_stage, r_end - r0);
    const int nd = cnt * n_src * CWP_SRC;
    __syncthreads();
    for (int k = threadIdx.x; k < nd; k += CWP_TOAS) sq[k] = src[int64_t(r0) * n_src * CWP_SRC + k];
    __syncthreads();
    if (p < 0) continue;
    for (int j = 0; j < cnt; ++j) {
      const int64_t r = r0 + j;
      double acc = 0.0;
      for (int s = 0; s < n_src; ++s) {
        const double* pp = psr + ((r * n_src + s) * n_psr + p) * CWP_PSR;
        const double v = cwpop_term<MODE>(sq + (j * n_src + s) * CWP_SRC, pp, toa, psr_term);
        acc += isnan(v) ? 0.0 : v;
      }
      double* row = rows + r * ld + i;
      *row += acc;
    }
  }
}

}  // namespace ptar

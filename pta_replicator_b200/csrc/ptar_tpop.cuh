// Per-realization transient populations (ptar_transient_population): every realization gets its own n_src bursts with
// memory (family PTAR_TPOP_BWM) or sine-Gaussian bursts (PTAR_TPOP_BURST), drawn on the device from the priors of a
// ptar_tpop_model and added to its row of residuals.
//
// tpop_draw_kernel  one thread per (realization, source).  Draws the PTAR_TPOP_NPAR parameters from the Philox stream
//                   PTAR_K_BWMPOP or PTAR_K_BURSTPOP (counter layout in ptar_rng.cuh) through cwpop_param, and writes
//                     rec[r][s][4]     = {t0 [s], 2 pi f0, 1 / tau, phase0}            (BWM: {t0, 0, 0, 0})
//                     coef[r][s][p][2] = {alpha_p, beta_p} of g (alpha cos Phi + beta sin Phi)  (BWM: {pol_p h, 0})
//                   and, on request, the parameter table.  A source within PTAR_CWPOP_POLE_TOL of a pulsar's line of
//                   sight, or antipodal to it, has pattern (0, 0) there, as antenna_patterns() in engine.py.
// tpop_add_kernel   rows[r][i] += sum_s term(r, s, t_i) over the packed TOA axis, in cwpop_add_kernel's shape: a CTA
//                   covers TP_TOAS slots x TP_RB realizations, a thread keeps its slot's t and pulsar in registers and
//                   walks the realizations with their (r, s) records staged in shared memory, so each row access is one
//                   coalesced read-modify-write.  A slot whose terms are all exactly 0 (before every t0 of the
//                   realization for BWM, g underflowed for every burst) is neither read nor written; alignment slots
//                   (psr < 0) are never touched.
#pragma once
#include <stdint.h>

#include "ptar_cwpop.cuh"
#include "ptar_rng.cuh"

namespace ptar {

constexpr int TP_REC = 4;         // doubles per (r, s) record
constexpr int TP_COEF = 2;        // doubles per (r, s, p) coefficient
constexpr int TP_TOAS = 256;      // TOA slots per CTA of the add kernel (one per thread)
constexpr int TP_RB = 16;         // realizations per CTA of the add kernel
constexpr int TP_STAGE = 1024;    // doubles of (r, s) records staged in shared memory at once (8 KB)
constexpr double TP_G_ZERO = 750.0;   // (t - t0)^2 / tau^2 past this: exp(-x) < 1e-325 rounds to 0, the term is 0
constexpr uint32_t K_BWMPOP = 9, K_BURSTPOP = 10;

__global__ void tpop_draw_kernel(double* __restrict__ rec, double* __restrict__ coef, double* __restrict__ table,
                                 ptar_tpop_model m, int32_t nreal, int64_t real0, uint64_t seed) {
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= int64_t(nreal) * m.n_src) return;
  const int s = static_cast<int>(idx % m.n_src);
  const uint64_t rg = static_cast<uint64_t>(real0 + idx / m.n_src);
  const PhiloxKeys K = philox_keys(seed);
  const bool burst = m.family == PTAR_TPOP_BURST;
  double v[PTAR_TPOP_NPAR];
#pragma unroll
  for (int j = 0; j < PTAR_TPOP_NPAR; j += 2) {
    double u[2];
    cwpop_uniforms(u, static_cast<uint32_t>(s * 16 + j / 2), 0, rg, K, burst ? K_BURSTPOP : K_BWMPOP);
    v[j] = cwpop_param(m.kind[j], m.lo[j], m.width[j], u[0]);
    v[j + 1] = cwpop_param(m.kind[j + 1], m.lo[j + 1], m.width[j + 1], u[1]);
  }
  const double t0_mjd = v[PTAR_TPOP_T0], gwtheta = v[PTAR_TPOP_GWTHETA], gwphi = v[PTAR_TPOP_GWPHI];
  const double pol = v[PTAR_TPOP_POL], phase0 = v[PTAR_TPOP_PHASE0], eps = v[PTAR_TPOP_EPS], Q = v[PTAR_TPOP_Q];
  const double amp = exp10(v[PTAR_TPOP_LOG10_AMP]);
  const double f0 = burst ? exp10(v[PTAR_TPOP_LOG10_F0]) : 0.0;
  const double w = 6.283185307179586 * f0;
  double s2, c2;
  sincos(2 * pol, &s2, &c2);
  double* o = rec + idx * TP_REC;
  o[0] = __dmul_rn(t0_mjd, 86400.0);
  o[1] = w;
  o[2] = burst ? w / Q : 0.0;
  o[3] = burst ? phase0 : 0.0;
  if (table) {
    double* q = table + idx * PTAR_TPOP_TABLE;
#pragma unroll
    for (int k = 0; k < PTAR_TPOP_TABLE; ++k) q[k] = 0.0;
    q[0] = t0_mjd;
    q[1] = v[PTAR_TPOP_LOG10_AMP];
    q[2] = amp;
    if (burst) {
      double sp, cp;
      sincos(phase0, &sp, &cp);
      q[3] = v[PTAR_TPOP_LOG10_F0]; q[4] = f0; q[5] = Q; q[6] = Q / w;
      q[7] = gwtheta; q[8] = gwphi; q[9] = pol; q[10] = phase0; q[11] = eps;
      q[12] = amp * (c2 * cp - eps * s2 * sp);
      q[13] = amp * (-c2 * sp - eps * s2 * cp);
      q[14] = amp * (s2 * cp + eps * c2 * sp);
      q[15] = amp * (-s2 * sp + eps * c2 * cp);
    } else {
      q[3] = gwtheta; q[4] = gwphi; q[5] = pol;
    }
  }
  double cgt, sgt, cgp, sgp;
  sincos(gwtheta, &sgt, &cgt);
  sincos(gwphi, &sgp, &cgp);
  const double mx = sgp, my = -cgp;
  const double nx = -cgt * cgp, ny = -cgt * sgp, nz = sgt;
  const double ox = -sgt * cgp, oy = -sgt * sgp, oz = -cgt;
  double* pr = coef + idx * int64_t(m.n_psr) * TP_COEF;
  for (int p = 0; p < m.n_psr; ++p) {
    const double px = m.phat[3 * p], py = m.phat[3 * p + 1], pz = m.phat[3 * p + 2];
    const double mdp = mx * px + my * py, ndp = nx * px + ny * py + nz * pz, odp = ox * px + oy * py + oz * pz;
    // 1 + Omega.p as (m.p^2 + n.p^2) / (1 - Omega.p), as cwpop_draw_kernel
    const double den = (mdp * mdp + ndp * ndp) / (1 - odp);
    const bool ok = den > PTAR_CWPOP_POLE_TOL;   // false also for NaN (a source antipodal to the pulsar)
    const double fp = ok ? 0.5 * (mdp * mdp - ndp * ndp) / den : 0.0;
    const double fx = ok ? (mdp * ndp) / den : 0.0;
    double* q = pr + int64_t(p) * TP_COEF;
    if (burst) {
      q[0] = -amp * (fp * c2 + fx * s2);
      q[1] = eps * amp * (fp * s2 - fx * c2);
    } else {
      q[0] = (c2 * fp + s2 * fx) * amp;
      q[1] = 0.0;
    }
  }
}

template <int FAMILY>
__global__ void __launch_bounds__(TP_TOAS) tpop_add_kernel(double* __restrict__ rows, int64_t ld, int32_t nreal,
                                                           const double* __restrict__ rec, const double* __restrict__ coef,
                                                           const double* __restrict__ slot_t,
                                                           const int32_t* __restrict__ slot_psr, int n_psr, int n_src) {
  __shared__ double sq[TP_STAGE];
  const int64_t i = int64_t(blockIdx.x) * TP_TOAS + threadIdx.x;
  const int p = i < ld ? slot_psr[i] : -1;
  const double toa = p >= 0 ? slot_t[i] : 0.0;
  const int r_begin = blockIdx.y * TP_RB;
  const int r_end = min(nreal, r_begin + TP_RB);
  const int per_stage = TP_STAGE / (n_src * TP_REC);   // n_src <= 64: at least 4 realizations per stage
  for (int r0 = r_begin; r0 < r_end; r0 += per_stage) {
    const int cnt = min(per_stage, r_end - r0);
    const int nd = cnt * n_src * TP_REC;
    __syncthreads();
    for (int k = threadIdx.x; k < nd; k += TP_TOAS) sq[k] = rec[int64_t(r0) * n_src * TP_REC + k];
    __syncthreads();
    if (p < 0) continue;
    for (int j = 0; j < cnt; ++j) {
      const int64_t r = r0 + j;
      double acc = 0.0;
      bool hit = false;
      for (int s = 0; s < n_src; ++s) {
        const double* q = sq + (j * n_src + s) * TP_REC;
        const double* c = coef + ((r * n_src + s) * n_psr + p) * TP_COEF;
        if (FAMILY == PTAR_TPOP_BWM) {
          if (toa < q[0]) continue;   // the ramp is 0 before t0 (memory_kernel's test)
          acc += __dmul_rn(__ldg(c), __dsub_rn(toa, q[0]));
        } else {
          const double dt = toa - q[0];
          const double x = dt * q[2];
          const double e = x * x;
          if (!(e < TP_G_ZERO)) continue;
          const double2 ab = __ldg(reinterpret_cast<const double2*>(c));
          double sn, cs;
          sincos(fma(q[1], dt, q[3]), &sn, &cs);
          acc += exp(-e) * (ab.x * cs + ab.y * sn);
        }
        hit = true;
      }
      if (hit) {
        double* row = rows + r * ld + i;
        *row += acc;
      }
    }
  }
}

}  // namespace ptar

/* ptar.h -- C ABI of the H100 synthetic-PTA residual generator (libptar_b200.so).
 *
 * The reference (bencebecsy/pta_replicator) has no FFI: its boundary is a set of
 * Python functions.  Each entry point below replaces the arithmetic body of one of
 * them and is what a binding on the reference side would call (INTEGRATION.md shows
 * the ctypes stub).  Conventions: plain pointers and sizes, no torch types; every
 * pointer is a DEVICE pointer unless the name ends in _host; the library never
 * allocates or frees user memory; all work is enqueued on the given cudaStream_t
 * (passed as void*); return 0 on success, negative on bad arguments / launch errors
 * (text from ptar_last_error()).  All floating point is IEEE fp64 unless noted.
 *
 * Non-finite inputs.  The summary entry points take maps and statistics a caller may supply, so NaN and +-inf reach
 * them in normal use; they follow one rule.
 *   - Every (max, argmax) -- ptar_curn_reduce, ptar_fp_reduce, ptar_fe_sky, ptar_fe_combine, ptar_os_aniso,
 *     ptar_bwm_sky, ptar_bwm_combine -- ranks by
 *     larger value, then lower index, with NaN above every number: the first NaN wins wherever it sits, otherwise the
 *     first maximum.
 *   - ptar_curn_reduce: -inf among finite entries is a zero likelihood and everything stays finite.  A NaN or +inf
 *     anywhere in a map makes ln_bayes, post_amp, post_gamma and ul_amp NaN (ul_amp is NaN whenever the posterior is
 *     not finite, never the last grid node).  An all -inf map gives lnL_max = -inf at indices (0, 0), ln_bayes = -inf,
 *     and NaN posteriors and ul_amp.
 *   - A false-alarm probability of a NaN statistic is NaN: ptar_fp_reduce_fap for a NaN Fp (0 for Fp = +inf), and
 *     ptar_os_null for a NaN observed S/N (column 0).  A NaN null column counts as an exceedance, the conservative
 *     side, so exceed[r] = n_col - 1 when column 0 is NaN.
 * For finite inputs none of this changes an output bit.
 *
 * Reference lines replaced (paths relative to /root/reference/pta_replicator/):
 *   ptar_cholesky_lower    np.linalg.cholesky(ORF)                      red_noise.py:235
 *   ptar_fourier_basis     create_fourier_design_matrix_red             red_noise.py:36-103
 *   ptar_gwb_mix           w draws + np.dot(M, w)                       red_noise.py:238-240, :268
 *   ptar_gwb_synth         sqrt(C) scale, Hermitian pack, ifft, crop    red_noise.py:269-285
 *   ptar_gwb_slice_i8 /    the same linear map on the int8 tensor cores (wgmma; exact int8 digit
 *   ptar_gwb_synth_i8      slices, int32 accumulators; throughput mode)       red_noise.py:269-285
 *   ptar_cgw_delay         add_cgw arithmetic                           deterministic.py:98-163
 *   ptar_cw_catalog        loop_over_CWs[_parallel] (numba)             deterministic.py:321-561
 *   ptar_burst_delay       add_burst polarisation mix                   deterministic.py:771-780
 *   ptar_memory_delay      add_gw_memory ramp                           deterministic.py:864-873
 *   ptar_generate          efac/equad draw                              white_noise.py:105-109
 *                          U @ (ecorr*z)                                white_noise.py:182
 *                          F @ (sqrt(prior)*z)                          red_noise.py:126-128
 *                          interp1d(ut, Res)(toas)                      red_noise.py:286-287
 *                          (+ CGW / deterministic delays)               deterministic.py:160-165
 *   ptar_philox_normals    np.random.randn (throughput-mode stream)     SURVEY.md 3.6
 *   ptar_timing_project    the linear timing fit of SimulatedPulsar.fit simulate.py:44-69 (weighted least squares
 *                          on a fixed design matrix; np.polyfit of add_burst(remove_quad) deterministic.py:777-779)
 *   ptar_os_project /      no counterpart: the frequentist optimal statistic of the realizations, reduced on the
 *   ptar_os_pairs          device instead of gathering the rows
 *   ptar_os_null           no counterpart: phase-shift / sky-scramble null distribution and p-value per realization
 *   ptar_os_aniso          no counterpart: spherical-harmonic fit, anisotropy chi^2 and radiometer sky map per realization
 *   ptar_os_pf             no counterpart: per-frequency optimal statistic (GW power at every f_k) per realization
 *   ptar_fp_project /      no counterpart: the incoherent Fp-statistic of continuous waves per realization and search
 *   ptar_fp_reduce         frequency, reduced on the device
 *   ptar_curn_grid /       no counterpart (an MCMC over enterprise's CURN model per realization): the common-process
 *   ptar_curn_reduce       likelihood on an (A, gamma) grid, its maximum, Bayes factor, marginals and upper limit
 *   ptar_hd_grid           no counterpart (an MCMC over enterprise's HD-correlated model per realization): the
 *                          ORF-correlated common-process likelihood on the CURN grid, reduced by ptar_curn_reduce
 *   ptar_rn_grid           no counterpart (a single-pulsar noise analysis per realization and pulsar): each pulsar's
 *                          intrinsic red-noise likelihood on an (A, gamma) grid, reduced by ptar_curn_reduce
 *   ptar_fs_grid           no counterpart (an MCMC over enterprise's free_spectrum model per realization): the
 *                          factorised free-spectrum likelihood, one log10 rho grid per GW frequency bin, uncorrelated or
 *                          ORF-correlated, reduced by ptar_curn_reduce
 *   ptar_fs_y2 /           no counterpart (a refit of a spectral model to the free spectrum per realization, as
 *   ptar_fs_refit          ceffyl does from KDEs): power-law, turnover or user spectra on a grid, exact in the factorised
 *                          per-bin likelihoods, reduced by ptar_curn_reduce
 *   ptar_cw_population     add_cgw per realization with parameters drawn from priors on the device (a population study
 *                          calls add_cgw once per realization)                   deterministic.py:13-163
 *   ptar_common_population no counterpart (a calibration study draws a common process per realization on the host): a
 *                          power-law or free-spectrum common process, uncorrelated or ORF-correlated, drawn from priors
 *                          on the device in the statistics' Fourier basis and added to every realization
 *   ptar_transient_        add_gw_memory / add_burst (sine-Gaussian waveforms) per realization with parameters drawn
 *   population             from priors on the device (a population study calls them once per realization)
 *                                                                                deterministic.py:718-884
 *   ptar_bwm_sky /         no counterpart (a matched-filter search of add_gw_memory's ramp per realization): the
 *   ptar_bwm_combine       coherent burst-with-memory statistic over epoch x sky and the pulsar-term statistic, reduced
 *                          on the device
 *   ptar_burst_ninv /      no counterpart (a wavelet search for add_burst / add_noise_transient per realization): the
 *   ptar_burst_project /   coherent sine-Gaussian statistic over a t0 x f0 x Q bank x sky (with ptar_fe_sky) and the
 *   ptar_burst_reduce      per-pulsar transient statistic, reduced on the device
 */
#ifndef PTAR_H
#define PTAR_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PTAR_VERSION 200  /* major*100 + minor; 2.0: column-major grid, g_ldr / c_rows, int8 GWB entry points, pshift phases.
                             Later additions leave every 2.0 struct layout and entry point unchanged: the timing-model fit
                             (ptar_timing_model, ptar_timing_project[_stage], ptar_run_job[_to_host]_tm) and the optimal
                             statistic (ptar_os_model, ptar_os_project[_stage], ptar_os_pairs), its null distributions
                             (ptar_os_null_model, ptar_os_null[_stage]) and anisotropy (ptar_os_aniso_model,
                             ptar_os_aniso[_stage], PTAR_OS_ANISO_MAX_LM / _SKY) and per-frequency form
                             (ptar_os_pf_model, ptar_os_pf), the Fp-statistic (ptar_fp_model,
                             ptar_fp_project, ptar_fp_reduce[_fap], PTAR_FP_MAX_FREQ), the CURN likelihood
                             (ptar_curn_model, ptar_curn_grid, ptar_curn_reduce, PTAR_CURN_MAX_NA / _NG) and the HD
                             likelihood (ptar_hd_model, ptar_hd_grid, PTAR_HD_MAX_N / _JB) and the single-pulsar
                             red-noise likelihood (ptar_rn_model, ptar_rn_grid, PTAR_RN_MAX_NC) and the burst-with-memory
                             search (ptar_bwm_model, ptar_bwm_sky, ptar_bwm_combine, PTAR_BWM_MAX_EPOCH) and the
                             free-spectrum likelihood (ptar_fs_model, ptar_fs_grid, PTAR_FS_MAX_PSR / _BIN / _JB) and the sine-Gaussian
                             burst search (ptar_burst_model, ptar_burst_ninv, ptar_burst_project, ptar_burst_reduce,
                             PTAR_BURST_MAX_TEMPLATE / _GROUP / _TB) and the free spectrum's spectral refit
                             (ptar_fs_refit_model, ptar_fs_y2, ptar_fs_refit, PTAR_FS_MAX_TEMPLATE) and chromatic noise in
                             the generator (ptar_chrom_model, ptar_generate_chrom, ptar_generate_stage_chrom,
                             ptar_run_job_to_host_chrom, PTAR_K_CHROM, PTAR_CHROM_SLOTS) and per-realization
                             continuous-wave populations (ptar_cwpop_model, ptar_cw_population[_stage], PTAR_K_CWPOP,
                             PTAR_CWPOP_*) and per-realization common-process populations (ptar_cpop_model,
                             ptar_common_population[_stage], PTAR_K_CPOP, PTAR_CPOP_*) and per-realization
                             burst-with-memory and sine-Gaussian burst populations (ptar_tpop_model,
                             ptar_transient_population[_stage], PTAR_K_BWMPOP, PTAR_K_BURSTPOP, PTAR_TPOP_*)
                             are new symbols only, so
                             a caller detects them by looking the symbol up.  ptar_os_project accepts nc up to
                             PTAR_RN_MAX_NC since the red-noise likelihood; nothing changes for nc <= PTAR_OS_MAX_NC. */

/* Geometry limits of the fused generator kernel. */
#define PTAR_TILE_TOAS   1024  /* TOAs per tile (256 threads x 4)            */
#define PTAR_TILE_EPOCHS 64    /* kernel-epochs per tile                     */
#define PTAR_TOA_ALIGN   4     /* every pulsar segment starts at a multiple  */

/* ptar_gen_params.flags */
#define PTAR_F_WHITE    1u   /* efac*sigma*z1 + w2*z2                         */
#define PTAR_F_ECORR    2u   /* ecorr[epoch] * z[bucket(epoch)]               */
#define PTAR_F_RED      4u   /* Fourier-basis red noise                       */
#define PTAR_F_GWB      8u   /* linear interpolation of the GWB time grid     */
#define PTAR_F_DET      16u  /* precomputed deterministic delay (CGW ...)     */
#define PTAR_F_WHITE1   32u  /* throughput mode only: one N(0, w1^2+w2^2) draw per TOA
                                instead of two (identical distribution)       */

/* Philox stream tags ("kind") -- part of the counter, see ptar_philox_normals. */
#define PTAR_K_WHITE1 1
#define PTAR_K_WHITE2 2
#define PTAR_K_ECORR  3
#define PTAR_K_RED    4
#define PTAR_K_GWB    5
#define PTAR_K_CHROM  6   /* chromatic coefficients: index = (slot << 16) | Fourier column */
#define PTAR_K_CWPOP  7   /* continuous-wave populations: index = source * 16 + parameter pair, see ptar_cw_population */
#define PTAR_K_CPOP   8   /* common-process populations: index = bin or PTAR_CPOP_HYPER + pair, see ptar_common_population */
#define PTAR_K_BWMPOP   9   /* burst-with-memory populations: index = source * 16 + parameter pair, see ptar_transient_population */
#define PTAR_K_BURSTPOP 10  /* sine-Gaussian burst populations: index = source * 16 + parameter pair, as PTAR_K_BWMPOP */

/* One tile of the packed TOA axis: <=1024 consecutive (time-sorted) TOAs of ONE pulsar
 * touching <=64 kernel-epochs. */
typedef struct {
  int32_t toa_start;   /* index into the packed per-TOA arrays (multiple of 4)          */
  int32_t n_toa;       /* real TOAs in this tile (<= PTAR_TILE_TOAS)                    */
  int32_t toa_local0;  /* index of toa_start within its pulsar (Philox counter base)    */
  int32_t ep_start;    /* first kernel-epoch (global index)                             */
  int32_t n_ep;        /* kernel-epochs touched (<= PTAR_TILE_EPOCHS)                   */
  int32_t psr;         /* pulsar index                                                  */
  int32_t nd;          /* Taylor terms used for red noise inside epochs (1..3)          */
  int32_t reserved;    /* c_row0: sum of n_ep over the preceding tiles (rows of the Cbuf blocks)        */
} ptar_tile;

typedef struct {
  /* geometry */
  int32_t n_psr;
  int32_t n_tiles;
  int32_t J;            /* red-noise basis columns (2 * components); 0 if no red noise  */
  int32_t npts;         /* GWB grid length; 0 if no GWB                                  */
  uint32_t flags;       /* PTAR_F_*                                                      */
  int32_t rn_convention;/* 0: (sin,cos) pairs, absolute t;  1: libstempo (cos,sin)      */
  const ptar_tile* tiles;
  /* per-TOA statics, packed axis of length ld_out */
  const double*   w1;    /* efac*sigma [s]                                               */
  const double*   w2;    /* efac*equad (t2equad) or equad (tnequad) [s]                  */
  const double*   dtau;  /* t - t_ref(epoch) [s]                                         */
  const uint16_t* eloc;  /* kernel-epoch index local to the tile                         */
  const double*   det;   /* deterministic delay [s]                                      */
  /* per-epoch statics (an epoch never straddles an ECORR bucket edge or a GWB grid knot) */
  const double*  ep_ecorr;   /* ecorr of the epoch's bucket [s]                          */
  const int32_t* ep_bucket;  /* ECORR bucket id within the pulsar                        */
  const int32_t* ep_gidx;    /* column of knot j in the compact grid G (knot j+1 is the next column) */
  const double*  ep_gw;      /* (t_ref - ut[j]) / (ut[j+1] - ut[j])                      */
  const double*  ep_ginv;    /* 1 / (ut[j+1] - ut[j])  [1/s]                             */
  const int64_t* psr_bucket_off; /* [n_psr]: offset of each pulsar in the injected zb axis */
  const double*  Ftile;      /* [n_tiles][J][64]: basis at epoch reference times          */
  /* per-pulsar red-noise statics */
  const double* rn_scale;    /* [n_psr][J] sqrt(prior)                                   */
  const double* rn_omega;    /* [n_psr][J/2] 2*pi*f_k                                    */
  /* compact GWB grid for this batch of realizations, COLUMN-major: G[q][g_ldr], q < g_ld compact knot columns (only
   * the knots next to some TOA of a pulsar are present, ptar_gwb_synth), row = realization of this call; g_ldr is a
   * multiple of 4 >= nreal rounded up to 4.  The synthesis writes 32 consecutive realizations per store and the
   * generator reads 4 consecutive realizations of a knot as one 32-byte sector. */
  const double* G;
  int64_t g_ld;
  int64_t g_ldr;
  /* injected standard-normal draws (parity mode); all NULL => Philox */
  const double* z1;   /* [nreal][ld_out]                                                 */
  const double* z2;   /* [nreal][ld_out]                                                 */
  const double* zb;   /* [nreal][n_bucket_total]                                         */
  const double* zrn;  /* [nreal][n_psr][J]                                               */
  int64_t n_bucket_total;
  /* RNG (throughput mode) */
  uint64_t seed;
  int64_t  real0;     /* global id of realization 0 of this call (multiple of 4)         */
  /* output: out[r][ld_out] */
  double* out;
  int64_t ld_out;
  int32_t nreal;
  int32_t rc;         /* realizations per CTA: 16 (256 threads) or 32 (512 threads); 0 = default */
  /* optional scratch for the two-kernel schedule (epoch kernel -> TOA kernel): at least
   * c_rows * ceil(nreal/rc) * (3 rc + 2) doubles (rc = 16: 50 per row); NULL selects the fused kernel.
   * The library checks cbuf_len against that size before it launches. */
  double* Cbuf;
  int64_t cbuf_len;   /* doubles available at Cbuf */
  int64_t c_rows;     /* sum of n_ep over all tiles (rows of the epoch blocks)  */
} ptar_gen_params;

int         ptar_version(void);
const char* ptar_last_error(void);

/* Lower Cholesky factor of `batch` SPD matrices A[b][n][n] (row-major) -> L (strict upper
 * part zeroed).  info[b] = 0, or k>0 if the leading minor of order k is not PD.  n <= 1024. */
int ptar_cholesky_lower(double* L, const double* A, int n, int batch, int* info, void* stream);

/* F[row][2k], F[row][2k+1] = trig(2*pi * tprime[row] * freqs[psr(row)][k] (+ phase[psr(row)][k])) in the reference's
 * operation order; convention 0 -> (sin, cos), 1 -> (cos, sin); phase = NULL or the `pshift` random phases
 * (red_noise.py:83-84).  out index: out[row_off[row] + col*col_stride] so the caller chooses row-major or per-tile
 * layouts. */
int ptar_fourier_basis(double* out, const int64_t* row_off, int64_t col_stride,
                       const double* tprime, const int32_t* row_psr, const double* freqs, const double* phase,
                       int K, int convention, int64_t nrows, void* stream);

/* Continuous-wave delay per TOA.  src[16] and psr_par[n_psr][4] = {fplus, fcross, cosMu, pd_sec}
 * are the scalar pre-factors of deterministic.py:51-105; mode 0 evolve, 1 phase_approx, 2 mono.
 * out[i] (+)= delay(t[i]) ; t = mjd*86400 - tref. */
int ptar_cgw_delay(double* out, const double* t, const int32_t* psr_of_toa, const double* psr_par,
                   const double* src, int mode, int psr_term, int accumulate, int64_t n, void* stream);

/* Sum of many continuous-wave sources for ONE pulsar (add_catalog_of_cws, deterministic.py:188-561; SURVEY.md
 * 8f row f1).  cat[8][n_src] = gwtheta, gwphi, mc [Msun], dist [Mpc], fgw [Hz], phase0, psi, inc (device);
 * phat_host[3] = pulsar unit vector (HOST); pdist in kpc or pphase (use_pphase); mode / psr_term as in
 * ptar_cgw_delay; NaN contributions are dropped like the reference does.  Scratch: pre[n_src][16],
 * partial[n_slices][n_toa] (device).  out[i] (+)= sum_s delay_s(t[i]); t = mjd*86400 - tref. */
int ptar_cw_catalog(double* out, const double* t, int64_t n_toa, const double* phat_host, const double* cat,
                    int64_t n_src, double pdist_kpc, double pphase, int use_pphase, int mode, int psr_term,
                    int accumulate, double* pre, double* partial, int n_slices, void* stream);

/* Burst of arbitrary waveform (add_burst, deterministic.py:718-793; SURVEY.md 8f row f4).  hplus / hcross are the
 * caller's waveform callables sampled at t = mjd*86400 - tref (the callables are Python objects in the reference too);
 * fplus / fcross the antenna pattern (:757-759).  out[i] (+)= -fplus (h+ cos2psi - hx sin2psi) - fcross (h+ sin2psi +
 * hx cos2psi), every product rounded separately like numpy. */
int ptar_burst_delay(double* out, const double* hplus, const double* hcross, double fplus, double fcross, double cos2psi,
                     double sin2psi, int accumulate, int64_t n, void* stream);

/* Burst with memory (add_gw_memory, deterministic.py:822-884): out[i] (+)= t[i] < t0 ? 0 : amp (t[i] - t0), with
 * t = mjd*86400, t0 = t0_mjd*86400 and amp = (cos(2 pol) fplus + sin(2 pol) fcross) * strain. */
int ptar_memory_delay(double* out, const double* t, double amp, double t0, int accumulate, int64_t n, void* stream);

/* Zm[p][r][j] = sum_q M[p][q] z[r][q][j]  (output pulsar-major: [n_psr][nreal][J]).  z is read from
 * zin[r][q][j] (parity) or drawn from Philox (zin == NULL; stream PTAR_K_GWB).  M is n_psr x n_psr lower
 * triangular, row-major. */
int ptar_gwb_mix(double* Zm, const double* M, const double* zin, int n_psr, int J,
                 int64_t nreal, uint64_t seed, int64_t real0, void* stream);

/* Compact grid: G[r][q] = sum_j A[knots[q]][j] * Zm[p(q)][r][j] for every column q of the knot list
 * (knots[g_ld]: per pulsar the sorted rows of A that its TOAs interpolate, each pulsar block starting at an
 * even column and padded to even length with -1).  tile_list[n_tiles][4] = {pulsar, first column, columns
 * (<= 64), k extent} enumerates 64-column blocks, heaviest first; with lower_tri the k loop stops at the
 * tile's k extent (A[n][j] == 0 for j > n). */
int ptar_gwb_synth(double* G, int64_t g_ld, int64_t g_ldr, const double* A, int64_t lda, const double* Zm, int J, int64_t nreal,
                   const int32_t* tile_list, int n_tiles, const int32_t* knots, int lower_tri, void* stream);

/* int8 tensor-core path of the synthesis (throughput mode; csrc/ptar_gwb_i8.cuh).  Both operands are fixed-point numbers with
 * PTAR_I8_SLICES signed radix-256 digits: value = scale * sum_s digit_s 2^(-8(s+1)), |value / scale| <= 1/4.
 * ptar_gwb_slice_i8: Zm[p][r][J] (fp64) -> ZS, int8 digits in the tensor core's K-major core-matrix tile layout
 *   [slice][pulsar][rcap/128 r-blocks][Jpad/32 k-chunks][16][2][8][16]; zinv[p] = 2^48 / zscale[p]; rcap (multiple of 128)
 *   is the row capacity the buffer was laid out for (>= nreal), Jpad a multiple of 32 (>= J).
 * ptar_gwb_synth_i8: G[q][r] = sum_j A[knot(q)][j] Zm[p(q)][r][j] from the digit slices; AS holds the digits of the
 *   gathered rows of A tile by tile, in tile_list order: [tile][Jpad/32][slice][4][2][8][16]; colscale[q] = (scale of
 *   row knot(q) of A) * 2^-16; tile_list as in ptar_gwb_synth but with 32-column blocks ( A lower triangular: k stops at the
 *    tile's k extent).  Exact int8 x int8 -> int32 products on wgmma .s32.s8.s8; the slice pairs s + t <= 6 are kept
 *   (dropped weight <= 2^-56 of full scale), the result is rounded once per output in fp64.
 * ptar_gwb_mix_i8: ptar_gwb_mix (Philox draws) with the slicing fused into its epilogue: ZS directly, no fp64 Zm
 *   (n_psr <= 72; larger arrays use ptar_gwb_mix + ptar_gwb_slice_i8). */
#define PTAR_I8_SLICES 6
int ptar_gwb_mix_i8(int8_t* ZS, const double* M, const double* zinv, int n_psr, int J, int Jpad, int64_t nreal, int64_t rcap,
                    uint64_t seed, int64_t real0, void* stream);
int ptar_gwb_slice_i8(int8_t* ZS, const double* Zm, const double* zinv, int n_psr, int J, int Jpad, int64_t nreal,
                      int64_t rcap, void* stream);
int ptar_gwb_synth_i8(double* G, int64_t g_ld, int64_t g_ldr, const int8_t* AS, const double* colscale, const int8_t* ZS,
                      const double* zscale, int n_psr, int J, int Jpad, int64_t nreal, int64_t rcap,
                      const int32_t* tile_list, int n_tiles, void* stream);

/* Diagnostics: buf (device, n_tiles * 8 int64, or NULL to switch off) receives clock64() stamps of the phases of
 * ptar_gwb_synth_i8 for the CTAs of r-block 0 (start, setup, loads issued, first stage landed, MMAs issued,
 * accumulators complete, epilogue done, k-chunks). */
int ptar_debug_i8_timestamps(void* buf);

/* The fused generator: out[r][i] = white + ecorr + red + gwb + det for nreal realizations. */
int ptar_generate(const ptar_gen_params* p, void* stream);

/* The two launches of the two-kernel schedule one at a time (p->Cbuf != NULL): stage 1 = epoch kernel
 * (Fourier GEMM, ECORR, GWB grid -> Cbuf), stage 2 = TOA kernel (Cbuf + white noise -> out).  ptar_generate
 * issues both; this entry exists so a caller can time them separately. */
int ptar_generate_stage(const ptar_gen_params* p, int stage, void* stream);

/* Chromatic Gaussian processes (DM variations, scattering) on top of ptar_generate: up to PTAR_CHROM_SLOTS slots, each
 *     out[r][i] += w_s[i] * sum_j F_s(t_i)_j scale_s[psr][j] z_j
 * with the per-TOA weight w_s[i] = (fref / nu_i)^idx_s and F_s the (sin, cos)(2 pi f t) basis on absolute time.  Like the
 * red noise, each slot is evaluated per (kernel-epoch, realization) as a quadratic in dt (its own Fourier GEMM in the
 * epoch stage) and the TOA stage adds w_s[i] times its Horner value; the tile's nd holds for every process.
 * A pulsar without a slot has on_s[psr] = 0 (its weights, scales and draws are never read).  Throughput-mode
 * coefficients are drawn on their own Philox stream (PTAR_K_CHROM, index (s << 16) | column), so every other draw is
 * the one ptar_generate makes.  The parity mode (p->z* set) needs zchr [nreal][n_psr][J_0 + ... + J_{n_slot-1}].
 * cm == NULL runs exactly ptar_generate / ptar_generate_stage.  With p->Cbuf the scratch must hold
 * c_rows * ceil(nreal/rc) * (3 rc (1 + n_slot) + 2) doubles. */
#define PTAR_CHROM_SLOTS 2
typedef struct {
  int32_t n_slot;                          /* 1 .. PTAR_CHROM_SLOTS                                     */
  int32_t J[PTAR_CHROM_SLOTS];             /* basis columns of each slot (2 * components, even)         */
  int32_t reserved;
  const double*  Ftile[PTAR_CHROM_SLOTS];  /* [n_tiles][J_s][64]: basis at the epoch reference times    */
  const double*  scale[PTAR_CHROM_SLOTS];  /* [n_psr][J_s] sqrt(prior)                                  */
  const double*  omega[PTAR_CHROM_SLOTS];  /* [n_psr][J_s/2] 2*pi*f_k                                   */
  const double*  weight[PTAR_CHROM_SLOTS]; /* [ld_out] per-TOA weight (fref / nu)^idx                   */
  const int32_t* on[PTAR_CHROM_SLOTS];     /* [n_psr] 1 = the pulsar carries this slot                  */
  const double*  zchr;                     /* parity mode: [nreal][n_psr][sum_s J_s] standard normals   */
} ptar_chrom_model;

int ptar_generate_chrom(const ptar_gen_params* p, const ptar_chrom_model* cm, void* stream);
int ptar_generate_stage_chrom(const ptar_gen_params* p, const ptar_chrom_model* cm, int stage, void* stream);

/* Raw throughput-mode normals (fp32 Box-Muller of Philox4x32-10), for tests:
 * out[k] = normal(kind, psr, realization, idx0 + k), k < n.  Counter = (idx, kind | psr << 8,
 * realization >> 2); the four outputs of a counter are realizations 4g .. 4g+3, so a shard of
 * realizations is reproduced bit-for-bit wherever it is generated.  idx = TOA index within the
 * pulsar (white), ECORR bucket, Fourier column (red), grid column (GWB). */
int ptar_philox_normals(float* out, int kind, int psr, int64_t realization, int64_t idx0,
                        int64_t n, uint64_t seed, void* stream);

/* Linear timing-model fit per pulsar (post-fit residuals).  For pulsar p with design matrix M_p (n_p x k_p) and
 * per-TOA weights w = 1/sigma^2, the host factors the whitened matrix once, W^{1/2} M_p = Q_p R_p (thin QR, Q_p
 * orthonormal columns), and the device applies
 *     r' = r - W^{-1/2} Q_p (Q_p^T W^{1/2} r)
 * to every realization row: the weighted least-squares residual r - M (M^T W M)^{-1} M^T W r without any k x k solve.
 * Two kernels: the reduce kernel writes per (tile, realization) the k sums Q^T W^{1/2} r over the tile's TOAs
 * (scratch partial[n_tiles][nreal][kmax]); the apply kernel adds a pulsar's tile partials in tile order and
 * subtracts W^{-1/2} Q c.  Every sum runs in an order fixed by the tile and the TOA index only, so a post-fit row is
 * bit-identical whatever nreal, chunking, real0 or launch grid produced it.  Only the n_p real TOAs of pulsars
 * that have tiles are written; alignment slots and pulsars without a model are never touched. */
#define PTAR_TM_KMAX 32   /* columns per pulsar */
typedef struct {
  int32_t n_psr;
  int32_t n_tiles;          /* tiles of the pulsars that have a model                                      */
  const ptar_tile* tiles;   /* [n_tiles]: toa_start, n_toa (<= PTAR_TILE_TOAS), toa_local0, psr are used; pulsar-
                               major, tiles of one pulsar consecutive and in time order                      */
  const int64_t* seg_off;   /* [n_psr] packed index of the pulsar's first TOA                               */
  const int32_t* seg_len;   /* [n_psr] n_p, real TOAs of the pulsar                                         */
  const int32_t* k;         /* [n_psr] k_p model columns (0: no model)                                      */
  const int64_t* q_off;     /* [n_psr] offset of the pulsar's Q block: Q[q_off[p] + j * n_p + i], i local   */
  const int32_t* tile0;     /* [n_psr] first tile of the pulsar in tiles[]                                  */
  const int32_t* n_tile;    /* [n_psr] tiles of the pulsar                                                  */
  const double* Q;          /* orthonormal columns of W^{1/2} M, engine (time-sorted) order                 */
  const double* sqrtw;      /* [ld_out] 1/sigma per TOA on the packed axis                                  */
  int32_t kmax;             /* max k_p (<= PTAR_TM_KMAX): row pitch of the partial sums                     */
  int32_t reserved;
} ptar_timing_model;

/* out[r][ld_out], r < nreal, in place.  scratch: at least n_tiles * nreal * kmax doubles (device).
 * ptar_timing_project_stage runs one of the two launches (stage 1 = reduce, 2 = apply) so a caller can time them. */
int ptar_timing_project(double* out, int64_t ld_out, int32_t nreal, const ptar_timing_model* tm, double* scratch,
                        int64_t scratch_len, void* stream);
int ptar_timing_project_stage(double* out, int64_t ld_out, int32_t nreal, const ptar_timing_model* tm, double* scratch,
                              int64_t scratch_len, int stage, void* stream);

/* Optimal statistic (csrc/ptar_os.cuh).  The host derives, once per recipe, C_a = P_a^{-1} F_gw,a for every pulsar
 * (P_a the noise covariance with the timing model marginalised, F_gw,a the 2K sin/cos columns of the GW basis), the
 * pair normalisations t_ab = tr(Z_a phi~ Z_b phi~) with Z_a = F_gw,a^T C_a, the template weights Gamma^o_ab and the
 * inverse F^{-1} of the multiple-component Fisher matrix.  Per realization r:
 *   ptar_os_project  X[r][p][j] = sum_i C[i][j] rows[r][i] over the TOAs i of pulsar p.  Two launches: a tile GEMM on
 *                    the fp64 tensor cores (partial[n_tiles][nreal][ncp]) and the sum of each pulsar's tile partials
 *                    in tile order.  rows: ld % 4 == 0, 32-byte aligned; alignment slots of the packed axis are ignored.
 *   ptar_os_pairs    x_p = X[r][p] phi~^{1/2};  d_ab = x_a . x_b (a < b, the order of `pairs`);
 *                    rho[r][q] = d_ab / t_ab (rho may be NULL);  b_o = sum_q orf[o][q] d_q;
 *                    a2[r][o] = b_o / dnorm[o];  snr[r][o] = b_o / dsqrt[o];  a2_mc[r][o] = sum_o' finv[o][o'] b_o'.
 * Every sum runs in an order fixed by the tile, the TOA index and the pair list only: outputs are bit-identical
 * whatever nreal, chunking, real0 or launch grid produced the rows.  ptar_os_project_stage runs one of the two
 * launches of ptar_os_project (stage 1 = tile GEMM, 2 = tile sums) so a caller can time them.  ptar_os_project alone
 * takes nc up to PTAR_RN_MAX_NC (the red-noise likelihood's bases); every other entry point of a ptar_os_model needs
 * nc <= PTAR_OS_MAX_NC. */
#define PTAR_OS_MAX_NC  32    /* GW-basis columns (2K)                 */
#define PTAR_RN_MAX_NC  64    /* basis columns of ptar_os_project and ptar_rn_grid (2 x 32 red-noise components) */
#define PTAR_OS_MAX_ORF 4     /* templates                             */
#define PTAR_OS_MAX_PSR 256   /* pulsars (pair kernel: x in shared memory) */
typedef struct {
  int32_t n_psr;
  int32_t n_tiles;
  const ptar_tile* tiles;   /* [n_tiles]: toa_start, n_toa (<= PTAR_TILE_TOAS), psr are used; tiles of one pulsar
                               consecutive and in time order                                                    */
  const int32_t* tile0;     /* [n_psr] first tile of the pulsar                                                 */
  const int32_t* n_tile;    /* [n_psr] tiles of the pulsar                                                      */
  const double* C;          /* [ld][ncp] row i = C_a[i][0..nc) of the TOA's pulsar, zero in columns >= nc and in
                               alignment slots                                                                  */
  int32_t nc;               /* 2K <= PTAR_OS_MAX_NC                                                             */
  int32_t ncp;              /* nc rounded up to a multiple of 8                                                 */
  const double* sqrt_phi;   /* [ncp] phi~^{1/2} per column                                                      */
  int32_t n_pairs;
  int32_t n_orf;            /* <= PTAR_OS_MAX_ORF                                                               */
  const int32_t* pairs;     /* [n_pairs][2] (a, b), a < b                                                       */
  const double* t_ab;       /* [n_pairs]                                                                        */
  const double* orf;        /* [n_orf][n_pairs] Gamma^o_ab                                                      */
  const double* dnorm;      /* [n_orf] D_o = sum_q Gamma^o_q^2 t_q                                              */
  const double* dsqrt;      /* [n_orf] sqrt(D_o)                                                                */
  const double* finv;       /* [n_orf][n_orf] F^{-1}, F_oo' = sum_q Gamma^o_q Gamma^o'_q t_q                    */
} ptar_os_model;

/* partial: >= n_tiles * nreal * ncp doubles; X: [nreal][n_psr][ncp]. */
int ptar_os_project(const double* rows, int64_t ld, int32_t nreal, const ptar_os_model* os, double* partial,
                    int64_t partial_len, double* X, void* stream);
int ptar_os_project_stage(const double* rows, int64_t ld, int32_t nreal, const ptar_os_model* os, double* partial,
                          int64_t partial_len, double* X, int stage, void* stream);
/* rho: [nreal][n_pairs] or NULL; a2, snr, a2_mc: [nreal][n_orf]. */
int ptar_os_pairs(const double* X, int32_t nreal, const ptar_os_model* os, double* rho, double* a2, double* snr,
                  double* a2_mc, void* stream);

/* Null distribution of one template's S/N (csrc/ptar_os_null.cuh): phase shifts or sky scrambles, drawn once on the
 * host and shared by every realization.  Columns s = 0..n_col-1: column 0 is the unshifted, unscrambled template,
 * columns 1.. the null set.  Per realization r, from the X of ptar_os_project and x = X phi~^{1/2}:
 *   S/N[r][s] = (sum_kd U[r][kd] V[kd][s]) / dsqrt[s]
 *     PTAR_OS_NULL_PHASE_SHIFT   kd = (q, k, c), kd = 2 (q K + k) + c, K = nc / 2, q = (a, b) the pairs of os:
 *                                U[(q,k,0)] = x_a,2k x_b,2k + x_a,2k+1 x_b,2k+1;  U[(q,k,1)] = x_a,2k+1 x_b,2k - x_a,2k x_b,2k+1
 *                                V[(q,k,0)][s] = Gamma_q cos(phi_s,a,k - phi_s,b,k);  V[(q,k,1)][s] = Gamma_q sin(...)
 *     PTAR_OS_NULL_SKY_SCRAMBLE  kd = q:  U[q] = x_a . x_b;  V[q][s] = Gamma^s_q (the template at scrambled positions)
 *   exceed[r] = #{s >= 1 : not S/N[r][s] < S/N[r][0]} (S/N[r][s] >= S/N[r][0], and a NaN column counts);
 *   fap[r] = (1 + exceed[r]) / n_col, NaN when S/N[r][0] is NaN.
 * Three launches: prepare (U, zero past kd), the GEMM on the fp64 tensor cores, count.  Each output is summed in an
 * order fixed by kd only: outputs are bit-identical whatever nreal, chunking or real0.  ptar_os_null_stage runs one
 * launch (stage 1 = prepare, 2 = GEMM, 3 = count; 0 = all three) so a caller can time them. */
#define PTAR_OS_MAX_NULL 65536          /* null columns (n_col - 1) */
#define PTAR_OS_NULL_PHASE_SHIFT  1
#define PTAR_OS_NULL_SKY_SCRAMBLE 2
typedef struct {
  int32_t method;           /* PTAR_OS_NULL_PHASE_SHIFT or PTAR_OS_NULL_SKY_SCRAMBLE                             */
  int32_t n_col;            /* columns: 2 .. PTAR_OS_MAX_NULL + 1                                                */
  int32_t n_colp;           /* n_col rounded up to a multiple of 64                                              */
  int32_t reserved;
  int64_t kd;               /* 2 K n_pairs (phase shift) or n_pairs (sky scramble)                               */
  int64_t kdp;              /* kd rounded up to a multiple of 32                                                 */
  const double* V;          /* [n_colp][kdp]: V^T, row s = column s of V, zero past kd and in rows >= n_col      */
  const double* dsqrt;      /* [n_col] sqrt(D_s)                                                                 */
} ptar_os_null_model;

/* U: scratch of nreal * kdp doubles; snr: [nreal][n_col]; exceed: [nreal] int64; fap: [nreal].  X and os as for
 * ptar_os_pairs. */
int ptar_os_null(const double* X, int32_t nreal, const ptar_os_model* os, const ptar_os_null_model* null_model,
                 double* U, double* snr, int64_t* exceed, double* fap, void* stream);
int ptar_os_null_stage(const double* X, int32_t nreal, const ptar_os_model* os, const ptar_os_null_model* null_model,
                       double* U, double* snr, int64_t* exceed, double* fap, int stage, void* stream);

/* Anisotropy of the optimal statistic (csrc/ptar_os_aniso.cuh): spherical-harmonic fits and radiometer sky maps, from
 * statics derived once on the host.  Per realization r, from the X of ptar_os_project, x = X phi~^{1/2} and the pair
 * correlations d_q = x_a . x_b (q = (a, b) the pairs of os):
 *   map[r][c] = (sum_q d_q V[q][c]) / dsqrt[c],  columns c = [c^_lm (n_lm) | z (n_z) | radiometer S/N (n_sky)]
 *   clm[r][j] = map[r][j];  z[r][j] = map[r][n_lm + j];  chi2[r] = sum_j z[r][j]^2 (fixed tree);
 *   snr_max[r] = max_k map[r][n_lm + n_z + k], argmax[r] = the first k attaining it (NaN ranks above every number);
 *   radio_map[r][k] = map[r][n_lm + n_z + k] when radio_map is not NULL.
 * Three launches: the prepare and GEMM of ptar_os_null (sky-scramble operands: kd = n_pairs) and the reduction.  Each
 * output is summed in an order fixed by q only: outputs are bit-identical whatever nreal, chunking or real0.
 * ptar_os_aniso_stage runs one launch (stage 1 = prepare, 2 = GEMM, 3 = reduce; 0 = all three). */
#define PTAR_OS_ANISO_MAX_LM  64        /* spherical-harmonic coefficients: lmax <= 7 */
#define PTAR_OS_ANISO_MAX_SKY 12288     /* radiometer pixels (HEALPix nside 32)       */
typedef struct {
  int32_t n_lm;             /* (lmax + 1)^2 coefficients, 0 without a spherical-harmonic basis                   */
  int32_t n_z;              /* n_lm - 1 whitened anisotropy components (0 when n_lm <= 1)                         */
  int32_t n_sky;            /* radiometer pixels, 0 without a radiometer; n_lm + n_sky >= 1                       */
  int32_t n_col;            /* n_lm + n_z + n_sky                                                                  */
  int32_t n_colp;           /* n_col rounded up to a multiple of 64                                                */
  int32_t reserved;
  int64_t kd;               /* n_pairs                                                                             */
  int64_t kdp;              /* kd rounded up to a multiple of 32                                                   */
  const double* V;          /* [n_colp][kdp]: V^T, row c = column c of V, zero past kd and in rows >= n_col        */
  const double* dsqrt;      /* [n_col] column divisors (1 for c^ and z, sqrt(F_kk) for the radiometer)             */
} ptar_os_aniso_model;

/* U: scratch of nreal * kdp doubles; map: scratch [nreal][n_col]; clm [nreal][n_lm], z [nreal][n_z], chi2 [nreal]
 * (may be NULL when n_lm = 0; z also when n_z = 0); snr_max [nreal], argmax [nreal] int64 (may be NULL when
 * n_sky = 0); radio_map [nreal][n_sky] or NULL.  X and os as for ptar_os_pairs. */
int ptar_os_aniso(const double* X, int32_t nreal, const ptar_os_model* os, const ptar_os_aniso_model* model, double* U,
                  double* map, double* clm, double* z, double* chi2, double* snr_max, int64_t* argmax,
                  double* radio_map, void* stream);
int ptar_os_aniso_stage(const double* X, int32_t nreal, const ptar_os_model* os, const ptar_os_aniso_model* model,
                        double* U, double* map, double* clm, double* z, double* chi2, double* snr_max, int64_t* argmax,
                        double* radio_map, int stage, void* stream);

/* Per-frequency optimal statistic (csrc/ptar_os_pf.cuh), from statics derived once on the host.  K = nc / 2 GW
 * frequencies f_k; Z_a[k] is the 2 x 2 diagonal block of Z_a at frequency k.  Per realization r, from the unscaled X of
 * ptar_os_project (no phi~ factor), frequency k, pair q = (a, b) of os and template o:
 *   d_qk = X_a,2k X_b,2k + X_a,2k+1 X_b,2k+1;  rho[r][k][q] = d_qk / t[k][q]  (rho may be NULL);
 *   b_ok = sum_q orf[o][q] d_qk;  phi[r][o][k] = b_ok / dnorm[o][k];  snr[r][o][k] = b_ok / dsqrt[o][k];
 *   phi_mc[r][o][k] = sum_o' finv[k][o][o'] b_o'k.
 * One launch.  Each sum runs in an order fixed by q and k only: outputs are bit-identical whatever nreal, chunking or
 * real0. */
typedef struct {
  const double* t;          /* [K][n_pairs] t_qk = tr(Z_a[k] Z_b[k])                                              */
  const double* dnorm;      /* [n_orf][K] D_ok = sum_q Gamma^o_q^2 t_qk                                           */
  const double* dsqrt;      /* [n_orf][K] sqrt(D_ok)                                                              */
  const double* finv;       /* [K][n_orf][n_orf] F_k^{-1}, (F_k)_oo' = sum_q Gamma^o_q Gamma^o'_q t_qk             */
} ptar_os_pf_model;

/* rho: [nreal][K][n_pairs] or NULL; phi, snr, phi_mc: [nreal][n_orf][K].  X as for ptar_os_pairs; os->nc even. */
int ptar_os_pf(const double* X, int32_t nreal, const ptar_os_model* os, const ptar_os_pf_model* pf, double* rho,
               double* phi, double* snr, double* phi_mc, void* stream);

/* Incoherent Fp-statistic (csrc/ptar_fp.cuh).  The host derives, once per recipe, for every pulsar a and search
 * frequency f the whitened basis C~_a(f) = P_a^{-1} F_f L_a(f)^{-T} (F_f = (sin, cos)(2 pi f t), P_a the noise
 * covariance with the timing model marginalised, L_a(f) L_a(f)^T = F_f^T P_a^{-1} F_f).  Per realization r:
 *   ptar_fp_project  amps[r][a][j] = sum_i Ct_a[i][j] rows[r][i] over the TOAs i of pulsar a, j = 2 f + c < 2 n_freq:
 *                    one fp64 tensor-core GEMM launch, one CTA per (pulsar, 64 realizations, 64 columns) walking all of
 *                    the pulsar's TOAs, no partial sums.  rows: ld % 4 == 0, 32-byte aligned; alignment slots ignored.
 *   ptar_fp_reduce   Fp[r][f] = 1/2 sum_a (amps[r][a][2f]^2 + amps[r][a][2f+1]^2), the sum in pulsar order;
 *                    Fp_max[r] = max_f Fp[r][f], Fp_argmax[r] = the first f attaining it (the first NaN above every
 *                    number).
 * Every sum runs in an order fixed by the TOA index and the pulsar only: outputs are bit-identical whatever nreal,
 * chunking, real0 or launch grid produced the rows.  The columns are generic: any whitened basis laid out as Ct is
 * projected the same way (ptar_bwm_sky reads the projection of the whitened memory ramps, column j = epoch j). */
#define PTAR_FP_MAX_FREQ 256   /* search frequencies (the reduce kernel: one thread per frequency) */
typedef struct {
  int32_t n_psr;
  int32_t n_freq;             /* Nf: 1 .. PTAR_FP_MAX_FREQ                                                         */
  int32_t n_cb;               /* column blocks of 64: ceil(2 Nf / 64)                                              */
  int32_t reserved;
  int64_t ld;                 /* TOA pitch of Ct (the packed axis)                                                 */
  const double* Ct;           /* [n_cb][ld][64]: Ct[b][i][(n + 8 (i & 1)) & 63] = C~[i][64 b + n] of the TOA's pulsar;
                                 zero in alignment slots and columns >= 2 Nf                                       */
  const int32_t* psr_order;   /* [n_psr] pulsars in grid order (descending TOA count: the longest CTAs start first) */
  const int64_t* seg_off;     /* [n_psr] packed index of the pulsar's first TOA (multiple of 4)                    */
  const int32_t* seg_len;     /* [n_psr] TOAs of the pulsar                                                        */
} ptar_fp_model;

/* amps: [nreal][n_psr][2 n_freq]. */
int ptar_fp_project(const double* rows, int64_t ld, int32_t nreal, const ptar_fp_model* fp, double* amps, void* stream);
/* Fp: [nreal][n_freq]; Fp_max, Fp_argmax: [nreal]. */
int ptar_fp_reduce(const double* amps, int32_t nreal, const ptar_fp_model* fp, double* Fp, double* Fp_max,
                   int64_t* Fp_argmax, void* stream);
/* ptar_fp_reduce and, when fap is not NULL, fap[r][f] = Q(n_psr, Fp[r][f]) = Gamma(n_psr, Fp) / Gamma(n_psr), the
 * single-frequency false-alarm probability ([nreal][n_freq]).  Evaluated as the finite sum e^{-x} sum_{k < n_psr} x^k / k!
 * from its largest term: relative error <= 4 (Fp + n_psr) 2^-53 (worst measured on an H100: 0.46 of that over every branch, down
 * to subnormal values, where 4 subnormal ulps are added), deterministic per element; 1 at Fp = 0, 0 at +inf, NaN for NaN. */
int ptar_fp_reduce_fap(const double* amps, int32_t nreal, const ptar_fp_model* fp, double* Fp, double* Fp_max,
                       int64_t* Fp_argmax, double* fap, void* stream);

/* Coherent Fe-statistic over a sky grid (csrc/ptar_fe.cuh), from the amplitudes X^ of ptar_fp_project.  The host
 * derives, once per recipe, L_a(f) (M_a(f) = L L^T of the Fp plan), the Earth-term antenna patterns e_a(s) = (F+, Fx)
 * of every pulsar a at every sky point s and, per (f, s), the inverse Cholesky factor of
 * M4(f, s) = sum_a e_a e_a^T (x) M_a(f) (4 x 4, index 2 pol + c, c = 0 sin, 1 cos).  Per realization r:
 *   ptar_fe_sky      N_a(f) = L_a(f) X^[r][a][f] (formed while the operand is staged), then the fp64 tensor-core GEMM
 *                    N4[(f, r, c)][(s, pol)] = sum_a N_a(f)[c] e_a(s)[pol] (the sum in pulsar order) with the epilogue
 *                    Fe[r][f][s] = 1/2 |L4^-1 N4|^2 in registers, and fmax[r][f] = max_s Fe, fargmax[r][f] = the first
 *                    s attaining it.  maps != NULL also writes Fe [nreal][n_freq][n_sky]; otherwise no map is written.
 *   ptar_fe_combine  fe_max[r] = max_f fmax[r][f]; argmax_f[r] = the first f attaining it, argmax_sky[r] = its fargmax.
 * Outputs are bit-identical whatever nreal, chunking or real0 produced the amplitudes. */
#define PTAR_FE_MAX_PSR 128     /* pulsars: the staged N tile and two antenna stages, 199 KB of shared memory at 128 */
#define PTAR_FE_MAX_SKY 12288   /* sky points: 12 nside^2 at nside 32 */
typedef struct {
  int32_t n_psr;              /* 1 .. PTAR_FE_MAX_PSR                                                              */
  int32_t n_freq;             /* as the Fp model                                                                   */
  int32_t n_sky;              /* S: 1 .. PTAR_FE_MAX_SKY                                                           */
  int32_t n_sb;               /* sky blocks of 32: ceil(S / 32)                                                    */
  int32_t kp;                 /* n_psr rounded up to a multiple of 16                                              */
  int32_t reserved;
  const double* Lf;           /* [n_freq][n_psr][3]: l11, l21, l22 of M_a(f)                                       */
  const double* ant;          /* [n_sb][kp][64]: ant[b][a][(j + 8 (a & 1)) & 63] = e_a(32 b + j / 2)[j & 1]; zero
                                 past n_psr and n_sky                                                              */
  const double* linv;         /* [n_freq][32 n_sb][10]: L4^-1 packed by rows (00, 10, 11, 20, 21, 22, 30 .. 33);
                                 zero past n_sky                                                                   */
} ptar_fe_model;

/* amps: [nreal][n_psr][2 n_freq] (ptar_fp_project); fmax: [nreal][n_freq]; fargmax: [nreal][n_freq] int64. */
int ptar_fe_sky(const double* amps, int32_t nreal, const ptar_fe_model* fe, double* fmax, int64_t* fargmax, double* maps,
                void* stream);
/* fe_max, argmax_f, argmax_sky: [nreal]. */
int ptar_fe_combine(const double* fmax, const int64_t* fargmax, int32_t nreal, const ptar_fe_model* fe, double* fe_max,
                    int64_t* argmax_f, int64_t* argmax_sky, void* stream);

/* Burst-with-memory search over epoch x sky (csrc/ptar_bwm.cuh), from the amplitudes X^ of ptar_fp_project run with a
 * ptar_fp_model whose Ct holds the whitened ramps (n_freq = ceil(T / 2), column j = epoch j, zero for an unseen epoch).
 * The host derives, once per recipe, for every pulsar a and burst epoch t0 the ramp u = (t - t0) [t >= t0], its Fisher
 * information m_a(t0) = u^T P_a^-1 u (P_a the noise covariance with the timing model marginalised; 0 for an epoch the
 * pulsar does not see), C~_a(t0) = P_a^-1 u / sqrt(m_a(t0)), the Earth-term antenna patterns e_a(s) = (F+, Fx) and, per
 * (t0, s), the inverse Cholesky factor of M2(t0, s) = sum_a e_a e_a^T m_a(t0).  Per realization r:
 *   ptar_bwm_sky      N2[(r, t)][(s, pol)] = sum_a sqrt(m_a(t)) X^[r][a][t] e_a(s)[pol] on the fp64 tensor cores (the sum
 *                     in pulsar order) with the epilogue B[r][t][s] = 1/2 |L2^-1 N2|^2 in registers (2B ~ chi^2_2 under the
 *                     noise model); t0max[r][t] = max_s B, t0argmax[r][t] = the first s attaining it.  maps != NULL also
 *                     writes B [nreal][n_t0][n_sky]; otherwise no map is written.
 *   ptar_bwm_combine  bwm_max[r] = max_t t0max[r][t], argmax_t0[r] = the first t attaining it, argmax_sky[r] = its
 *                     t0argmax; fap[r] = exp(-bwm_max); at that cell b^ = M2^-1 N2 (N2 re-formed in pulsar order),
 *                     strain[r] = |b^|, pol[r] = 1/2 atan2(b^_x, b^_+) mod pi.  Per (r, a) over the epochs a sees:
 *                     psr_max[r][a] = max_t 1/2 X^[r][a][t]^2, psr_argmax_t0 the first t attaining it, psr_slope =
 *                     X^ / sqrt(m_a(t)) there and psr_fap = erfc(sqrt(psr_max)); a pulsar that sees no epoch gets -inf,
 *                     index -1 and NaN slope and fap.
 * Outputs are bit-identical whatever nreal, chunking or real0 produced the amplitudes. */
#define PTAR_BWM_MAX_EPOCH 512   /* burst epochs: 2 PTAR_FP_MAX_FREQ projection columns */
typedef struct {
  int32_t n_psr;              /* 1 .. PTAR_FE_MAX_PSR                                                              */
  int32_t n_t0;               /* T: 1 .. PTAR_BWM_MAX_EPOCH                                                        */
  int32_t n_sky;              /* S: 1 .. PTAR_FE_MAX_SKY                                                           */
  int32_t n_sb;               /* sky blocks of 32: ceil(S / 32)                                                    */
  int32_t kp;                 /* n_psr rounded up to a multiple of 16                                              */
  int32_t reserved;
  const double* sqm;          /* [ceil(T / 2)][n_psr][2]: sqrt(m_a(2 q + c)); zero for an unseen epoch and past T     */
  const uint8_t* seen;        /* [n_psr][T]: 1 where pulsar a sees epoch t                                          */
  const double* ant;          /* [n_sb][kp][64]: the layout of ptar_fe_model.ant                                   */
  const double* antenna;      /* [n_psr][n_sky][2]: e_a(s) = (F+, Fx)                                              */
  const double* linv;         /* [ceil(T / 2)][32 n_sb][6]: L2^-1 (00, 10, 11) of epoch 2 q, then of 2 q + 1; zero past
                                 n_sky and T                                                                       */
} ptar_bwm_model;

/* amps: [nreal][n_psr][2 ceil(T / 2)] (ptar_fp_project); t0max: [nreal][n_t0]; t0argmax: [nreal][n_t0] int64. */
int ptar_bwm_sky(const double* amps, int32_t nreal, const ptar_bwm_model* bw, double* t0max, int64_t* t0argmax,
                 double* maps, void* stream);
/* bwm_max, strain, pol, fap: [nreal]; argmax_t0, argmax_sky: [nreal] int64; psr_max, psr_slope, psr_fap: [nreal][n_psr];
 * psr_argmax_t0: [nreal][n_psr] int64. */
int ptar_bwm_combine(const double* amps, const double* t0max, const int64_t* t0argmax, int32_t nreal,
                     const ptar_bwm_model* bw, double* bwm_max, int64_t* argmax_t0, int64_t* argmax_sky, double* strain,
                     double* pol, double* fap, double* psr_max, int64_t* psr_argmax_t0, double* psr_slope,
                     double* psr_fap, void* stream);

/* Sine-Gaussian burst search over a t0 x f0 x Q template bank and the sky (csrc/ptar_burst.cuh).  Template j = (t0, f0,
 * Q), tau = Q / (2 pi f0), W_j(t) = exp(-(t - t0)^2 / tau^2) (cos, sin)(2 pi f0 (t - t0)) on the TOAs of its static window
 * [lo, hi) (the range spanning |t - t0| <= 6 tau; zero outside), t = MJD 86400.  The host derives, once per recipe, with
 * P_a^-1 = N^-1 - N^-1 T S^-1 T^T N^-1 (N = white + ECORR, T = timing model, red noise and common basis, S = L_S L_S^T):
 * the z columns N^-1 T L_S^-T (a ptar_fp_model: ptar_fp_project gives z_a = L_S^-1 T^T N^-1 r_a), H_a(j) =
 * L_S^-1 T^T N^-1 W_j, M_a(j) = W_j^T P_a^-1 W_j = L L^T and the sky statics of ptar_fe_sky.  Per realization r:
 *   ptar_burst_ninv     y = N^-1 r on the packed axis (1/d per TOA, one Sherman-Morrison term per ECORR run, runs summed
 *                       in TOA order); only the TOAs of the runs are written.
 *   ptar_burst_project  for the templates of group g (bank indices 256 g .. 256 g + Jg - 1, Jg <= PTAR_BURST_GROUP):
 *                       amps[r][a][2 jl + c] = (L^-1 (W_j^T y_a - H_a(j)^T z_a))[c], 0 for an unseen (a, j): the layout of
 *                       ptar_fp_project with n_freq = Jg, so ptar_fe_sky (Lf = l11, l21, l22 of M_a(j)) runs on it unchanged.
 *                       W_j is generated per TOA chunk on the device; the GEMM runs on the fp64 tensor cores and walks only
 *                       the union of a 16-template block's windows.  y: ld % 4 == 0, 32-byte aligned.
 *   ptar_burst_reduce   from the amps of every group (group g's block at amps + 256 g nreal n_psr 2) and ptar_fe_sky's
 *                       per-template maxima jmax / jargmax (group g's [nreal][Jg] block at + 256 g nreal): B_tmpl[r][j] and
 *                       B_tmpl_sky[r][j] (their copy in bank order), B_max[r] = max_j, argmax_tmpl / argmax_sky (ties to the
 *                       lower template, then the lower sky index), fap[r] = e^-B (1 + B) and amp[r][4] = -M4^-1 N4 at that
 *                       cell (add_burst's h+ = a0 g cos + a1 g sin, hx = a2 g cos + a3 g sin at psi = 0).  Per (r, a) over
 *                       the templates a sees: Bt_max[r][a] = max 1/2 |X^|^2, argmax_psr, fap_psr = e^-Bt and, when amp_psr
 *                       is not NULL, amp_psr[r][a][2] = M_a^-1 N_a (add_noise_transient's waveform = a0 g cos + a1 g sin); a
 *                       pulsar that sees no template gets -inf, index -1 and NaN.  bt_maps != NULL also writes every
 *                       1/2 |X^|^2 [nreal][n_psr][n_tmpl].
 * Outputs are bit-identical whatever nreal, chunking or real0 produced the rows. */
#define PTAR_BURST_MAX_TEMPLATE 4096   /* templates of a bank */
#define PTAR_BURST_GROUP 256           /* templates per ptar_burst_project / ptar_fe_sky call: PTAR_FP_MAX_FREQ */
#define PTAR_BURST_TB 16               /* templates per CTA of ptar_burst_project (blk holds one range per block) */
typedef struct {
  int32_t n_psr;              /* 2 .. PTAR_FE_MAX_PSR                                                              */
  int32_t n_tmpl;             /* J: 1 .. PTAR_BURST_MAX_TEMPLATE                                                   */
  int32_t n_zc;               /* z columns per pulsar: 2 n_freq of the z projection's ptar_fp_model                */
  int32_t n_run;              /* N^-1 runs on the packed axis                                                      */
  int32_t n_sky;              /* S, as ptar_fe_model                                                               */
  int32_t n_sb;               /* ceil(S / 32)                                                                      */
  const double* t;            /* [ld] MJD 86400 of every TOA                                                       */
  const double* dinv;         /* [ld] 1 / white variance                                                           */
  const int64_t* run_start;   /* [n_run] packed index of the run's first TOA                                       */
  const int32_t* run_len;     /* [n_run]                                                                           */
  const double* run_coef;     /* [n_run] e^2 / (1 + e^2 sum 1/d) of the run's ECORR e (0 without)                  */
  const int32_t* toa_run;     /* [ld] run of every TOA, -1 in alignment slots                                      */
  const double* tmpl;         /* [J][4]: t0 [s], 1 / tau, 2 f0, 0                                                  */
  const int32_t* win;         /* [n_psr][J][2]: window [lo, hi) of local TOA indices (lo = hi: empty)              */
  const int32_t* blk;         /* [n_psr][ceil(J / 16)][2]: union of the block's windows, lo a multiple of 4        */
  const double* H;            /* [n_psr][J][2][n_zc]: H_a(j)^T, zero past the pulsar's rank                        */
  const double* wl;           /* [n_psr][J][3]: L^-1 packed (00, 10, 11); zero for an unseen cell                  */
  const double* Lf;           /* [J][n_psr][3]: l11, l21, l22 of M_a(j); zero for an unseen cell                   */
  const double* linv;         /* [J][32 n_sb][10]: L4^-1 of M4(j, s) as ptar_fe_model.linv                         */
  const double* antenna;      /* [n_psr][n_sky][2]: e_a(s) = (F+, Fx)                                              */
  const uint8_t* seen;        /* [n_psr][J]: 1 where pulsar a sees template j                                      */
  const int32_t* psr_order;   /* [n_psr] pulsars in grid order (descending TOA count)                              */
  const int64_t* seg_off;     /* [n_psr] packed index of the pulsar's first TOA (multiple of 4)                    */
} ptar_burst_model;

/* y: [nreal][ld]. */
int ptar_burst_ninv(const double* rows, int64_t ld, int32_t nreal, const ptar_burst_model* bm, double* y, void* stream);
/* z: [nreal][n_psr][n_zc] (ptar_fp_project); amps: [nreal][n_psr][2 Jg] of group `group`. */
int ptar_burst_project(const double* y, int64_t ld, int32_t nreal, const double* z, const ptar_burst_model* bm, int32_t group,
                       double* amps, void* stream);
/* amps: every group's block; jmax, jargmax: every group's [nreal][Jg] block; B_tmpl, B_tmpl_sky: [nreal][J]; B_max, fap,
 * argmax_tmpl, argmax_sky: [nreal]; amp: [nreal][4]; Bt_max, fap_psr, argmax_psr: [nreal][n_psr]; amp_psr: [nreal][n_psr][2]
 * or NULL; bt_maps: [nreal][n_psr][J] or NULL. */
int ptar_burst_reduce(const double* amps, const double* jmax, const int64_t* jargmax, int32_t nreal, const ptar_burst_model* bm,
                      double* B_tmpl, int64_t* B_tmpl_sky, double* B_max, int64_t* argmax_tmpl, int64_t* argmax_sky,
                      double* fap, double* amp, double* Bt_max, int64_t* argmax_psr, double* fap_psr, double* amp_psr,
                      double* bt_maps, void* stream);

/* Common uncorrelated red process (CURN) likelihood on an (A, gamma) grid (csrc/ptar_curn.cuh), from the X of
 * ptar_os_project run with a ptar_os_model that holds only the projection fields (tiles, tile0, n_tile, C, nc, ncp).
 * The host derives, once per recipe, for every pulsar a and grid gamma the eigendecomposition
 * phi~^{1/2} Z_a phi~^{1/2} = U diag(lambda) U^T (Z_a = F^T P_a^{-1} F, phi~ the power law at A = 1 and gamma),
 * V_a(gamma) = U^T phi~^{1/2}, ldet[g][k] = sum_a sum_j log1p(A_k^2 lambda_j), and the trapezoid weights and prior of
 * the grid.  Per realization r:
 *   ptar_curn_grid    lnL[r][g][k] = 1/2 sum_a sum_j w_j y_j^2 - 1/2 ldet[g][k],  y = V_a(gamma_g) X[r][a],
 *                     w_j = A_k^2 / (1 + A_k^2 lambda_j): two chained GEMMs on the fp64 tensor cores, the pulsar sum in
 *                     index order.  X: [nreal][n_psr][ncp], 32-byte aligned.
 *   ptar_curn_reduce  lnL_max[r], its first (g, k) (gamma-major) in ml_gamma[r], ml_amp[r];
 *                     ln_bayes[r] = ln sum_{g,k} wg_g wx_k prior_k exp(lnL[r][g][k]);
 *                     post_amp[r][k] = sum_g wg_g prior_k exp(lnL) / B;  post_gamma[r][g] = sum_k wx_k prior_k exp(lnL) / B;
 *                     ul_amp[r] = the quantile ul of the trapezoid CDF of post_amp over log10_A, linear between nodes.
 *                     Non-finite maps: see "Non-finite inputs" at the top.
 * Every sum runs in an order fixed by the pulsar, the grid index and the realization's own data: outputs are
 * bit-identical whatever nreal, chunking or real0. */
#define PTAR_CURN_MAX_NA 256    /* log10 A grid points (one reduce thread per point) */
#define PTAR_CURN_MAX_NG 256    /* gamma grid points                                 */
typedef struct {
  int32_t n_psr;
  int32_t nc;                 /* 2K <= PTAR_OS_MAX_NC                                                              */
  int32_t ncp;                /* nc rounded up to a multiple of 8 (as the ptar_os_model of the projection)         */
  int32_t n_gamma;            /* 1 .. PTAR_CURN_MAX_NG                                                             */
  int32_t n_amp;              /* 2 .. PTAR_CURN_MAX_NA                                                             */
  int32_t reserved;
  const double* V;            /* [n_psr][n_gamma][ncp][ncp]: row j = eigenvector j of phi~^1/2 Z_a phi~^1/2 times
                                 phi~^1/2; zero in rows and columns >= nc                                          */
  const double* lam;          /* [n_psr][n_gamma][ncp]: eigenvalues (>= 0), zero past nc                           */
  const double* a2;           /* [n_amp] A^2 = 10^(2 log10_A)                                                      */
  const double* ldet;         /* [n_gamma][n_amp]                                                                  */
  const double* log10_A;      /* [n_amp] strictly increasing                                                       */
  const double* wg;           /* [n_gamma] trapezoid weights in gamma (1 for one point)                            */
  const double* wx;           /* [n_amp] trapezoid weights in log10 A                                              */
  const double* prior;        /* [n_amp] prior density, normalised: sum_g sum_k wg wx prior = 1                    */
  double ul;                  /* upper-limit quantile in (0, 1)                                                    */
} ptar_curn_model;

/* ptar_curn_grid reads every field; ptar_curn_reduce reads, and checks, only the grid: log10_A, wg, wx, prior, n_amp,
 * n_gamma and ul.  lnL: [nreal][n_gamma][n_amp]. */
int ptar_curn_grid(const double* X, int32_t nreal, const ptar_curn_model* cm, double* lnL, void* stream);
/* lnL_max, ln_bayes, ul_amp: [nreal]; ml_gamma, ml_amp: [nreal] int64; post_amp: [nreal][n_amp];
 * post_gamma: [nreal][n_gamma]. */
int ptar_curn_reduce(const double* lnL, int32_t nreal, const ptar_curn_model* cm, double* lnL_max, int64_t* ml_gamma,
                     int64_t* ml_amp, double* ln_bayes, double* post_amp, double* post_gamma, double* ul_amp,
                     void* stream);

/* Hellings-Downs (ORF-correlated) common-process likelihood (csrc/ptar_hd.cuh) on the grid of a ptar_curn_model, from
 * the same X.  With the ORF Gamma = B B^T (n_psr x n_psr, positive semi-definite) and G = B (x) phi~^{1/2}, the host
 * derives once per recipe, for every grid gamma, the eigendecomposition G^T Z G = U diag(lambda) U^T of size
 * n = n_psr nc (Z = blockdiag(Z_a)), V(gamma) = U^T G^T and ldet[g][k] = sum_j log1p(A_k^2 lambda_j).  Per realization r:
 *   ptar_hd_grid  lnL[r][g][k] = 1/2 sum_j w_j y_j^2 - 1/2 ldet[g][k],  y = V(gamma_g) X[r] (X[r] stacked over the
 *                 pulsars), w_j = A_k^2 / (1 + A_k^2 lambda_j): two chained GEMMs on the fp64 tensor cores, j and the
 *                 stacked X axis in index order.  X: [nreal][n_psr][ncp], 32-byte aligned.
 * The summaries of the map are ptar_curn_reduce's, with the ptar_curn_model of the grid.  Outputs are bit-identical
 * whatever nreal, chunking or real0. */
#define PTAR_HD_MAX_N 4096      /* n = n_psr nc eigen-rows                                    */
#define PTAR_HD_JB    32        /* eigen-rows per block: np = n rounded up to a multiple of 32 */
typedef struct {
  int32_t n_psr;
  int32_t nc;                 /* 2K <= PTAR_OS_MAX_NC                                                              */
  int32_t ncp;                /* nc rounded up to a multiple of 8 (as the ptar_os_model of the projection)         */
  int32_t n_gamma;            /* 1 .. PTAR_CURN_MAX_NG                                                             */
  int32_t n_amp;              /* 2 .. PTAR_CURN_MAX_NA                                                             */
  int32_t n;                  /* n_psr nc <= PTAR_HD_MAX_N                                                          */
  int32_t np;                 /* n rounded up to a multiple of PTAR_HD_JB                                           */
  int32_t reserved;
  const double* V;            /* [n_gamma][np][n_psr][ncp]: row j = eigenvector j of G^T Z G times G^T; zero in rows
                                 >= n and in the columns of each pulsar >= nc; 16-byte aligned                     */
  const double* lam;          /* [n_gamma][np]: eigenvalues (>= 0), zero past n                                    */
  const double* a2;           /* [n_amp] A^2 = 10^(2 log10_A)                                                      */
  const double* ldet;         /* [n_gamma][n_amp]                                                                  */
} ptar_hd_model;

/* lnL: [nreal][n_gamma][n_amp]. */
int ptar_hd_grid(const double* X, int32_t nreal, const ptar_hd_model* hm, double* lnL, void* stream);

/* Single-pulsar intrinsic red-noise likelihood on an (A, gamma) grid (csrc/ptar_rn.cuh), from the X of ptar_os_project
 * run on each pulsar's own red-noise basis F_a (f_k = k / T_a, nc = 2K <= PTAR_RN_MAX_NC).  The host derives, once per
 * recipe, for every pulsar a and grid gamma the eigendecomposition phi~_a^{1/2} Z_a phi~_a^{1/2} = U diag(lambda) U^T
 * (Z_a = F_a^T P_a^{-1} F_a, P_a without the pulsar's own red noise, phi~_a the power law at A = 1, gamma and T_a),
 * V_a(gamma) = U^T phi~_a^{1/2} and ldet[a][g][k] = sum_j log1p(A_k^2 lambda_j).  Per realization r:
 *   ptar_rn_grid  lnL[r][a][g][k] = 1/2 sum_j w_j y_j^2 - 1/2 ldet[a][g][k],  y = V_a(gamma_g) X[r][a],
 *                 w_j = A_k^2 / (1 + A_k^2 lambda_j): two chained GEMMs on the fp64 tensor cores, no sum over pulsars.
 *                 X: [nreal][n_psr][ncp], 32-byte aligned.
 * The summaries of the nreal * n_psr maps [r][a] are ptar_curn_reduce's, called with nreal * n_psr and a
 * ptar_curn_model carrying only the grid (log10_A, wg, wx, prior, ul, n_amp, n_gamma).  Outputs are bit-identical whatever
 * nreal, chunking or real0. */
typedef struct {
  int32_t n_psr;              /* n_psr * ceil(n_gamma / 16) <= 65535                                               */
  int32_t nc;                 /* 2K <= PTAR_RN_MAX_NC                                                              */
  int32_t ncp;                /* nc rounded up to a multiple of 8 (as the ptar_os_model of the projection)         */
  int32_t n_gamma;            /* 1 .. PTAR_CURN_MAX_NG                                                             */
  int32_t n_amp;              /* 2 .. PTAR_CURN_MAX_NA                                                             */
  int32_t reserved;
  const double* V;            /* [n_psr][n_gamma][ncp][ncp]: row j = eigenvector j of phi~_a^1/2 Z_a phi~_a^1/2 times
                                 phi~_a^1/2; zero in rows and columns >= nc; 16-byte aligned                       */
  const double* lam;          /* [n_psr][n_gamma][ncp]: eigenvalues (>= 0), zero past nc                           */
  const double* a2;           /* [n_amp] A^2 = 10^(2 log10_A)                                                      */
  const double* ldet;         /* [n_psr][n_gamma][n_amp]                                                           */
} ptar_rn_model;

/* lnL: [nreal][n_psr][n_gamma][n_amp]. */
int ptar_rn_grid(const double* X, int32_t nreal, const ptar_rn_model* rm, double* lnL, void* stream);

/* Factorised free-spectrum likelihood on a log10 rho grid (csrc/ptar_fs.cuh), one 1-D grid per GW frequency bin k, from
 * the X of ptar_os_project on the 2K columns of the bins (column pair k of C is P_a,k^{-1} F_k, P_a,k the noise model of
 * bin k).  The model of bin k is a common process in bin k alone, phi_k = rho^2 per Fourier coefficient, uncorrelated
 * (Gamma = I) or with an ORF Gamma = B B^T.  The host derives, once per recipe, for every bin the eigendecomposition
 * G^T Z[k] G = U diag(lambda) U^T of size n = 2 n_psr (Z[k] = blockdiag_a F_k^T P_a,k^{-1} F_k, G = B (x) I_2),
 * V_k = U^T G^T and ldet[k][i] = sum_j log1p(rho_i^2 lambda_j).  Per realization r:
 *   ptar_fs_grid  lnL[r][k][i] = 1/2 sum_j w_j y_j^2 - 1/2 ldet[k][i],  y = V_k X_k[r] with X_k[r][2a + c] =
 *                 X[r][a][2k + c] (the bin-k columns of every pulsar, gathered), w_j = rho_i^2 / (1 + rho_i^2 lambda_j):
 *                 two chained GEMMs on the fp64 tensor cores, j and the gathered axis in index order.
 *                 X: [nreal][n_psr][ncp], 32-byte aligned.
 * The summaries of the nreal * n_bin maps [r][k] are ptar_curn_reduce's, called with nreal * n_bin and a ptar_curn_model
 * carrying only the grid (log10_A = log10 rho, wg = {1}, wx, prior, ul, n_amp, n_gamma = 1).  Outputs are bit-identical
 * whatever nreal, chunking or real0. */
#define PTAR_FS_MAX_PSR 256     /* pulsars: n = 2 n_psr eigen-rows per bin                     */
#define PTAR_FS_MAX_BIN 32      /* frequency bins (2K <= PTAR_RN_MAX_NC projection columns)    */
#define PTAR_FS_JB      32      /* eigen-rows per block: np = 2 n_psr rounded up to a multiple of 32 */
typedef struct {
  int32_t n_psr;              /* 1 .. PTAR_FS_MAX_PSR                                                              */
  int32_t ncp;                /* 2 n_bin rounded up to a multiple of 8 (as the ptar_os_model of the projection)    */
  int32_t n_bin;              /* K, 1 .. PTAR_FS_MAX_BIN                                                           */
  int32_t n_amp;              /* 2 .. PTAR_CURN_MAX_NA log10 rho points                                            */
  int32_t n2p;                /* 2 n_psr rounded up to a multiple of 8: the row pitch of V                          */
  int32_t np;                 /* 2 n_psr rounded up to a multiple of PTAR_FS_JB                                    */
  const double* V;            /* [n_bin][np][n2p]: row j = eigenvector j of G^T Z[k] G times G^T on the gathered axis
                                 (2a + c); zero in rows >= 2 n_psr and columns >= 2 n_psr; 16-byte aligned        */
  const double* lam;          /* [n_bin][np]: eigenvalues (>= 0), zero past 2 n_psr                                */
  const double* a2;           /* [n_amp] rho^2 = 10^(2 log10 rho)                                                  */
  const double* ldet;         /* [n_bin][n_amp]                                                                    */
} ptar_fs_model;

/* lnL: [nreal][n_bin][n_amp]. */
int ptar_fs_grid(const double* X, int32_t nreal, const ptar_fs_model* fm, double* lnL, void* stream);

/* Spectral refit of the factorised free spectrum (csrc/ptar_fs_refit.cuh): for a spectral model on a grid of n_tmpl
 * templates t, each with a GW variance rho_k(t)^2 per Fourier coefficient in every bin k of a free-spectrum model
 * (a ptar_fs_model, uncorrelated or ORF-correlated), the sum over the bins of its per-bin log-likelihood ratios,
 *   lnL[r][t] = sum_k ln L_k(rho_k(t)) = 1/2 sum_k sum_j w_kj(t) y_kj^2 - 1/2 ldet[t],
 *   w_kj(t) = rho_k(t)^2 / (1 + rho_k(t)^2 lambda_kj),  y_k = V_k X_k[r],  ldet[t] = sum_k sum_j log1p(rho_k(t)^2 lambda_kj),
 * exact for the factorised model at any rho (no interpolation in a log10 rho grid).
 *   ptar_fs_y2     y2[r][k][j] = (V_k X_k[r])_j^2 for j < np (0 past 2 n_psr) with the ptar_fs_model fm (reads n_psr, ncp,
 *                  n_bin, n2p, np and V), the first GEMM of ptar_fs_grid.  X: [nreal][n_psr][ncp], 32-byte aligned;
 *                  y2: [nreal][n_bin][np], 16-byte aligned.
 *   ptar_fs_refit  lnL[r][t] from y2: one GEMM of depth n_bin np on the fp64 tensor cores, W formed on the fly, the
 *                  depth in (k, j) index order.  lnL: [nreal][n_tmpl].
 * A model grid (x [Nx], y [Ny]) is laid out t = i_y Nx + i_x, so its summaries are ptar_curn_reduce's with a
 * ptar_curn_model carrying only that grid (log10_A = x, gamma = y, n_amp = Nx, n_gamma = Ny).  Outputs are
 * bit-identical whatever nreal, chunking or real0. */
#define PTAR_FS_MAX_TEMPLATE 65536   /* templates: the 256 x 256 grid of ptar_curn_reduce */
typedef struct {
  int32_t n_bin;              /* K, 1 .. PTAR_FS_MAX_BIN                                                           */
  int32_t np;                 /* the np of the ptar_fs_model: 2 n_psr rounded up to a multiple of PTAR_FS_JB       */
  int32_t n_tmpl;             /* 1 .. PTAR_FS_MAX_TEMPLATE                                                         */
  int32_t reserved;
  const double* lam;          /* [n_bin][np]: the ptar_fs_model's eigenvalues (>= 0), zero past 2 n_psr            */
  const double* rho2;         /* [n_bin][n_tmpl] rho_k(t)^2 (finite, >= 0)                                         */
  const double* ldet;         /* [n_tmpl]                                                                          */
} ptar_fs_refit_model;

int ptar_fs_y2(const double* X, int32_t nreal, const ptar_fs_model* fm, double* y2, void* stream);
int ptar_fs_refit(const double* y2, int32_t nreal, const ptar_fs_refit_model* rm, double* lnL, void* stream);

/* Per-realization continuous-wave populations (csrc/ptar_cwpop.cuh).  Every realization r of [real0, real0 + nreal)
 * gets n_src sources; each source parameter j is fixed (kind PTAR_CWPOP_FIXED: lo), uniform (PTAR_CWPOP_UNIFORM:
 * lo + width u) or isotropic (PTAR_CWPOP_ACOS: acos(lo + width u), lo = -1, width = 2), the affine map rounded operation
 * by operation.  The uniforms u are 53-bit, (a >> 5) 2^26 + (b >> 6) times 2^-53, from the Philox4x32-10 words
 * (a, b) = (w.x, w.y) and (w.z, w.w) of the counter (source * 16 + j / 2, PTAR_K_CWPOP, r & 0xffffffff, r >> 32):
 * parameter j takes the first word pair for even j and the second for odd j.  With pphase the pulsar-term phase of pulsar
 * p is 2 pi u, u the first pair of (source * 16 + 4, PTAR_K_CWPOP | p << 8, r).  Parameters are drawn whether or not
 * they are used, so a draw does not depend on the others' kinds; the noise streams (kinds 1-6) are untouched.
 * From the draws: h0, fgw and Mc are 10^(log10 value); d_L = 2 Mc^(5/3) (pi fgw)^(2/3) / h0 (geometric units), and the
 * source is then add_cgw's (deterministic.py:13-163) with pdist [kpc] or the drawn pulsar phase, mode 0 (evolve),
 * 1 (phase_approx) or 2 (monochromatic) and psr_term.  A source whose 1 + Omega.p is below PTAR_CWPOP_POLE_TOL
 * (or NaN) at pulsar p has antenna pattern (0, 0) there; a NaN contribution (a merged binary) is dropped.
 *   stage 1 (draw)  scratch <- per-(r, s) source scalars [nreal][n_src][16] and per-(r, s, p) pulsar constants
 *                   [nreal][n_src][n_psr][8]; params (optional) <- [nreal][n_src][PTAR_CWPOP_TABLE] = {gwtheta, gwphi,
 *                   phase0, psi, inc, log10_h0, log10_fgw, log10_mc, dist [Mpc], fgw, Mc, h0, 0, 0, 0, 0}, followed with
 *                   pphase by [nreal][n_src][n_psr] pulsar phases.
 *   stage 2 (add)   rows[r][i] += sum_s delay of source s at slot i for every slot with slot_psr[i] >= 0.
 * ptar_cw_population runs both (stage 0 of ptar_cw_population_stage); with rows == NULL it only draws.
 * scratch_len >= nreal * n_src * (16 + 8 n_psr).  Outputs are bit-identical whatever nreal, chunking or real0. */
#define PTAR_CWPOP_MAX_SRC 64    /* sources per realization                                               */
#define PTAR_CWPOP_NPAR    8     /* drawn parameters per source                                           */
#define PTAR_CWPOP_TABLE   16    /* doubles per (r, s) row of the parameter table                          */
#define PTAR_CWPOP_POLE_TOL 1e-12
#define PTAR_CWPOP_FIXED   0
#define PTAR_CWPOP_UNIFORM 1
#define PTAR_CWPOP_ACOS    2
#define PTAR_CWPOP_LOG10_H0  0   /* parameter indices: the order of the counter's parameter pairs          */
#define PTAR_CWPOP_LOG10_FGW 1
#define PTAR_CWPOP_LOG10_MC  2
#define PTAR_CWPOP_GWTHETA   3
#define PTAR_CWPOP_GWPHI     4
#define PTAR_CWPOP_PHASE0    5
#define PTAR_CWPOP_PSI       6
#define PTAR_CWPOP_INC       7
typedef struct {
  int32_t n_psr;                       /* >= 1                                                                 */
  int32_t n_src;                       /* 1 .. PTAR_CWPOP_MAX_SRC                                              */
  int32_t mode;                        /* 0 evolve, 1 phase_approx, 2 monochromatic                            */
  int32_t psr_term;                    /* 1: Earth and pulsar terms, 0: Earth term only                        */
  int32_t pphase;                      /* 1: pulsar-term phase drawn per (r, s, p), pd from it; 0: pd = pdist  */
  int32_t kind[PTAR_CWPOP_NPAR];       /* PTAR_CWPOP_FIXED / _UNIFORM / _ACOS                                  */
  int32_t reserved;
  double lo[PTAR_CWPOP_NPAR];
  double width[PTAR_CWPOP_NPAR];
  const double* phat;                  /* [n_psr][3] pulsar unit vectors                                       */
  const double* pdist;                 /* [n_psr] pulsar distances [kpc] (may be NULL with pphase)             */
  const double* slot_t;                /* [ld] TOA (MJD 86400) - tref [s] per slot of the packed axis          */
  const int32_t* slot_psr;             /* [ld] pulsar of each slot, -1 for alignment slots (never written)     */
} ptar_cwpop_model;

int ptar_cw_population(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed, const ptar_cwpop_model* m,
                       double* scratch, int64_t scratch_len, double* params, void* stream);
int ptar_cw_population_stage(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed,
                             const ptar_cwpop_model* m, double* scratch, int64_t scratch_len, double* params, int stage,
                             void* stream);

/* Per-realization common-process populations (csrc/ptar_cpop.cuh).  Every realization r of [real0, real0 + nreal)
 * gets the Fourier coefficients c[r][a][2k + s] = sqrt(phi_k(r)) sum_b B_ab z[r][b][2k + s] of a common process on the
 * basis F_a = (sin, cos)(2 pi f_k t) (s = 0, 1), f_k = freqs[k], k < K, and rows[r][i] += sum_j c[r][p(i)][j] F_j(t_i).
 * Hyperparameters: uniforms u through cwpop_param's affine map (kind PTAR_CWPOP_FIXED: lo, PTAR_CWPOP_UNIFORM:
 * lo + width u, each operation rounded once).  The power law (PTAR_CPOP_POWERLAW) draws h = (log10_A, gamma) and has
 * phi_k = A^2 phi~_k, A = 10^log10_A, phi~_k = (pl_x[k]^-gamma / pl_den) pl_y3 (engine._powerlaw_prior's operations:
 * pl_x[k] = f_k yr, pl_den = 12 pi^2 Tspan, pl_y3 = yr^3); the free spectrum (PTAR_CPOP_FREE) draws h = log10_rho_k
 * per bin (kind[0], lo[0], width[0] for every bin) and has sqrt(phi_k) = 10^log10_rho_k.
 * Counters of Philox4x32-10, (c.z, c.w) = the full global realization id:
 *   hyperparameter pair j / 2:  (PTAR_CPOP_HYPER + j / 2, PTAR_K_CPOP, r); h_j takes the word pair (w.x, w.y) for even
 *                               j and (w.z, w.w) for odd j, each a 53-bit uniform (a >> 5) 2^26 + (b >> 6) times 2^-53;
 *   normals of pulsar b, bin k: (k, PTAR_K_CPOP | b << 8, r); u1, u2 the two 53-bit uniforms, rho = sqrt(-2 ln(1 - u1)),
 *                               theta = 2 pi u2: z[r][b][2k] = rho cos theta, z[r][b][2k + 1] = rho sin theta (fp64).
 * The noise streams (kinds 1-7) are untouched, so every realization's noise is what it is without a population, and
 * the draws do not depend on nreal, chunking or real0.  B (Bt = B^T, row-major [n_psr][n_psr]) is the ORF factor,
 * Gamma = B B^T; Bt == NULL is Gamma = I (uncorrelated).  The mixing sums over b in index order, unfused.
 *   stage 1 (draw)  scratch <- c [nreal][n_psr][2K]; params (optional) <- [nreal][2] (log10_A, gamma) or [nreal][K]
 *                   (log10_rho_k).
 *   stage 2 (add)   rows[r][i] += sum_j c[r][slot_psr[i]][j] F_j(slot_t[i]) for every slot with slot_psr[i] >= 0,
 *                   the argument rounded as (2 pi t) f_k; alignment slots are never touched.
 * ptar_common_population runs both (stage 0 of ptar_common_population_stage); with rows == NULL it only draws.
 * scratch_len >= nreal * n_psr * 2K.  Outputs are bit-identical whatever nreal, chunking or real0. */
#define PTAR_CPOP_MAX_K    32         /* Fourier bins                                                          */
#define PTAR_CPOP_MAX_PSR  2048       /* pulsars (the draw kernel holds one bin's 2 n_psr normals in shared)   */
#define PTAR_CPOP_HYPER    0x10000    /* first counter element of the hyperparameter pairs                     */
#define PTAR_CPOP_POWERLAW 0
#define PTAR_CPOP_FREE     1
typedef struct {
  int32_t n_psr;                       /* 1 .. PTAR_CPOP_MAX_PSR                                               */
  int32_t K;                           /* 1 .. PTAR_CPOP_MAX_K                                                 */
  int32_t spectrum;                    /* PTAR_CPOP_POWERLAW / PTAR_CPOP_FREE                                  */
  int32_t kind[2];                     /* PTAR_CWPOP_FIXED / _UNIFORM of (log10_A, gamma); free: kind[0]       */
  int32_t reserved;
  double lo[2];
  double width[2];
  double pl_den;                       /* 12 pi^2 Tspan (power law)                                            */
  double pl_y3;                        /* yr^3 [s^3] (power law)                                               */
  const double* pl_x;                  /* [K] f_k yr (power law)                                               */
  const double* freqs;                 /* [K] f_k [Hz]                                                         */
  const double* Bt;                    /* [n_psr][n_psr] B^T of Gamma = B B^T, or NULL (Gamma = I)             */
  const double* slot_t;                /* [ld] absolute TDB time [s] per slot of the packed axis               */
  const int32_t* slot_psr;             /* [ld] pulsar of each slot, -1 for alignment slots (never written)     */
} ptar_cpop_model;

int ptar_common_population(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed,
                           const ptar_cpop_model* m, double* scratch, int64_t scratch_len, double* params, void* stream);
int ptar_common_population_stage(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed,
                                 const ptar_cpop_model* m, double* scratch, int64_t scratch_len, double* params,
                                 int stage, void* stream);

/* Per-realization transient populations (csrc/ptar_tpop.cuh): burst-with-memory (family PTAR_TPOP_BWM) or sine-Gaussian
 * bursts (PTAR_TPOP_BURST).  Every realization r of [real0, real0 + nreal) gets n_src sources; parameter j is drawn as in
 * ptar_cw_population (kind PTAR_CWPOP_FIXED: lo, _UNIFORM: lo + width u, _ACOS: acos(lo + width u), each operation of
 * the affine map rounded once), u the 53-bit uniforms (a >> 5) 2^26 + (b >> 6) times 2^-53 of the Philox4x32-10 words
 * (a, b) = (w.x, w.y) for even j and (w.z, w.w) for odd j of the counter
 *   (source * 16 + j / 2, PTAR_K_BWMPOP or PTAR_K_BURSTPOP, r & 0xffffffff, r >> 32).
 * All PTAR_TPOP_NPAR parameters are drawn whether or not the family uses them; the other streams (kinds 1-8) are
 * untouched, so every realization's noise and the other populations' draws are what they are without this one, and the
 * two families never share a uniform.  With t0 = t0_mjd 86400 (rounded once), t = slot_t (MJD 86400), the pattern
 * (F+, Fx) of add_cgw's formula with 1 + Omega.p = (m.p^2 + n.p^2) / (1 - Omega.p), and (0, 0) where that is below
 * PTAR_CWPOP_POLE_TOL (or NaN):
 *   BWM    h = 10^log10_amp, pol = bwm_pol: delay_a(t) = (pol_a h) (t - t0) for t >= t0, else 0, pol_a = cos 2pol F+ +
 *          sin 2pol Fx (add_gw_memory's Earth-term ramp, deterministic.py:822-884);
 *   BURST  A = 10^log10_amp, f0 = 10^log10_f0, tau = Q / (2 pi f0), c = cos 2pol, s = sin 2pol (pol = psi):
 *          delay_a(t) = g (alpha_a cos Phi + beta_a sin Phi), g = exp(-(t - t0)^2 / tau^2), Phi = 2 pi f0 (t - t0) + phase0,
 *          alpha_a = -A (F+ c + Fx s), beta_a = eps A (F+ s - Fx c): add_burst (deterministic.py:718-793, tref = 0) of
 *          h+ = A g cos Phi, hx = eps A g sin Phi.  Not truncated: a term is skipped only where g is 0.
 *   stage 1 (draw)  scratch <- per-(r, s) records [nreal][n_src][4] = {t0 [s], 2 pi f0, 1 / tau, phase0} (BWM: {t0, 0,
 *                   0, 0}) and per-(r, s, p) coefficients [nreal][n_src][n_psr][2] = {pol_a h, 0} or {alpha_a, beta_a};
 *                   params (optional) <- [nreal][n_src][PTAR_TPOP_TABLE]:
 *                     BWM   {t0_mjd, log10_strain, strain, gwtheta, gwphi, bwm_pol, 0 ...}
 *                     BURST {t0_mjd, log10_amp, amp, log10_f0, f0, Q, tau, gwtheta, gwphi, psi, phase0, eps, a1, a2, a3,
 *                            a4}, (a1 .. a4) the burst search's amplitudes of this source (its psi = 0, x = 2 pi f0 (t - t0)):
 *                            a1 = A (c cos phase0 - eps s sin phase0), a2 = A (-c sin phase0 - eps s cos phase0),
 *                            a3 = A (s cos phase0 + eps c sin phase0), a4 = A (-s sin phase0 + eps c cos phase0).
 *   stage 2 (add)   rows[r][i] += sum_s delay of source s at slot i for every slot with slot_psr[i] >= 0 whose sum has
 *                   at least one non-zero term (a slot before every t0 of its realization, or where every g is 0, is
 *                   not read or written); alignment slots are never touched.
 * ptar_transient_population runs both (stage 0 of ptar_transient_population_stage); with rows == NULL it only draws.
 * scratch_len >= nreal * n_src * (4 + 2 n_psr).  Outputs are bit-identical whatever nreal, chunking or real0. */
#define PTAR_TPOP_BWM      0
#define PTAR_TPOP_BURST    1
#define PTAR_TPOP_MAX_SRC  64    /* sources per realization                                               */
#define PTAR_TPOP_NPAR     10    /* drawn parameters per source (5 counter pairs)                          */
#define PTAR_TPOP_TABLE    16    /* doubles per (r, s) row of the parameter table                          */
#define PTAR_TPOP_T0         0   /* parameter indices: the order of the counter's parameter pairs          */
#define PTAR_TPOP_LOG10_AMP  1   /* log10_strain (BWM) / log10_amp (burst)                                 */
#define PTAR_TPOP_GWTHETA    2
#define PTAR_TPOP_GWPHI      3
#define PTAR_TPOP_POL        4   /* bwm_pol (BWM) / psi (burst)                                            */
#define PTAR_TPOP_LOG10_F0   5   /* burst only, as are the rest                                            */
#define PTAR_TPOP_Q          6
#define PTAR_TPOP_PHASE0     7
#define PTAR_TPOP_EPS        8   /* index 9: unused                                                        */
typedef struct {
  int32_t family;                      /* PTAR_TPOP_BWM / PTAR_TPOP_BURST                                      */
  int32_t n_psr;                       /* >= 1                                                                 */
  int32_t n_src;                       /* 1 .. PTAR_TPOP_MAX_SRC                                               */
  int32_t kind[PTAR_TPOP_NPAR];        /* PTAR_CWPOP_FIXED / _UNIFORM / _ACOS                                  */
  int32_t reserved;
  double lo[PTAR_TPOP_NPAR];
  double width[PTAR_TPOP_NPAR];
  const double* phat;                  /* [n_psr][3] pulsar unit vectors                                       */
  const double* slot_t;                /* [ld] TOA (MJD 86400) [s] per slot of the packed axis                 */
  const int32_t* slot_psr;             /* [ld] pulsar of each slot, -1 for alignment slots (never written)     */
} ptar_tpop_model;

int ptar_transient_population(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed,
                              const ptar_tpop_model* m, double* scratch, int64_t scratch_len, double* params, void* stream);
int ptar_transient_population_stage(double* rows, int64_t ld, int32_t nreal, int64_t real0, uint64_t seed,
                                    const ptar_tpop_model* m, double* scratch, int64_t scratch_len, double* params,
                                    int stage, void* stream);

/* End-to-end job: GWB mix + synth + generate for realizations [real0, real0+nreal), then
 * (ptar_run_job_to_host) copy the residuals to pinned host memory, chunk by chunk, with the
 * copy of chunk c overlapping the generation of chunk c+1 on a second stream. */
typedef struct {
  ptar_gen_params gen;      /* gen.G / gen.out / gen.nreal / gen.real0 are set per chunk  */
  const double* M;          /* [n_psr][n_psr] lower Cholesky factor of the ORF            */
  const double* A;          /* [npts][lda] GWB synthesis matrix                           */
  int64_t lda;
  int32_t Jg;               /* columns of A                                               */
  int32_t lower_tri;
  const int32_t* tile_list; /* [n_syn_tiles][4], see ptar_gwb_synth                       */
  const int32_t* knots;     /* [gen.g_ld]                                                 */
  int32_t n_syn_tiles;
  int32_t reserved;
  double* Zm;               /* scratch [n_psr][chunk][Jg]                                 */
  double* Gbuf;             /* scratch [gen.g_ld][gen.g_ldr]                              */
  const double* gwb_zin;    /* parity mode: [nreal][n_psr][Jg] or NULL                    */
  /* int8 tensor-core synthesis (throughput mode only; all NULL / 0 selects the fp64 DMMA kernel) */
  const int8_t* AS;         /* digit slices of the gathered rows of A, tile_list_i8 order */
  const double* colscale;   /* [gen.g_ld]                                                 */
  int8_t* ZS;               /* scratch: digit slices of Zm, PTAR_I8_SLICES*n_psr*rcap*Jpad bytes */
  const double* zscale;     /* [n_psr]                                                    */
  const double* zinv;       /* [n_psr] 2^48 / zscale                                      */
  const int32_t* tile_list_i8; /* [n_syn_tiles_i8][4]: 32-column blocks, pulsar-major     */
  int64_t rcap;             /* row capacity of ZS (multiple of 128, >= chunk)             */
  int32_t Jpad;             /* multiple of 32, >= Jg                                      */
  int32_t n_syn_tiles_i8;
} ptar_job;

/* Peer delivery over NVLink without a collective library (multi-GPU row of SURVEY.md 8e; the reference has no
 * distributed code): a rank exports its result buffer (CUDA IPC), every other rank maps it into its own address space
 * and pushes its realization chunks straight into it with the copy engines, overlapped with generation.
 * ptar_peer_export: handle_host[64] <- IPC handle of the allocation that contains dev_ptr, *offset <- dev_ptr - base.
 * ptar_peer_open:   maps an exported allocation into the current device's context (lazy peer access); *base_out is the
 *                   mapped base (add the exporter's offset); ptar_peer_close unmaps it.
 * ptar_peer_copy:   asynchronous device-to-device copy (UVA) between local and mapped peer memory on `stream`. */
int ptar_peer_export(const void* dev_ptr, void* handle_host, int64_t* offset);
int ptar_peer_open(const void* handle_host, void** base_out);
int ptar_peer_close(void* base);
int ptar_peer_copy(void* dst, const void* src, int64_t bytes, void* stream);

int ptar_run_job(const ptar_job* job, int64_t real0, int32_t nreal, double* out, void* stream);
int ptar_run_job_to_host(const ptar_job* job, int64_t real0, int64_t nreal, int32_t chunk,
                         double* out_host, double* dev_buf0, double* dev_buf1, void* stream0, void* stream1);

/* The same two with the timing-model fit applied to every chunk right after ptar_generate (post-fit residuals);
 * tm == NULL runs exactly ptar_run_job / ptar_run_job_to_host.  scratch: >= tm->n_tiles * chunk * tm->kmax doubles
 * (chunk = nreal for ptar_run_job_tm). */
int ptar_run_job_tm(const ptar_job* job, const ptar_timing_model* tm, double* scratch, int64_t scratch_len, int64_t real0,
                    int32_t nreal, double* out, void* stream);
int ptar_run_job_to_host_tm(const ptar_job* job, const ptar_timing_model* tm, double* scratch, int64_t scratch_len,
                            int64_t real0, int64_t nreal, int32_t chunk, double* out_host, double* dev_buf0,
                            double* dev_buf1, void* stream0, void* stream1);

/* ptar_run_job_to_host_tm with chromatic noise (ptar_generate_chrom); tm and cm may each be NULL, and with cm == NULL this
 * is exactly ptar_run_job_to_host_tm.  A parity-mode cm->zchr advances with the chunks like gen.zrn. */
int ptar_run_job_to_host_chrom(const ptar_job* job, const ptar_timing_model* tm, const ptar_chrom_model* cm, double* scratch,
                               int64_t scratch_len, int64_t real0, int64_t nreal, int32_t chunk, double* out_host,
                               double* dev_buf0, double* dev_buf1, void* stream0, void* stream1);

#ifdef __cplusplus
}
#endif
#endif /* PTAR_H */

"""ctypes binding of ``libptar_b200.so`` (C ABI declared in ``include/ptar.h``).

The shared library is built in-tree by ``__graft_entry__.build()`` (plain ``nvcc``; no torch
in the ABI).  There is no CPU fallback: if the library is missing, or there is no CUDA
device, the product raises instead of computing anywhere else.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# PTAR_B200_LIB points at an alternative build of the same library (A/B measurements of kernel variants)
LIB_PATH = os.environ.get("PTAR_B200_LIB") or os.path.join(_HERE, "csrc", "libptar_b200.so")

TILE_TOAS = 1024
TILE_EPOCHS = 64
TOA_ALIGN = 4
I8_SLICES, I8_BM, I8_BN, I8_BK = 6, 128, 48, 32   # int8 wgmma GWB synthesis: ZS r-block, knots per tile, k-chunk (csrc/ptar_gwb_i8.cuh)
MIX_I8_MAX_PSR = 72                                # pulsars of ptar_gwb_mix_i8, the fused int8 mix (8 * MX_MAXNT, ptar_gwb.cuh)
MIX_MAX_PSR = 112                                  # pulsars of ptar_gwb_mix: M and the draws of one item in 227 KB of shared memory
SMEM_MAX = 227 * 1024                              # dynamic shared memory per block (sm_90)
EPK_RB = 32                                        # realizations per CTA of the two-kernel schedule's epoch kernel


def gen_smem_bytes(J, rc):
    """Shared memory of the fused generator / its epoch stage at rc realizations (gen_smem_bytes, ptar_generate.cuh)."""
    return 16 + 8 * max(J * TILE_EPOCHS + 3 * J * rc, TILE_EPOCHS * (3 * rc + 2))


def epoch_smem_bytes(J):
    """Shared memory of the standalone epoch kernel (epoch_smem_bytes, ptar_generate.cuh)."""
    return 16 + 8 * (max(J * TILE_EPOCHS + 3 * J * EPK_RB, 3 * 24 * 64) + TILE_EPOCHS * EPK_RB * 2)


def gen_chrom_smem_bytes(Jo, rc, n_slot, split_epoch=False):
    """Shared memory of the chromatic generator's epoch stage (gen_chrom_smem_bytes / epoch_smem_bytes of
    ptar_generate.cuh) for the widest basis Jo and n_slot chromatic slots; the larger of the schedule's kernels."""
    if split_epoch and rc != 32:
        return max(epoch_smem_bytes(Jo), 16 + 8 * TILE_EPOCHS * (3 * 16 * (1 + n_slot) + 2))
    rc = rc or 16
    return 16 + 8 * (max(Jo * TILE_EPOCHS + 3 * Jo * rc, TILE_EPOCHS * (3 * rc + 2)) + TILE_EPOCHS * (3 * rc * n_slot + 2))


def max_red_columns(rc=16, split_epoch=False):
    """The largest (even) red-noise basis width J whose epoch stage fits shared memory in the given schedule: 258 fused at
    rc = 16, 180 at rc = 32 (fused or two-kernel), 154 in the two-kernel schedule's epoch kernel (rc = 16)."""
    need = epoch_smem_bytes if (split_epoch and rc != 32) else (lambda J: gen_smem_bytes(J, rc or 16))
    J = 2
    while need(J + 2) <= SMEM_MAX:
        J += 2
    return J

F_WHITE, F_ECORR, F_RED, F_GWB, F_DET, F_WHITE1 = 1, 2, 4, 8, 16, 32
TM_KMAX = 32                                       # timing-model columns per pulsar (PTAR_TM_KMAX)
K_WHITE1, K_WHITE2, K_ECORR, K_RED, K_GWB, K_CHROM, K_CWPOP, K_CPOP = 1, 2, 3, 4, 5, 6, 7, 8
K_BWMPOP, K_BURSTPOP = 9, 10
CHROM_SLOTS = 2                                    # chromatic slots of ptar_generate_chrom (PTAR_CHROM_SLOTS)

EXPORTS = ("ptar_version", "ptar_last_error", "ptar_cholesky_lower", "ptar_fourier_basis", "ptar_cgw_delay", "ptar_cw_catalog", "ptar_burst_delay", "ptar_memory_delay",
           "ptar_gwb_mix", "ptar_gwb_synth", "ptar_gwb_mix_i8", "ptar_gwb_slice_i8", "ptar_gwb_synth_i8", "ptar_debug_i8_timestamps", "ptar_generate", "ptar_generate_stage", "ptar_philox_normals", "ptar_peer_export", "ptar_peer_open", "ptar_peer_close", "ptar_peer_copy", "ptar_run_job",
           "ptar_run_job_to_host", "ptar_timing_project", "ptar_timing_project_stage",
           "ptar_run_job_tm", "ptar_run_job_to_host_tm", "ptar_os_project", "ptar_os_project_stage", "ptar_os_pairs",
           "ptar_os_null", "ptar_os_null_stage", "ptar_os_aniso", "ptar_os_aniso_stage", "ptar_os_pf", "ptar_fp_project", "ptar_fp_reduce",
           "ptar_fp_reduce_fap", "ptar_fe_sky", "ptar_fe_combine", "ptar_curn_grid", "ptar_curn_reduce",
           "ptar_hd_grid", "ptar_rn_grid", "ptar_bwm_sky", "ptar_bwm_combine", "ptar_fs_grid",
           "ptar_burst_ninv", "ptar_burst_project", "ptar_burst_reduce", "ptar_fs_y2", "ptar_fs_refit",
           "ptar_generate_chrom", "ptar_generate_stage_chrom", "ptar_run_job_to_host_chrom",
           "ptar_cw_population", "ptar_cw_population_stage", "ptar_common_population", "ptar_common_population_stage",
           "ptar_transient_population", "ptar_transient_population_stage")
OS_MAX_NC, OS_MAX_ORF, OS_MAX_PSR = 32, 4, 256     # optimal statistic: GW-basis columns, templates, pulsars (ptar.h)
OS_MAX_NULL = 65536                                # null columns of ptar_os_null (PTAR_OS_MAX_NULL)
OS_NULL_PHASE_SHIFT, OS_NULL_SKY_SCRAMBLE = 1, 2
OS_NULL_BK, OS_NULL_BN = 32, 64                    # kd / column padding of ptar_os_null_model (csrc/ptar_os_null.cuh)
OS_ANISO_MAX_LM, OS_ANISO_MAX_SKY = 64, 12288      # anisotropy: harmonic coefficients (lmax <= 7), radiometer pixels (ptar.h)
FP_MAX_FREQ = 256                                  # search frequencies of the Fp-statistic (PTAR_FP_MAX_FREQ)
FE_MAX_PSR, FE_MAX_SKY = 128, 12288                # Fe-statistic: pulsars (shared-memory tile), sky points (ptar.h)
FE_SB = 32                                         # sky points per stage of ptar_fe_sky (csrc/ptar_fe.cuh)
CURN_MAX_NA, CURN_MAX_NG = 256, 256                # CURN likelihood grid: log10 A and gamma points (ptar.h)
HD_MAX_N, HD_JB = 4096, 32                         # HD likelihood: n_psr 2K eigen-rows, rows per block (ptar.h)
RN_MAX_NC = 64                                     # red-noise likelihood: basis columns of ptar_rn_grid / ptar_os_project
BWM_MAX_EPOCH = 512                                # burst-with-memory search: burst epochs (PTAR_BWM_MAX_EPOCH)
FS_MAX_PSR, FS_MAX_BIN, FS_JB = 256, 32, 32       # free-spectrum likelihood: pulsars, bins, eigen-rows per block (ptar.h)
FS_MAX_TEMPLATE = 65536                            # spectral refit: templates of one model (PTAR_FS_MAX_TEMPLATE)
BURST_MAX_TEMPLATE, BURST_GROUP, BURST_TB = 4096, 256, 16   # burst search: templates, per group, per CTA (ptar.h)
CWPOP_MAX_SRC, CWPOP_NPAR, CWPOP_TABLE = 64, 8, 16  # CW populations: sources per realization, drawn parameters, table row
CWPOP_SRC, CWPOP_PSR = 16, 8                       # doubles per (r, s) and per (r, s, p) record of the scratch (ptar_cwpop.cuh)
CWPOP_FIXED, CWPOP_UNIFORM, CWPOP_ACOS = 0, 1, 2   # parameter kinds of ptar_cwpop_model
CPOP_MAX_K, CPOP_MAX_PSR, CPOP_HYPER = 32, 2048, 0x10000   # common-process populations: bins, pulsars, hyper counters
CPOP_POWERLAW, CPOP_FREE = 0, 1                    # spectra of ptar_cpop_model
TPOP_BWM, TPOP_BURST = 0, 1                        # families of ptar_tpop_model
TPOP_MAX_SRC, TPOP_NPAR, TPOP_TABLE = 64, 10, 16   # transient populations: sources per realization, parameters, table row
TPOP_REC, TPOP_COEF = 4, 2                         # doubles per (r, s) and per (r, s, p) record of the scratch (ptar_tpop.cuh)
BWM_LINV = 6                                       # packed L2^-1 doubles per (epoch pair, sky point) (csrc/ptar_bwm.cuh)


class Tile(C.Structure):
    _fields_ = [("toa_start", C.c_int32), ("n_toa", C.c_int32), ("toa_local0", C.c_int32), ("ep_start", C.c_int32),
                ("n_ep", C.c_int32), ("psr", C.c_int32), ("nd", C.c_int32), ("reserved", C.c_int32)]


class GenParams(C.Structure):
    _fields_ = [
        ("n_psr", C.c_int32), ("n_tiles", C.c_int32), ("J", C.c_int32), ("npts", C.c_int32),
        ("flags", C.c_uint32), ("rn_convention", C.c_int32),
        ("tiles", C.c_void_p),
        ("w1", C.c_void_p), ("w2", C.c_void_p), ("dtau", C.c_void_p), ("eloc", C.c_void_p), ("det", C.c_void_p),
        ("ep_ecorr", C.c_void_p), ("ep_bucket", C.c_void_p), ("ep_gidx", C.c_void_p), ("ep_gw", C.c_void_p),
        ("ep_ginv", C.c_void_p), ("psr_bucket_off", C.c_void_p), ("Ftile", C.c_void_p),
        ("rn_scale", C.c_void_p), ("rn_omega", C.c_void_p),
        ("G", C.c_void_p), ("g_ld", C.c_int64), ("g_ldr", C.c_int64),
        ("z1", C.c_void_p), ("z2", C.c_void_p), ("zb", C.c_void_p), ("zrn", C.c_void_p),
        ("n_bucket_total", C.c_int64),
        ("seed", C.c_uint64), ("real0", C.c_int64),
        ("out", C.c_void_p), ("ld_out", C.c_int64), ("nreal", C.c_int32), ("rc", C.c_int32),
        ("Cbuf", C.c_void_p), ("cbuf_len", C.c_int64), ("c_rows", C.c_int64),
    ]


class ChromModel(C.Structure):
    _fields_ = [("n_slot", C.c_int32), ("J", C.c_int32 * CHROM_SLOTS), ("reserved", C.c_int32)] + [
        (k, C.c_void_p * CHROM_SLOTS) for k in ("Ftile", "scale", "omega", "weight", "on")] + [("zchr", C.c_void_p)]


class Job(C.Structure):
    _fields_ = [("gen", GenParams), ("M", C.c_void_p), ("A", C.c_void_p), ("lda", C.c_int64), ("Jg", C.c_int32),
                ("lower_tri", C.c_int32), ("tile_list", C.c_void_p), ("knots", C.c_void_p), ("n_syn_tiles", C.c_int32),
                ("reserved", C.c_int32), ("Zm", C.c_void_p), ("Gbuf", C.c_void_p), ("gwb_zin", C.c_void_p),
                ("AS", C.c_void_p), ("colscale", C.c_void_p), ("ZS", C.c_void_p), ("zscale", C.c_void_p), ("zinv", C.c_void_p),
                ("tile_list_i8", C.c_void_p), ("rcap", C.c_int64), ("Jpad", C.c_int32), ("n_syn_tiles_i8", C.c_int32)]
    chrom = None   # the engine's ChromModel of the job (not part of the C struct): None without chromatic noise


class TimingModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("n_tiles", C.c_int32), ("tiles", C.c_void_p), ("seg_off", C.c_void_p),
                ("seg_len", C.c_void_p), ("k", C.c_void_p), ("q_off", C.c_void_p), ("tile0", C.c_void_p),
                ("n_tile", C.c_void_p), ("Q", C.c_void_p), ("sqrtw", C.c_void_p), ("kmax", C.c_int32),
                ("reserved", C.c_int32)]


class OsModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("n_tiles", C.c_int32), ("tiles", C.c_void_p), ("tile0", C.c_void_p),
                ("n_tile", C.c_void_p), ("C", C.c_void_p), ("nc", C.c_int32), ("ncp", C.c_int32), ("sqrt_phi", C.c_void_p),
                ("n_pairs", C.c_int32), ("n_orf", C.c_int32), ("pairs", C.c_void_p), ("t_ab", C.c_void_p),
                ("orf", C.c_void_p), ("dnorm", C.c_void_p), ("dsqrt", C.c_void_p), ("finv", C.c_void_p)]


class OsNullModel(C.Structure):
    _fields_ = [("method", C.c_int32), ("n_col", C.c_int32), ("n_colp", C.c_int32), ("reserved", C.c_int32),
                ("kd", C.c_int64), ("kdp", C.c_int64), ("V", C.c_void_p), ("dsqrt", C.c_void_p)]


class OsAnisoModel(C.Structure):
    _fields_ = [("n_lm", C.c_int32), ("n_z", C.c_int32), ("n_sky", C.c_int32), ("n_col", C.c_int32),
                ("n_colp", C.c_int32), ("reserved", C.c_int32), ("kd", C.c_int64), ("kdp", C.c_int64), ("V", C.c_void_p),
                ("dsqrt", C.c_void_p)]


class OsPfModel(C.Structure):
    _fields_ = [("t", C.c_void_p), ("dnorm", C.c_void_p), ("dsqrt", C.c_void_p), ("finv", C.c_void_p)]


class FpModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("n_freq", C.c_int32), ("n_cb", C.c_int32), ("reserved", C.c_int32),
                ("ld", C.c_int64), ("Ct", C.c_void_p), ("psr_order", C.c_void_p), ("seg_off", C.c_void_p),
                ("seg_len", C.c_void_p)]


class FeModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("n_freq", C.c_int32), ("n_sky", C.c_int32), ("n_sb", C.c_int32),
                ("kp", C.c_int32), ("reserved", C.c_int32), ("Lf", C.c_void_p), ("ant", C.c_void_p), ("linv", C.c_void_p)]


class BwmModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("n_t0", C.c_int32), ("n_sky", C.c_int32), ("n_sb", C.c_int32),
                ("kp", C.c_int32), ("reserved", C.c_int32), ("sqm", C.c_void_p), ("seen", C.c_void_p), ("ant", C.c_void_p),
                ("antenna", C.c_void_p), ("linv", C.c_void_p)]


class BurstModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("n_tmpl", C.c_int32), ("n_zc", C.c_int32), ("n_run", C.c_int32),
                ("n_sky", C.c_int32), ("n_sb", C.c_int32)] + [
        (k, C.c_void_p) for k in ("t", "dinv", "run_start", "run_len", "run_coef", "toa_run", "tmpl", "win", "blk", "H",
                                  "wl", "Lf", "linv", "antenna", "seen", "psr_order", "seg_off")]


class CurnModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("nc", C.c_int32), ("ncp", C.c_int32), ("n_gamma", C.c_int32),
                ("n_amp", C.c_int32), ("reserved", C.c_int32), ("V", C.c_void_p), ("lam", C.c_void_p), ("a2", C.c_void_p),
                ("ldet", C.c_void_p), ("log10_A", C.c_void_p), ("wg", C.c_void_p), ("wx", C.c_void_p),
                ("prior", C.c_void_p), ("ul", C.c_double)]


class HdModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("nc", C.c_int32), ("ncp", C.c_int32), ("n_gamma", C.c_int32),
                ("n_amp", C.c_int32), ("n", C.c_int32), ("np", C.c_int32), ("reserved", C.c_int32), ("V", C.c_void_p),
                ("lam", C.c_void_p), ("a2", C.c_void_p), ("ldet", C.c_void_p)]


class RnModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("nc", C.c_int32), ("ncp", C.c_int32), ("n_gamma", C.c_int32),
                ("n_amp", C.c_int32), ("reserved", C.c_int32), ("V", C.c_void_p), ("lam", C.c_void_p), ("a2", C.c_void_p),
                ("ldet", C.c_void_p)]


class FsModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("ncp", C.c_int32), ("n_bin", C.c_int32), ("n_amp", C.c_int32),
                ("n2p", C.c_int32), ("np", C.c_int32), ("V", C.c_void_p), ("lam", C.c_void_p), ("a2", C.c_void_p),
                ("ldet", C.c_void_p)]


class FsRefitModel(C.Structure):
    _fields_ = [("n_bin", C.c_int32), ("np", C.c_int32), ("n_tmpl", C.c_int32), ("reserved", C.c_int32),
                ("lam", C.c_void_p), ("rho2", C.c_void_p), ("ldet", C.c_void_p)]


class CwPopModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("n_src", C.c_int32), ("mode", C.c_int32), ("psr_term", C.c_int32),
                ("pphase", C.c_int32), ("kind", C.c_int32 * CWPOP_NPAR), ("reserved", C.c_int32),
                ("lo", C.c_double * CWPOP_NPAR), ("width", C.c_double * CWPOP_NPAR), ("phat", C.c_void_p),
                ("pdist", C.c_void_p), ("slot_t", C.c_void_p), ("slot_psr", C.c_void_p)]


class CpopModel(C.Structure):
    _fields_ = [("n_psr", C.c_int32), ("K", C.c_int32), ("spectrum", C.c_int32), ("kind", C.c_int32 * 2),
                ("reserved", C.c_int32), ("lo", C.c_double * 2), ("width", C.c_double * 2), ("pl_den", C.c_double),
                ("pl_y3", C.c_double), ("pl_x", C.c_void_p), ("freqs", C.c_void_p), ("Bt", C.c_void_p),
                ("slot_t", C.c_void_p), ("slot_psr", C.c_void_p)]


class TpopModel(C.Structure):
    _fields_ = [("family", C.c_int32), ("n_psr", C.c_int32), ("n_src", C.c_int32), ("kind", C.c_int32 * TPOP_NPAR),
                ("reserved", C.c_int32), ("lo", C.c_double * TPOP_NPAR), ("width", C.c_double * TPOP_NPAR),
                ("phat", C.c_void_p), ("slot_t", C.c_void_p), ("slot_psr", C.c_void_p)]


_lib = None


class PtarError(RuntimeError):
    pass


def lib():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise PtarError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                        "(nvcc -gencode arch=compute_90a,code=sm_90a).  There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, u64 = C.c_void_p, C.c_int, C.c_int64, C.c_uint64
    L.ptar_version.restype = C.c_int
    L.ptar_last_error.restype = C.c_char_p
    L.ptar_cholesky_lower.argtypes = [vp, vp, i32, i32, vp, vp]
    L.ptar_fourier_basis.argtypes = [vp, vp, i64, vp, vp, vp, vp, i32, i32, i64, vp]
    L.ptar_cgw_delay.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i64, vp]
    L.ptar_cw_catalog.argtypes = [vp, vp, i64, C.POINTER(C.c_double), vp, i64, C.c_double, C.c_double, i32, i32, i32, i32, vp, vp, i32, vp]
    L.ptar_burst_delay.argtypes = [vp, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double, i32, i64, vp]
    L.ptar_memory_delay.argtypes = [vp, vp, C.c_double, C.c_double, i32, i64, vp]
    L.ptar_gwb_mix.argtypes = [vp, vp, vp, i32, i32, i64, u64, i64, vp]
    L.ptar_gwb_synth.argtypes = [vp, i64, i64, vp, i64, vp, i32, i64, vp, i32, vp, i32, vp]
    L.ptar_gwb_mix_i8.argtypes = [vp, vp, vp, i32, i32, i32, i64, i64, u64, i64, vp]
    L.ptar_gwb_slice_i8.argtypes = [vp, vp, vp, i32, i32, i32, i64, i64, vp]
    L.ptar_gwb_synth_i8.argtypes = [vp, i64, i64, vp, vp, vp, vp, i32, i32, i32, i64, i64, vp, i32, vp]
    L.ptar_debug_i8_timestamps.argtypes = [vp]
    L.ptar_generate.argtypes = [C.POINTER(GenParams), vp]
    L.ptar_generate_stage.argtypes = [C.POINTER(GenParams), i32, vp]
    L.ptar_philox_normals.argtypes = [vp, i32, i32, i64, i64, i64, u64, vp]
    L.ptar_peer_export.argtypes = [vp, vp, C.POINTER(C.c_int64)]
    L.ptar_peer_open.argtypes = [vp, C.POINTER(C.c_void_p)]
    L.ptar_peer_close.argtypes = [vp]
    L.ptar_peer_copy.argtypes = [vp, vp, i64, vp]
    L.ptar_run_job.argtypes = [C.POINTER(Job), i64, C.c_int32, vp, vp]
    L.ptar_run_job_to_host.argtypes = [C.POINTER(Job), i64, i64, C.c_int32, vp, vp, vp, vp, vp]
    L.ptar_timing_project.argtypes = [vp, i64, C.c_int32, vp, vp, i64, vp]       # tm: address of a TimingModel
    L.ptar_timing_project_stage.argtypes = [vp, i64, C.c_int32, vp, vp, i64, i32, vp]
    L.ptar_run_job_tm.argtypes = [C.POINTER(Job), vp, vp, i64, i64, C.c_int32, vp, vp]
    L.ptar_run_job_to_host_tm.argtypes = [C.POINTER(Job), vp, vp, i64, i64, i64, C.c_int32, vp, vp, vp, vp, vp]
    L.ptar_os_project.argtypes = [vp, i64, C.c_int32, vp, vp, i64, vp, vp]            # os: address of an OsModel
    L.ptar_os_project_stage.argtypes = [vp, i64, C.c_int32, vp, vp, i64, vp, i32, vp]
    L.ptar_os_pairs.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp, vp]
    L.ptar_os_null.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp, vp, vp]                # null: address of an OsNullModel
    L.ptar_os_null_stage.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp, vp, i32, vp]
    L.ptar_os_aniso.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]   # model: an OsAnisoModel
    L.ptar_os_aniso_stage.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp]
    L.ptar_os_pf.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp, vp, vp]                  # pf: address of an OsPfModel
    L.ptar_fp_project.argtypes = [vp, i64, C.c_int32, vp, vp, vp]                        # fp: address of an FpModel
    L.ptar_fp_reduce.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp]
    L.ptar_fp_reduce_fap.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp, vp]
    L.ptar_fe_sky.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp]                         # fe: address of an FeModel
    L.ptar_fe_combine.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, vp]
    L.ptar_bwm_sky.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp]                        # bw: address of a BwmModel
    L.ptar_bwm_combine.argtypes = [vp, vp, vp, C.c_int32, vp] + [vp] * 10 + [vp]
    L.ptar_burst_ninv.argtypes = [vp, i64, C.c_int32, vp, vp, vp]                     # bm: address of a BurstModel
    L.ptar_burst_project.argtypes = [vp, i64, C.c_int32, vp, vp, C.c_int32, vp, vp]
    L.ptar_burst_reduce.argtypes = [vp, vp, vp, C.c_int32, vp] + [vp] * 12 + [vp]
    L.ptar_curn_grid.argtypes = [vp, C.c_int32, vp, vp, vp]                           # cm: address of a CurnModel
    L.ptar_curn_reduce.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.ptar_hd_grid.argtypes = [vp, C.c_int32, vp, vp, vp]                             # hm: address of an HdModel
    L.ptar_rn_grid.argtypes = [vp, C.c_int32, vp, vp, vp]                             # rm: address of an RnModel
    L.ptar_fs_grid.argtypes = [vp, C.c_int32, vp, vp, vp]                             # fm: address of an FsModel
    L.ptar_fs_y2.argtypes = [vp, C.c_int32, vp, vp, vp]
    L.ptar_fs_refit.argtypes = [vp, C.c_int32, vp, vp, vp]                            # rm: address of an FsRefitModel
    L.ptar_generate_chrom.argtypes = [C.POINTER(GenParams), C.POINTER(ChromModel), vp]
    L.ptar_generate_stage_chrom.argtypes = [C.POINTER(GenParams), C.POINTER(ChromModel), i32, vp]
    L.ptar_run_job_to_host_chrom.argtypes = [C.POINTER(Job), vp, C.POINTER(ChromModel), vp, i64, i64, i64, C.c_int32, vp, vp,
                                             vp, vp, vp]
    L.ptar_cw_population.argtypes = [vp, i64, C.c_int32, i64, u64, vp, vp, i64, vp, vp]   # m: address of a CwPopModel
    L.ptar_cw_population_stage.argtypes = [vp, i64, C.c_int32, i64, u64, vp, vp, i64, vp, i32, vp]
    L.ptar_common_population.argtypes = [vp, i64, C.c_int32, i64, u64, vp, vp, i64, vp, vp]   # m: address of a CpopModel
    L.ptar_common_population_stage.argtypes = [vp, i64, C.c_int32, i64, u64, vp, vp, i64, vp, i32, vp]
    L.ptar_transient_population.argtypes = [vp, i64, C.c_int32, i64, u64, vp, vp, i64, vp, vp]   # m: address of a TpopModel
    L.ptar_transient_population_stage.argtypes = [vp, i64, C.c_int32, i64, u64, vp, vp, i64, vp, i32, vp]
    for name in EXPORTS:
        if name not in ("ptar_version", "ptar_last_error"):
            getattr(L, name).restype = C.c_int
    _lib = L
    return L


def check(rc: int, what: str = "ptar"):
    if rc != 0:
        raise PtarError(f"{what} failed ({rc}): {lib().ptar_last_error().decode()}")


def require_cuda():
    """The product path runs on the GPU only."""
    import torch
    if not torch.cuda.is_available():
        raise PtarError("pta_replicator_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback.")
    lib()
    return torch.device("cuda", torch.cuda.current_device())


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def current_stream():
    import torch
    return torch.cuda.current_stream().cuda_stream

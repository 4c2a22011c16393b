"""numpy restatement of the continuous-wave population draws (``csrc/ptar_cwpop.cuh``, ``ptar_cw_population``): the
53-bit uniform stream of Philox kind PTAR_K_CWPOP and the draw transform of ``cwpop_draw_kernel``.

The integer part and the affine maps (lo + width u, each operation rounded once) are bit-exact; ``arccos`` and the
powers are numpy's, within a few ulp of CUDA's."""
from __future__ import annotations

import numpy as np

from oracle.philox import MASK, philox4x32_10

K_CWPOP = 7
FIXED, UNIFORM, ACOS = 0, 1, 2
PARAMS = ("log10_h0", "log10_fgw", "log10_mc", "gwtheta", "gwphi", "phase0", "psi", "inc")   # counter order (ptar.h)
PPHASE_SLOT = len(PARAMS) // 2                                                                # element s * 16 + 4
SOLAR2S, MPC2S, KPC2S = 4.925838061995516e-06, 102927125054338.98, 102927125054.33899


def uniform53(a, b):
    """(a >> 5) 2^26 + (b >> 6), times 2^-53: a uniform on [0, 1) with 53 random bits."""
    a, b = np.asarray(a, dtype=np.uint64), np.asarray(b, dtype=np.uint64)
    return (((a >> np.uint64(5)) << np.uint64(26)) | (b >> np.uint64(6))).astype(np.float64) * 2.0 ** -53


def words(elem, psr, realization, seed):
    """The 4 Philox words of counter (elem, K_CWPOP | psr << 8, r & 0xffffffff, r >> 32) (arrays broadcast)."""
    r = np.asarray(realization, dtype=np.uint64)
    c1 = np.uint64(K_CWPOP) | (np.asarray(psr, dtype=np.uint64) << np.uint64(8))
    return philox4x32_10(elem, c1, r & MASK, r >> np.uint64(32), seed)


def uniforms53(elem, psr, realization, seed):
    """[..., 2]: the two uniforms of one counter, from the word pairs (w.x, w.y) and (w.z, w.w)."""
    w = words(elem, psr, realization, seed)
    return np.stack([uniform53(w[0], w[1]), uniform53(w[2], w[3])], axis=-1)


def transform(kind, lo, width, u):
    """One parameter from its uniform: lo (fixed), lo + width u (uniform) or arccos(lo + width u) (isotropic)."""
    if kind == FIXED:
        return np.full(np.shape(u), lo)
    x = np.float64(lo) + np.float64(width) * np.asarray(u, dtype=np.float64)   # two roundings, as __dadd_rn(__dmul_rn)
    return np.arccos(x) if kind == ACOS else x


def draw(pop, realizations, seed, n_psr=0):
    """The parameters of ``PulsarBatch._cwpop`` ``pop`` for the global realization ids ``realizations``: dict of
    [R, n_src] arrays (PARAMS and the linear h0, fgw, mc) and, with a drawn pulsar phase, ``pphase`` [R, n_src, n_psr]."""
    r = np.asarray(realizations, dtype=np.uint64)[:, None]
    S = pop["n_src"]
    s = np.arange(S, dtype=np.uint64)[None, :]
    out = {}
    for j, name in enumerate(PARAMS):
        u = uniforms53(s * np.uint64(16) + np.uint64(j // 2), 0, r, seed)[..., j & 1]
        out[name] = transform(pop["kind"][j], pop["lo"][j], pop["width"][j], u)
    for k in ("h0", "fgw", "mc"):
        out[k] = 10.0 ** out["log10_" + k]
    if pop["pphase"]:
        p = np.arange(n_psr, dtype=np.uint64)[None, None, :]
        u = uniforms53((s * np.uint64(16) + np.uint64(PPHASE_SLOT))[..., None], p, r[..., None], seed)[..., 0]
        out["pphase"] = 6.283185307179586 * u
    return out


def dist_mpc(h0, fgw, mc):
    """d_L [Mpc] of h0 = 2 Mc^(5/3) (pi fgw)^(2/3) / d_L (geometric units), as the draw kernel derives it."""
    mc53 = (mc * SOLAR2S) ** (5 / 3)
    return 2 * mc53 * (np.pi * fgw) ** (2 / 3) / h0 / MPC2S


def source_scalars(fgw, mc, h0, phase0, psi, inc):
    """The draw kernel's per-(r, s) record {w0, fac1, fac2, fac3, phase0/2, w0^-5/3, incfac1, incfac2, cos 2psi,
    sin 2psi} (fac3 from the derived distance)."""
    mc53 = (mc * SOLAR2S) ** (5 / 3)
    w0 = np.pi * fgw
    dist_s = 2 * mc53 * w0 ** (2 / 3) / h0
    return np.array([w0, 256 / 5 * mc53 * w0 ** (8 / 3), 1 / 32 / mc53, mc53 / dist_s, phase0 / 2, w0 ** (-5 / 3),
                     0.5 * (3 + np.cos(2 * inc)), 2 * np.cos(inc), np.cos(2 * psi), np.sin(2 * psi)])


def pulsar_constants(phat, gwtheta, gwphi, fgw, pdist_kpc, pphase=None, tol=1e-12):
    """The draw kernel's per-pulsar (F+, Fx, cosMu, pd [s]) [n_psr, 4] of one source: F from the pole-safe
    1 + Omega.p = (m.p^2 + n.p^2) / (1 - Omega.p), (0, 0) and pd = 0 where it is below ``tol``."""
    cgt, sgt, cgp, sgp = np.cos(gwtheta), np.sin(gwtheta), np.cos(gwphi), np.sin(gwphi)
    m = np.array([sgp, -cgp, 0.0])
    n = np.array([-cgt * cgp, -cgt * sgp, sgt])
    om = np.array([-sgt * cgp, -sgt * sgp, -cgt])
    mp, npr, op = phat @ m, phat @ n, phat @ om
    cosmu = -op
    with np.errstate(invalid="ignore", divide="ignore"):
        den = (mp * mp + npr * npr) / (1 - op)
    ok = den > tol
    den = np.where(ok, den, 1.0)
    pd = np.broadcast_to(np.asarray(pdist_kpc, dtype=float), cosmu.shape)
    if pphase is not None:
        with np.errstate(invalid="ignore", divide="ignore"):
            pd = pphase / (2 * np.pi * fgw * (1 - cosmu)) / KPC2S
    return np.stack([np.where(ok, 0.5 * (mp * mp - npr * npr) / den, 0.0), np.where(ok, mp * npr / den, 0.0), cosmu,
                     np.where(ok, pd * KPC2S, 0.0)], axis=1)

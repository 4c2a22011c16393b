"""numpy restatement of the transient population draws (``csrc/ptar_tpop.cuh``, ``ptar_transient_population``): the
53-bit uniform streams of Philox kinds PTAR_K_BWMPOP and PTAR_K_BURSTPOP, the draw transform of ``tpop_draw_kernel``,
its per-pulsar coefficients and the waveforms it injects.

The integer part and the affine maps (lo + width u, each operation rounded once) are bit-exact; ``arccos``, the powers and
the trigonometry are numpy's, within a few ulp of CUDA's."""
from __future__ import annotations

import numpy as np

from oracle.philox import MASK, philox4x32_10
from tests.cwpop_oracle import transform, uniform53

K_BWMPOP, K_BURSTPOP = 9, 10
BWM, BURST = 0, 1
NPAR = 10
T0, LOG10_AMP, GWTHETA, GWPHI, POL, LOG10_F0, Q, PHASE0, EPS = range(9)   # parameter indices (ptar.h)


def words(kind, elem, realization, seed):
    """The 4 Philox words of counter (elem, kind, r & 0xffffffff, r >> 32) (arrays broadcast)."""
    r = np.asarray(realization, dtype=np.uint64)
    return philox4x32_10(elem, np.uint64(kind), r & MASK, r >> np.uint64(32), seed)


def uniforms(kind, elem, realization, seed):
    """[..., 2]: the two uniforms of counter (elem, kind, r), from the word pairs (w.x, w.y) and (w.z, w.w)."""
    w = words(kind, elem, realization, seed)
    return np.stack([uniform53(w[0], w[1]), uniform53(w[2], w[3])], axis=-1)


def draw(pop, realizations, seed):
    """The NPAR parameters of ``PulsarBatch._bwmpop`` / ``_burstpop`` ``pop`` for the global realization ids
    ``realizations``: [R, n_src, NPAR]."""
    kind = K_BURSTPOP if pop["family"] == BURST else K_BWMPOP
    r = np.asarray(realizations, dtype=np.uint64)[:, None]
    s = np.arange(pop["n_src"], dtype=np.uint64)[None, :]
    out = np.empty((r.shape[0], pop["n_src"], NPAR))
    for j in range(NPAR):
        u = uniforms(kind, s * np.uint64(16) + np.uint64(j // 2), r, seed)[..., j & 1]
        out[..., j] = transform(pop["kind"][j], pop["lo"][j], pop["width"][j], u)
    return out


def patterns(phat, gwtheta, gwphi, tol=1e-12):
    """[n_psr, 2] (F+, Fx) of one source by the draw kernel's pole-safe rule ((0, 0) below ``tol`` or NaN)."""
    cgt, sgt, cgp, sgp = np.cos(gwtheta), np.sin(gwtheta), np.cos(gwphi), np.sin(gwphi)
    m = np.array([sgp, -cgp, 0.0])
    n = np.array([-cgt * cgp, -cgt * sgp, sgt])
    om = np.array([-sgt * cgp, -sgt * sgp, -cgt])
    mp, npr, op = phat @ m, phat @ n, phat @ om
    with np.errstate(invalid="ignore", divide="ignore"):
        den = (mp * mp + npr * npr) / (1 - op)
    ok = den > tol
    den = np.where(ok, den, 1.0)
    return np.stack([np.where(ok, 0.5 * (mp * mp - npr * npr) / den, 0.0), np.where(ok, mp * npr / den, 0.0)], axis=1)


def coefficients(family, v, phat):
    """[n_psr, 2] of one source's parameters ``v`` [NPAR]: (pol_a h, 0) for BWM, (alpha_a, beta_a) for the burst."""
    F = patterns(phat, v[GWTHETA], v[GWPHI])
    c, s = np.cos(2 * v[POL]), np.sin(2 * v[POL])
    A = 10.0 ** v[LOG10_AMP]
    if family == BWM:
        return np.stack([(c * F[:, 0] + s * F[:, 1]) * A, np.zeros(len(F))], axis=1)
    return np.stack([-A * (F[:, 0] * c + F[:, 1] * s), v[EPS] * A * (F[:, 0] * s - F[:, 1] * c)], axis=1)


def search_amplitudes(v):
    """(a1, a2, a3, a4) of one burst source in the burst search's ``amp`` convention (psi = 0, x = 2 pi f0 (t - t0))."""
    A, c, s, e = 10.0 ** v[LOG10_AMP], np.cos(2 * v[POL]), np.sin(2 * v[POL]), v[EPS]
    cp, sp = np.cos(v[PHASE0]), np.sin(v[PHASE0])
    return np.array([A * (c * cp - e * s * sp), A * (-c * sp - e * s * cp), A * (s * cp + e * c * sp),
                     A * (-s * sp + e * c * cp)])


def waveforms(v, t):
    """(h+, hx) of one burst source at t [s] (MJD 86400, tref = 0), untruncated."""
    f0 = 10.0 ** v[LOG10_F0]
    tau = v[Q] / (2 * np.pi * f0)
    dt = t - v[T0] * 86400.0
    g = np.exp(-(dt / tau) ** 2)
    ph = 2 * np.pi * f0 * dt + v[PHASE0]
    A = 10.0 ** v[LOG10_AMP]
    return A * g * np.cos(ph), v[EPS] * A * g * np.sin(ph)

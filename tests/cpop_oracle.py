"""numpy restatement of the common-process population draws (``csrc/ptar_cpop.cuh``, ``ptar_common_population``): the
Philox stream of kind PTAR_K_CPOP, the hyperparameter draws, the fp64 Box-Muller normals, the spectrum and the ORF mixing
of ``cpop_draw_kernel``, and the injection F_a c_a on the host.

The integer part, the affine maps and the mixing's operation order are restated exactly; log, sin, cos, pow and 10^x
are numpy's, within a few ulp of CUDA's."""
from __future__ import annotations

import numpy as np

from oracle.philox import MASK, philox4x32_10
from tests.cwpop_oracle import FIXED, UNIFORM, transform, uniform53

K_CPOP = 8
HYPER = 0x10000
TWO_PI = 6.283185307179586

__all__ = ("FIXED", "UNIFORM", "words", "hyper", "normals", "amplitude", "coefficients", "injection")


def words(elem, psr, realization, seed):
    """The 4 Philox words of counter (elem, K_CPOP | psr << 8, r & 0xffffffff, r >> 32) (arrays broadcast)."""
    r = np.asarray(realization, dtype=np.uint64)
    c1 = np.uint64(K_CPOP) | (np.asarray(psr, dtype=np.uint64) << np.uint64(8))
    return philox4x32_10(elem, c1, r & MASK, r >> np.uint64(32), seed)


def _hyper_uniform(j, realizations, seed):
    """The uniform of hyperparameter j: pair j // 2, word pair j & 1."""
    w = words(HYPER + j // 2, 0, realizations, seed)
    return uniform53(w[0], w[1]) if j % 2 == 0 else uniform53(w[2], w[3])


def hyper(pop, realizations, seed):
    """The hyperparameters of ``PulsarBatch._cpop`` ``pop`` for the global realization ids ``realizations``: dict
    ``log10_A``, ``gamma`` [R] (power law) or ``log10_rho`` [R, K] (free spectrum)."""
    r = np.asarray(realizations, dtype=np.uint64)
    if pop["spectrum"] == "powerlaw":
        return {name: transform(pop["kind"][j], pop["lo"][j], pop["width"][j], _hyper_uniform(j, r, seed))
                for j, name in enumerate(("log10_A", "gamma"))}
    return dict(log10_rho=np.stack([transform(pop["kind"][0], pop["lo"][0], pop["width"][0], _hyper_uniform(k, r, seed))
                                    for k in range(pop["K"])], axis=-1))


def normals(realizations, n_psr, K, seed):
    """z [R, n_psr, 2K]: per (pulsar b, bin k) the fp64 Box-Muller pair of counter (k, K_CPOP | b << 8, r),
    rho = sqrt(-2 ln(1 - u1)), theta = 2 pi u2, z[2k] = rho cos theta, z[2k + 1] = rho sin theta."""
    r = np.asarray(realizations, dtype=np.uint64)[:, None, None]
    b = np.arange(n_psr, dtype=np.uint64)[None, :, None]
    k = np.arange(K, dtype=np.uint64)[None, None, :]
    w = words(k, b, r, seed)
    u1, u2 = uniform53(w[0], w[1]), uniform53(w[2], w[3])
    rho = np.sqrt(-2.0 * np.log(1.0 - u1))
    th = TWO_PI * u2
    z = np.empty(u1.shape[:2] + (2 * K,))
    z[..., 0::2], z[..., 1::2] = rho * np.cos(th), rho * np.sin(th)
    return z


def amplitude(pop, hyp):
    """sqrt(phi_k) [R, K] of the draws ``hyp``: A sqrt(phi~_k) through A^2 phi~ with phi~ = _powerlaw_prior (power
    law), or rho_k = 10^log10_rho_k (free spectrum), in the kernel's order of operations."""
    from pta_replicator_b200 import constants as const
    f = np.arange(1, pop["K"] + 1) / pop["Tspan"]
    if pop["spectrum"] == "powerlaw":
        A = 10.0 ** hyp["log10_A"][:, None]
        pt = (f / (1 / const.YEAR_IN_SEC))[None, :] ** (-hyp["gamma"][:, None]) / (12 * np.pi**2 * pop["Tspan"]) \
            * const.YEAR_IN_SEC**3
        return np.sqrt((A * A) * pt)
    return 10.0 ** hyp["log10_rho"]


def coefficients(pop, realizations, seed, n_psr):
    """(c [R, P, 2K], envelope [R, P, 2K], z): c = sqrt(phi_k) sum_b B_ab z_b in the kernel's order (b ascending, each
    product and sum rounded once), and the envelope sqrt(phi_k) sum_b |B_ab| |z_b| that bounds the effect of an error in
    the normals."""
    hyp = hyper(pop, realizations, seed)
    a = np.repeat(amplitude(pop, hyp), 2, axis=-1)[:, None, :]                   # [R, 1, 2K]
    z = normals(realizations, n_psr, pop["K"], seed)
    B = None if pop["orf"] is None else pop["orf"]["B"]                      # Gamma = B B^T, None: Gamma = I
    if B is None:
        s, env = z, np.abs(z)
    else:
        s = np.zeros_like(z)
        for b in range(n_psr):                                                   # sequential, as the kernel sums
            s = s + B[None, :, b, None] * z[:, b, None, :]
        env = np.einsum("ab,rbj->raj", np.abs(B), np.abs(z))
    return a * s, a * env, z


def injection(batch, c, K, Tspan):
    """rows [R, ld] of F_a c_a on the host (engine._sincos_basis on absolute TDB time), 0 in alignment slots."""
    from pta_replicator_b200.engine import _sincos_basis
    f = np.arange(1, K + 1) / Tspan
    out = np.zeros((c.shape[0], batch.ld))
    for i in range(batch.n_psr):
        s, n = batch.toa_off[i], batch.ntoa[i]
        out[:, s:s + n] = c[:, i] @ _sincos_basis(batch.t_tdb[i], f).T
    return out

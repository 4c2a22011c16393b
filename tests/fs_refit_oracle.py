"""TEST INFRASTRUCTURE ONLY -- oracles of the free spectrum's spectral refit (``PulsarBatch.set_spectral_refit``).

``lnl_map`` is independent of the eigen statics: the sum over the bins of the dense per-bin likelihood of
``fs_oracle.lnl_map`` (explicit covariances, dense solves and ``slogdet``), each bin evaluated at the template's own
rho_k.  ``lnl_of_statics`` is the eigen form the kernels evaluate, in numpy on the plan's statics."""
from __future__ import annotations

import numpy as np

from tests import fs_oracle as FO


def lnl_map(b, rows, rho2, orf=None, **kw):
    """ln L [R, T] of engine-order rows [R, ld] for the templates rho2 [T, K] (rho_k(t)^2 > 0): sum_k of the dense
    ln L_k at rho_k(t)."""
    T, K = rho2.shape
    per = FO.lnl_map(b, rows, 0.5 * np.log10(rho2.ravel()), K, orf=orf, **kw)      # [R, K, T K]
    per = per.reshape(rows.shape[0], K, T, K)
    return sum(per[:, k, :, k] for k in range(K))


def lnl_of_statics(b, pf, pm, rows, prefix=""):
    """ln L [R, Ny, Nx] of one refit model (its statics ``pm`` = plan()["fs_refit"]["models"][name]) from the free
    spectrum's statics ``pf``: y = V_k X_k, w = rho^2 / (1 + rho^2 lambda), 1/2 sum_k sum_j w y^2 - 1/2 ldet."""
    n = 2 * b.n_psr
    X = FO.gather(b, pf, rows)
    V, lam = pf[prefix + "V"][:, :n, :n], pf[prefix + "lam"][:, :n]
    y2 = np.einsum("kji,rki->rkj", V, X) ** 2                                      # [R, K, n]
    r2 = pm["rho2_kt"]                                                              # [K, T]
    w = r2[:, :, None] / (1.0 + r2[:, :, None] * lam[:, None, :])                   # [K, T, n]
    q = np.einsum("rkj,ktj->rt", y2, w)
    return (0.5 * q - 0.5 * pm[prefix + "ldet"].ravel()[None]).reshape(rows.shape[0], *pm["ldet"].shape)

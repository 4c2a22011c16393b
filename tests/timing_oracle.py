"""TEST INFRASTRUCTURE ONLY -- oracle of the linear timing-model fit (``PulsarBatch.set_timing_model``).

An independent restatement: its own design matrix (powers of the standardised time, JUMP groups in sorted-name order
with the last one dropped, where the engine uses the normalised span and drops the earliest group; the post-fit
residual does not depend on either choice) and the SVD least-squares solver of LAPACK (``np.linalg.lstsq``, gelsd), no
QR.  Used by ``smoke()`` and the timing-model tests."""
from __future__ import annotations

import numpy as np


def timing_design_matrix(t_sec, poly=2, flag_values=None, extra=None):
    """Design matrix [n, k] in the caller's TOA order: powers 0..poly of (t - mean t) / std t (poly=None: none), one
    indicator column per distinct flag value (None = TOAs without the flag; with an offset column the LAST group in
    sorted-name order is dropped) and the columns of ``extra`` [n, m]."""
    t = np.asarray(t_sec, dtype=float)
    cols = []
    if poly is not None:
        x = (t - t.mean()) / (t.std() if t.std() > 0 else 1.0)
        cols += [x**d for d in range(poly + 1)]
    if flag_values is not None:
        fv = ["\0none" if v is None else str(v) for v in flag_values]
        groups = sorted(set(fv))
        if poly is not None:
            groups = groups[:-1]
        cols += [np.array([v == g for v in fv], dtype=float) for g in groups]
    if extra is not None:
        ex = np.asarray(extra, dtype=float)
        cols += list(ex.reshape(len(t), -1).T)
    return np.stack(cols, axis=1)


def postfit_lstsq(r, M, sigma):
    """Weighted least-squares post-fit residuals r - M beta, beta = argmin |W^{1/2} (r - M beta)|, W = diag(1/sigma^2),
    by the SVD solver (np.linalg.lstsq, LAPACK gelsd).  ``r`` is [n] or [R, n]."""
    r = np.asarray(r, dtype=float)
    w = 1.0 / np.asarray(sigma, dtype=float)
    rhs = (r * w).T
    beta = np.linalg.lstsq(M * w[:, None], rhs, rcond=None)[0]
    return r - (M @ beta).T

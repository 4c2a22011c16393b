"""Spectral models for the free spectrum's refit (``PulsarBatch.set_spectral_refit``).

A model is a 2-D grid of parameters (x, y) and the GW variance per Fourier coefficient it gives in every bin of the free
spectrum, rho_k(t)^2 in s^2 at f_k = k / Tspan: the free spectrum's own convention (``set_free_spectrum``), in which a
power law has rho_k^2 = A^2 phi~_k.  x is the amplitude-like axis: the amplitude prior, the upper limit and the ``_x_``
outputs of the refit refer to it.  The prior on y is uniform on the grid.
"""
from __future__ import annotations

from typing import Callable, NamedTuple

import numpy as np

from . import constants as const
from .engine import _powerlaw_prior


class SpectralModel(NamedTuple):
    """A spectral model on the grid x [Nx] (2..256 strictly increasing points) x y [Ny] (1..256): ``rho2(f [K], Tspan,
    x [Nx], y [Ny])`` -> rho_k^2 [Ny, Nx, K] in s^2, finite and >= 0."""
    x: np.ndarray
    y: np.ndarray
    rho2: Callable


def powerlaw(log10_A=np.linspace(-18, -12, 97), gamma=np.linspace(0, 7, 57)):
    """The power law of the CURN likelihood: rho_k^2 = 10^(2 x) phi~_k(gamma), phi~ the ``set_red`` power law at
    log10_A = 0 (the expression of the CURN statics), x = log10 A, y = gamma.  The defaults are the CURN defaults, so the
    two maps compare point for point."""
    def rho2(f, Tspan, x, y):
        pt = np.stack([_powerlaw_prior(f, g, Tspan)[0::2] for g in y])           # [Ny, K]
        return 10.0 ** (2 * x)[None, :, None] * pt[:, None, :]
    return SpectralModel(np.asarray(log10_A, dtype=float), np.asarray(gamma, dtype=float), rho2)


def turnover(log10_A=np.linspace(-18, -12, 97), log10_f0=np.linspace(-9.5, -7.5, 41), gamma=13.0 / 3.0, beta=1.0,
             power=1.0):
    """The turnover spectrum of ``set_gwb(turnover=True)``: h_c(f) = A (f / f_yr)^alpha / (1 + (f / f0)^(power (alpha -
    beta)))^(1 / power), alpha = (3 - gamma) / 2 and f_yr = 1 / 3.16e7 s (``set_gwb``'s year), as rho_k^2 = h_c(f_k)^2 /
    (12 pi^2 f_k^3 Tspan); x = log10 A, y = log10 f0 [Hz].  For f0 well below f_1 it is ``set_gwb``'s power law, which
    differs from ``powerlaw`` by the year alone (1 / 3.16e7 against 1 / 365.25 d: 0.13% in f_yr)."""
    for name, v in (("gamma", gamma), ("beta", beta), ("power", power)):
        if not np.isfinite(v):
            raise ValueError(f"{name} must be finite")
    if not power > 0:
        raise ValueError(f"power must be positive, got {power}")
    alpha = -0.5 * (gamma - 3)

    def rho2(f, Tspan, x, y):
        f = np.asarray(f, dtype=float)[None, None, :]
        hcf = 10.0 ** x[None, :, None] * (f / const.GWB_F1YR) ** alpha
        hcf = hcf / (1 + (f / 10.0 ** y[:, None, None]) ** (power * (alpha - beta))) ** (1 / power)
        return hcf**2 / (12 * np.pi**2 * f**3 * Tspan)
    return SpectralModel(np.asarray(log10_A, dtype=float), np.asarray(log10_f0, dtype=float), rho2)

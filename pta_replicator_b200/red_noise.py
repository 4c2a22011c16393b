"""Per-pulsar power-law red noise and the ORF-correlated GWB -- drop-in for
``/root/reference/pta_replicator/red_noise.py`` (``create_fourier_design_matrix_red`` :36-103,
``add_red_noise`` :106-135, ``add_gwb`` :138-298).

Draws come from the global legacy ``np.random`` stream in the reference's order (SURVEY.md 3.6);
the arithmetic runs on the GPU: ``ptar_fourier_basis`` + the epoch GEMM of ``ptar_generate`` for
``F @ y``; ``ptar_cholesky_lower`` + ``ptar_gwb_mix`` + ``ptar_gwb_synth`` (the reference's
Cholesky-colour / sqrt(C) / Hermitian-pack / IFFT / crop chain as one real linear map) + the
interpolation inside ``ptar_generate`` for the GWB.
"""
from __future__ import annotations

import numpy as np

from . import _cabi
from .engine import PulsarBatch
from .simulate import SimulatedPulsar, TimeArray


def extrap1d(interpolator):
    """Flat extrapolation wrapper for a 1-d interpolator exposing ``.x`` / ``.y`` (``red_noise.py:11-33``; used
    by the reference for ``userSpec``).  ``add_gwb`` / ``PulsarBatch.set_gwb`` apply the same rule vectorised."""
    xs, ys = np.asarray(interpolator.x), np.asarray(interpolator.y)

    def ufunclike(x):
        x = np.asarray(x, dtype=float)
        inside = np.clip(x, xs[0], xs[-1])
        return np.where(x < xs[0], ys[0], np.where(x > xs[-1], ys[-1], np.asarray(interpolator(inside))))

    return ufunclike


def create_fourier_design_matrix_red(toas: np.ndarray, nmodes: int = 30, Tspan: float = None, logf: bool = False,
                                     fmin: float = None, fmax: float = None, pshift: bool = False,
                                     libstempo_convention: bool = False, modes: np.ndarray = None) -> tuple:
    """Fourier design matrix ``F [N x 2 nmodes]`` and the repeated frequencies (computed on the GPU)."""
    import torch
    dev = _cabi.require_cuda()
    toas = np.asarray(toas, dtype=float)
    T = Tspan if Tspan is not None else toas.max() - toas.min()
    if modes is not None:
        f = np.asarray(modes, dtype=float)
        nmodes = len(f)
    elif fmin is None and fmax is None and not logf:
        f = 1.0 * np.arange(1, nmodes + 1) / T
    else:
        fmin = 1 / T if fmin is None else fmin
        fmax = nmodes / T if fmax is None else fmax
        f = np.logspace(np.log10(fmin), np.log10(fmax), nmodes) if logf else np.linspace(fmin, fmax, nmodes)
    # random phase per mode from the global legacy stream, exactly where the reference draws it (red_noise.py:83-84)
    ranphase = np.random.uniform(0.0, 2 * np.pi, nmodes) if pshift else None
    N = len(toas)
    tp = toas - toas[0] if libstempo_convention else toas
    F = torch.empty((N, 2 * nmodes), dtype=torch.float64, device=dev)
    off = torch.arange(N, dtype=torch.int64, device=dev) * (2 * nmodes)
    tp_d = torch.from_numpy(np.ascontiguousarray(tp)).to(dev)
    psr_d = torch.zeros(N, dtype=torch.int32, device=dev)
    f_d = torch.from_numpy(np.ascontiguousarray(f, dtype=np.float64)).to(dev)
    ph_d = None if ranphase is None else torch.from_numpy(np.ascontiguousarray(ranphase, dtype=np.float64)).to(dev)
    _cabi.check(_cabi.lib().ptar_fourier_basis(F.data_ptr(), off.data_ptr(), 1, tp_d.data_ptr(), psr_d.data_ptr(),
                                               f_d.data_ptr(), _cabi.ptr(ph_d), nmodes, int(bool(libstempo_convention)), N,
                                               _cabi.current_stream()), "ptar_fourier_basis")
    out = F.cpu().numpy()   # synchronises; the temporaries above stay referenced until here
    return out, np.repeat(f, 2)


def add_red_noise(psr: SimulatedPulsar, log10_amplitude: float, spectral_index: float, components: int = 30,
                  seed: int = None, modes: np.ndarray = None, Tspan: float = None, libstempo_convention: bool = False):
    """Red noise with P(f) = A^2/(12 pi^2) (f yr)^-gamma yr^3 on ``components`` Fourier bases.
    (``Tspan`` is accepted and ignored, as in the reference: red_noise.py:124.)"""
    if seed is not None:
        np.random.seed(seed)
    if modes is not None:
        print("Must use linear spacing.")
    batch = PulsarBatch([psr], exact_epochs=True)
    batch.set_red(0, log10_amplitude, spectral_index, components=components, modes=modes,
                  libstempo_convention=libstempo_convention)
    J = 2 * len(batch._red["f"][0])
    _add_one(psr, batch, "zrn", np.random.randn(J), "red_noise",   # red_noise.py:127
             {"amplitude": log10_amplitude, "spectral_index": spectral_index})


def _add_one(psr, batch, key, z, suffix, params):
    """Generate the one-pulsar ``batch`` once with the draws ``z`` injected as ``inject[key]``, add the row to ``psr``'s
    TOAs and record it as the signal ``<name>_<suffix>`` with ``params``."""
    row = batch.generate(1, inject={key: batch.torch.from_numpy(z)[None, None, :]})[0]
    dt = TimeArray(batch.unpack(row, 0), "s")
    psr.update_added_signals("{}_{}".format(psr.name, suffix), params, dt)
    psr.toas.adjust_TOAs(dt.to("day"))
    psr.update_residuals()


def _add_chromatic(psr, slot, suffix, log10_amplitude, spectral_index, idx, components, seed, fref):
    """One chromatic slot of a one-pulsar exact-epochs batch, injected with ``np.random.randn(2 components)``."""
    if seed is not None:
        np.random.seed(seed)
    batch = PulsarBatch([psr], exact_epochs=True)
    batch._set_chrom(slot, 0, log10_amplitude, spectral_index, idx, components, None, fref)
    _add_one(psr, batch, "zchr", np.random.randn(2 * components), suffix,
             {"amplitude": log10_amplitude, "spectral_index": spectral_index, "idx": idx, "fref": fref})


def add_dm_noise(psr: SimulatedPulsar, log10_amplitude: float, spectral_index: float, components: int = 30,
                 seed: int = None, fref: float = 1400.0):
    """Dispersion-measure variations (extension; the reference has no chromatic noise): the power-law Gaussian process of
    ``add_red_noise`` on the basis (fref / nu)^2 (sin, cos)(2 pi k t / T), enterprise's ``createfourierdesignmatrix_dm``
    with the ``powerlaw`` prior.  Draws ``np.random.randn(2 components)``."""
    _add_chromatic(psr, 0, "dm_gp", log10_amplitude, spectral_index, 2.0, components, seed, fref)


def add_chromatic_noise(psr: SimulatedPulsar, log10_amplitude: float, spectral_index: float, idx: float = 4.0,
                        components: int = 30, seed: int = None, fref: float = 1400.0):
    """A chromatic Gaussian process (extension; scattering for ``idx`` = 4): as ``add_dm_noise`` with the weight
    (fref / nu)^idx, enterprise's ``createfourierdesignmatrix_chromatic``."""
    _add_chromatic(psr, 1, "chrom_gp", log10_amplitude, spectral_index, idx, components, seed, fref)


def add_gwb(psrs: list, log10_amplitude: float, spectral_index: float, no_correlations: bool = False,
            seed: int = None, turnover: bool = False, clm: list = [np.sqrt(4.0 * np.pi)], lmax: int = 0,
            f0: float = 1e-9, beta: float = 1, power: float = 1, userSpec: np.ndarray = None, npts: int = 600,
            howml: int = 10, nf: int = None):
    """GWB-induced residuals (Chamberlin et al. 2014 / libstempo ``createGWB``) for a list of pulsars.
    ``nf`` (extension) pins the number of frequency bins, which the reference derives from a
    rounding-fragile ``len(np.arange(...))`` (SURVEY.md 0.5)."""
    if seed is not None:
        np.random.seed(seed)
    batch = PulsarBatch(psrs, exact_epochs=True)
    batch.set_gwb(log10_amplitude, spectral_index, no_correlations=no_correlations, turnover=turnover, clm=clm,
                  lmax=lmax, f0=f0, beta=beta, power=power, userSpec=userSpec, npts=npts, howml=howml, nf=nf)
    Nf = batch._gwb["Nf"]
    P = len(psrs)
    z = np.zeros((1, P, 2 * (Nf - 2)))
    for ll in range(P):                 # red_noise.py:239-240: real part then imaginary part
        re = np.random.randn(Nf)
        im = np.random.randn(Nf)
        z[0, ll, 0::2] = re[1:Nf - 1]   # bins 0 and Nf-1 are zeroed at :271-272
        z[0, ll, 1::2] = im[1:Nf - 1]
    torch = batch.torch
    row = batch.generate(1, inject=dict(gwb_z=torch.from_numpy(z)))[0].cpu().numpy()
    for i, psr in enumerate(psrs):
        dt = TimeArray(batch.unpack(row, i) / 86400.0, "day")
        psr.toas.adjust_TOAs(dt)
        psr.update_added_signals("{}_gwb".format(psr.name),
                                 {"amplitude": log10_amplitude, "spectral_index": spectral_index}, dt)
        psr.update_residuals()

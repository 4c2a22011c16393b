"""Deterministic signals -- drop-ins for ``add_cgw`` (``/root/reference/pta_replicator/deterministic.py:13-185``,
the deterministic signal on the hot path, SURVEY.md section 8a row a11), ``add_catalog_of_cws`` (:188-561, row f1) and
``add_burst`` / ``add_noise_transient`` / ``add_gw_memory`` (:718-884, row f4).
"""
from __future__ import annotations

import numpy as np

from .constants import MPC2S, SOLAR2S
from .engine import PulsarBatch
from .simulate import TimeArray


def add_cgw(psr, gwtheta, gwphi, mc, dist, fgw, phase0, psi, inc, pdist=1.0, pphase=None, psrTerm=True, evolve=True,
            phase_approx=False, tref=0, signal_name="cw"):
    """Continuous-wave residuals of one circular SMBHB (Earth + optional pulsar term), evaluated by
    ``ptar_cgw_delay`` on the GPU.  Units as in the reference: mc [Msun], dist [Mpc], fgw [Hz],
    pdist [kpc], angles [rad], tref [s]."""
    batch = PulsarBatch([psr], exact_epochs=True)
    d = batch.cgw_delays(gwtheta, gwphi, mc, dist, fgw, phase0, psi, inc, pdist=pdist, pphase=pphase,
                         psrTerm=psrTerm, evolve=evolve, phase_approx=phase_approx, tref=tref)[0]
    res = np.empty(len(d))
    res[batch.order[0]] = d
    dt = TimeArray(res, "s")
    # the reference stores the unit-converted mc / dist and the halved phase0 (deterministic.py:51-56, :167-182)
    psr.update_added_signals("{}_".format(psr.name) + signal_name,
                             {"gwtheta": gwtheta, "gwphi": gwphi, "mc": mc * SOLAR2S, "dist": dist * MPC2S, "fgw": fgw,
                              "phase0": phase0 / 2, "psi": psi, "inc": inc, "pdist": pdist, "pphase": pphase,
                              "psrTerm": psrTerm, "evolve": evolve, "phase_approx": phase_approx, "tref": tref}, dt)
    psr.toas.adjust_TOAs(dt.to("day"))
    psr.update_residuals()


def add_catalog_of_cws(psr, gwtheta_list, gwphi_list, mc_list, dist_list, fgw_list, phase0_list, psi_list, inc_list,
                       pdist=1.0, pphase=None, psrTerm=True, evolve=True, phase_approx=False, tref=0,
                       chunk_size=10_000_000, signal_name="cw_catalog"):
    """Sum of many circular SMBHBs -- drop-in for ``add_catalog_of_cws`` (deterministic.py:188-318) with the numba
    loops (:321-561) replaced by ``ptar_cw_catalog`` (thread per TOA, catalog slices staged through shared memory,
    deterministic slice reduction, NaN contributions of already-merged binaries dropped).  ``chunk_size`` is accepted
    for compatibility; the whole catalog is processed in one call and recorded once in the ledger."""
    import ctypes as C

    import torch

    from . import _cabi
    from . import orf as orf_mod
    dev = _cabi.require_cuda()
    radec = orf_mod.psrlocs_from_pulsars([psr])[0]
    ptheta, pphi = np.pi / 2 - radec[1], radec[0]
    phat = (C.c_double * 3)(np.sin(ptheta) * np.cos(pphi), np.sin(ptheta) * np.sin(pphi), np.cos(ptheta))
    cat = np.ascontiguousarray(np.stack([np.asarray(a, dtype=np.float64) for a in
                                         (gwtheta_list, gwphi_list, mc_list, dist_list, fgw_list, phase0_list, psi_list,
                                          inc_list)]))
    n_src = cat.shape[1]
    toas = np.ascontiguousarray(np.asarray(psr.toas.get_mjds().value, dtype=np.float64) * 86400 - tref)
    n = len(toas)
    n_slices = int(max(1, min(64, (n_src + 255) // 256)))
    t_d, cat_d = torch.from_numpy(toas).to(dev), torch.from_numpy(cat).to(dev)
    out = torch.empty(n, dtype=torch.float64, device=dev)
    pre = torch.empty(n_src * 16, dtype=torch.float64, device=dev)
    partial = torch.empty(n_slices * n, dtype=torch.float64, device=dev)
    mode = 0 if evolve else (1 if phase_approx else 2)
    _cabi.check(_cabi.lib().ptar_cw_catalog(out.data_ptr(), t_d.data_ptr(), n, phat, cat_d.data_ptr(), n_src, float(pdist),
                                            float(pphase) if pphase is not None else 0.0, int(pphase is not None), mode,
                                            int(bool(psrTerm)), 0, pre.data_ptr(), partial.data_ptr(), n_slices,
                                            _cabi.current_stream()), "ptar_cw_catalog")
    dt = TimeArray(out.cpu().numpy(), "s")
    psr.update_added_signals("{}_".format(psr.name) + signal_name,
                             {"gwtheta_list": gwtheta_list, "gwphi_list": gwphi_list, "mc_list": mc_list, "dist_list": dist_list,
                              "fgw_list": fgw_list, "phase0_list": phase0_list, "psi_list": psi_list, "inc_list": inc_list,
                              "pdist": pdist, "pphase": pphase, "psrTerm": psrTerm, "evolve": evolve,
                              "phase_approx": phase_approx, "tref": tref}, dt)
    psr.toas.adjust_TOAs(dt.to("day"))
    psr.update_residuals()


def _antenna(psr, gwtheta, gwphi):
    """(fplus, fcross) of deterministic.py:733-759 (Sesana et al. 2010 / Ellis et al. 2012 conventions)."""
    from . import orf as orf_mod
    cgt, cgp, sgt, sgp = np.cos(gwtheta), np.cos(gwphi), np.sin(gwtheta), np.sin(gwphi)
    m = np.array([sgp, -cgp, 0.0])
    n = np.array([-cgt * cgp, -cgt * sgp, sgt])
    om = np.array([-sgt * cgp, -sgt * sgp, -cgt])
    radec = orf_mod.psrlocs_from_pulsars([psr])[0]
    ptheta, pphi = np.pi / 2 - radec[1], radec[0]
    phat = np.array([np.sin(ptheta) * np.cos(pphi), np.sin(ptheta) * np.sin(pphi), np.cos(ptheta)])
    fplus = 0.5 * (np.dot(m, phat) ** 2 - np.dot(n, phat) ** 2) / (1 + np.dot(om, phat))
    fcross = (np.dot(m, phat) * np.dot(n, phat)) / (1 + np.dot(om, phat))
    return float(fplus), float(fcross)


def _inject(psr, name, params, seconds):
    dt = TimeArray(np.asarray(seconds, dtype=np.float64), "s")
    psr.update_added_signals(name, params, dt)
    psr.toas.adjust_TOAs(dt.to("day"))
    psr.update_residuals()


def burst_delay(psr, gwtheta, gwphi, waveform_plus, waveform_cross, psi=0.0, tref=0, remove_quad=False, device=None):
    """The delay [s] ``add_burst`` adds to ``psr``, in its TOA table order: the two waveform callables of ``t - tref``
    [s] evaluated on the host (as in the reference), the polarisation mix and antenna projection in ``ptar_burst_delay``
    on ``device`` (default the current CUDA device) and, with ``remove_quad``, the quadratic fitted out by ``np.polyfit``
    as the reference does (:777-779)."""
    import torch

    from . import _cabi
    dev = _cabi.require_cuda() if device is None else device
    fplus, fcross = _antenna(psr, gwtheta, gwphi)
    toas = np.asarray(psr.toas.get_mjds().value, dtype=np.float64) * 86400 - tref
    def sample(w):  # a scalar-valued callable broadcasts like numpy would in the reference
        return torch.from_numpy(np.array(np.broadcast_to(np.asarray(w(toas), dtype=np.float64), toas.shape))).to(dev)

    hp, hx = sample(waveform_plus), sample(waveform_cross)
    out = torch.empty(len(toas), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _cabi.check(_cabi.lib().ptar_burst_delay(out.data_ptr(), hp.data_ptr(), hx.data_ptr(), fplus, fcross,
                                                 float(np.cos(2 * psi)), float(np.sin(2 * psi)), 0, len(toas),
                                                 _cabi.current_stream()), "ptar_burst_delay")
    res = out.cpu().numpy()
    if remove_quad:
        pp = np.polyfit(toas, res, 2)
        res = res - pp[0] * toas ** 2 - pp[1] * toas - pp[2]
    return res


def add_burst(psr, gwtheta, gwphi, waveform_plus, waveform_cross, psi=0.0, tref=0, remove_quad=False, signal_name="burst"):
    """GW burst of arbitrary waveform with elliptical polarisation -- drop-in for ``add_burst``
    (deterministic.py:718-793): the delay of ``burst_delay``."""
    res = burst_delay(psr, gwtheta, gwphi, waveform_plus, waveform_cross, psi, tref, remove_quad)
    _inject(psr, "{}_".format(psr.name) + signal_name,
            {"gwtheta": gwtheta, "gwphi": gwphi, "waveform_plus": waveform_plus, "waveform_cross": waveform_cross, "psi": psi,
             "tref": tref, "remove_quad": remove_quad}, res)


def noise_transient_delay(psr, waveform, tref=0):
    """The delay [s] ``add_noise_transient`` adds to ``psr``, in its TOA table order: the caller's callable sampled at
    ``t - tref`` [s] (t = MJD 86400)."""
    toas = np.asarray(psr.toas.get_mjds().value, dtype=np.float64) * 86400 - tref
    return np.array(np.broadcast_to(np.asarray(waveform(toas), dtype=np.float64), toas.shape))


def add_noise_transient(psr, waveform, tref=0, signal_name="noise_transient"):
    """Incoherent transient of arbitrary waveform in one pulsar -- drop-in for ``add_noise_transient``
    (deterministic.py:796-819).  The delay IS the caller's callable sampled at ``t - tref``; there is no arithmetic to
    move to the device, so this is ledger bookkeeping only."""
    _inject(psr, "{}_".format(psr.name) + signal_name, {"waveform": waveform, "tref": tref},
            noise_transient_delay(psr, waveform, tref))


def add_gw_memory(psr, strain, gwtheta, gwphi, bwm_pol, t0_mjd, signal_name="gw_memory"):
    """Burst with memory -- drop-in for ``add_gw_memory`` (deterministic.py:822-884): a ramp
    ``pol * strain * (t - t0)`` after the burst epoch, evaluated by ``ptar_memory_delay``."""
    import torch

    from . import _cabi
    dev = _cabi.require_cuda()
    fplus, fcross = _antenna(psr, gwtheta, gwphi)
    pol = np.cos(2 * bwm_pol) * fplus + np.sin(2 * bwm_pol) * fcross
    toas = np.asarray(psr.toas.get_mjds().value, dtype=np.float64) * 86400
    t_d = torch.from_numpy(np.ascontiguousarray(toas)).to(dev)
    out = torch.empty(len(toas), dtype=torch.float64, device=dev)
    _cabi.check(_cabi.lib().ptar_memory_delay(out.data_ptr(), t_d.data_ptr(), float(pol * strain), float(t0_mjd * 86400), 0,
                                              len(toas), _cabi.current_stream()), "ptar_memory_delay")
    _inject(psr, "{}_".format(psr.name) + signal_name,
            {"strain": strain, "gwtheta": gwtheta, "gwphi": gwphi, "bwm_pol": bwm_pol, "t0_mjd": t0_mjd}, out.cpu().numpy())


def add_gwb_plus_outlier_cws(psrs, vals, weights, fobs, T_obs, outlier_per_bin=100, seed=None):
    """Realistic data sets from a binary population -- drop-in for ``add_gwb_plus_outlier_cws``
    (deterministic.py:565-715; Becsy, Cornish & Kelley 2022): the loudest ``outlier_per_bin`` binaries of every
    frequency bin are injected one by one (``add_catalog_of_cws`` -> ``ptar_cw_catalog``), the rest as a GWB with a
    free spectrum (``add_gwb(userSpec=...)`` -> the GWB kernels).  ``vals`` = [Mtot [g], q, z, f_obs [Hz]] per
    population sample, ``weights`` = binaries per sample, ``fobs`` = bin edges [Hz], ``T_obs`` [s]; the holodeck
    helpers are restated in ``population.py``.  Same draw order from the global ``np.random`` stream and the same
    return tuple as the reference."""
    from .population import partition_population
    from .red_noise import add_gwb
    f_centers, free_spec, outlier_fo, outlier_hs, outlier_mc, outlier_dl = partition_population(
        vals, weights, fobs, T_obs, outlier_per_bin)
    add_gwb(psrs, None, None, userSpec=np.array([f_centers, np.sqrt(free_spec)]).T, howml=10, seed=seed)
    n_cw = outlier_hs.shape[0]
    gwthetas = np.arccos(np.random.uniform(low=-1.0, high=1.0, size=n_cw))       # deterministic.py:693-697
    gwphis = np.random.uniform(low=0.0, high=2 * np.pi, size=n_cw)
    phases = np.random.uniform(low=0.0, high=2 * np.pi, size=n_cw)
    psis = np.random.uniform(low=0.0, high=np.pi, size=n_cw)
    incs = np.arccos(np.random.uniform(low=-1.0, high=1.0, size=n_cw))
    for psr in psrs:
        add_catalog_of_cws(psr, gwtheta_list=gwthetas, gwphi_list=gwphis, mc_list=outlier_mc, dist_list=outlier_dl,
                           fgw_list=outlier_fo, phase0_list=phases, psi_list=psis, inc_list=incs, pdist=1.0, pphase=None,
                           psrTerm=True, evolve=True, phase_approx=False, tref=53000 * 86400)
    return f_centers, free_spec, outlier_fo, outlier_hs, outlier_mc, outlier_dl, gwthetas, gwphis, phases, psis, incs

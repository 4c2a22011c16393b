"""Synthetic NANOGrav-15yr-shaped data sets for the benchmark (SURVEY.md section 8d).

There is no network for the real 15-yr release, so the benchmark runs on synthetic TOAs of the
same shape: the 67 pulsars of the 15-yr noise dictionary that have a red-noise entry, positions
uniform on the sphere (stored as RAJ [h] / DECJ [deg]), 100-500 observing epochs per pulsar in
MJD 53000-58800, and per epoch either 10-60 sub-band TOAs spread over < 0.5 s ("full",
sum N_toa ~ 7e5) or one TOA ("epoch", ~2e4), sigma ~ U(0.1, 3) us, the backend cycling per epoch
over the pulsar's backends in the dictionary.  Seeded with ``np.random.default_rng(20250922)``.
"""
from __future__ import annotations

import numpy as np

from . import noise_dict as nd
from .simulate import make_ideal, pulsar_from_arrays


def make_ng15_like(kind: str = "full", seed: int = 20250922, npsr: int = None, noise_params: dict = None):
    """Return ``(psrs, noise)``: ideal ``SimulatedPulsar`` objects and ``{name: per_pulsar(...)}``."""
    noise_params = nd.load_noise_dict() if noise_params is None else noise_params
    names = nd.pulsar_names(noise_params)
    if npsr is not None:
        names = names[:npsr]
    rng = np.random.default_rng(seed)
    psrs, noise = [], {}
    for name in names:
        pp = nd.per_pulsar(noise_params, name)
        nep = int(rng.integers(100, 501))
        nsub = int(rng.integers(10, 61)) if kind == "full" else 1
        epochs = np.sort(rng.uniform(53000.0, 58800.0, nep))
        off = rng.uniform(0.0, 0.5, (nep, nsub)) / 86400.0
        mjd = (epochs[:, None] + off).reshape(-1)
        mjd = np.asarray(mjd, dtype=np.float64)
        sig = rng.uniform(0.1, 3.0, mjd.size)
        raj = float(rng.uniform(0.0, 24.0))
        decj = float(np.degrees(np.arcsin(rng.uniform(-1.0, 1.0))))
        be = pp["backends"]
        bidx = (np.arange(nep) % len(be))[:, None].repeat(nsub, axis=1).reshape(-1)
        flags = [{"f": be[b], "pta": "NANOGrav"} for b in bidx]
        p = pulsar_from_arrays(name, {"RAJ": raj, "DECJ": decj}, mjd.astype(np.longdouble), sig, flags=flags)
        make_ideal(p)
        psrs.append(p)
        noise[name] = pp
    return psrs, noise


def ng15_recipe(batch, noise, gw_log10_A=-14.6733, gw_gamma=13.0 / 3.0, components=30, coarsegrain=1.0 / 86400.0,
                white=True, ecorr=True, red=True, gwb=True):
    """Register the 15-yr recipe of ``examples/add_noise.ipynb`` cells 9 and 11 on a ``PulsarBatch``."""
    for i, p in enumerate(batch.psrs):
        pp = noise[p.name]
        be = np.array(pp["backends"])
        if white:
            batch.set_white(i, efac=pp["efac"], log10_equad=pp["log10_equad"], flagid="f", flags=be)
        if ecorr:
            batch.set_ecorr(i, pp["log10_ecorr"], flagid="f", flags=be, coarsegrain=coarsegrain)
        if red:
            batch.set_red(i, pp["rn_log10_A"], pp["rn_gamma"], components=components)
    if gwb:
        batch.set_gwb(gw_log10_A, gw_gamma)
    return batch


# receiver bands [MHz] by a substring of the backend name; anything else observes at L band
RECEIVER_BANDS = (("430", (422.0, 442.0)), ("Rcvr_800", (720.0, 920.0)), ("L-wide", (1150.0, 1880.0)),
                  ("Rcvr1_2", (1150.0, 1880.0)), ("S-wide", (1700.0, 2400.0)))


def spread_subband_frequencies(psrs):
    """Give every epoch's sub-band TOAs (runs < 10 s apart) radio frequencies spread evenly over the band of the epoch's
    backend (flag ``f``), in place, so that chromatic processes see a realistic frequency coverage."""
    for p in psrs:
        t = np.asarray(p.toas.table["tdbld"], dtype=np.float64) * 86400.0
        fl = p.toas.table["flags"]
        o = np.argsort(t, kind="stable")
        starts = np.flatnonzero(np.r_[True, np.diff(t[o]) > 10.0])
        for a, z in zip(starts, np.r_[starts[1:], len(o)]):
            be = str(fl[int(o[a])].get("f"))
            lo, hi = next((b for key, b in RECEIVER_BANDS if key in be), (1150.0, 1880.0))
            p.toas.freq[o[a:z]] = np.linspace(lo, hi, z - a) if z - a > 1 else 0.5 * (lo + hi)
    return psrs

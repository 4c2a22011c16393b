"""Pulsar container and ingest for the H100 residual generator (PINT-free).

Mirrors the public surface of ``/root/reference/pta_replicator/simulate.py``:
``SimulatedPulsar`` (:23-95), ``simulate_pulsar`` (:98-135), ``load_pulsar``
(:138-167), ``load_from_directories`` (:170-190), ``make_ideal`` (:193-202) --
same names, argument meaning, ledger semantics and error behaviour -- but the
container holds plain arrays instead of PINT objects: the injection kernels only
need per-TOA times, uncertainties and flags, and the pulsar's sky position.

Residuals without PINT: the loaded TOAs are taken to be the timing model's ideal
arrival times, so the post-fit-like residual is the sum of injected delays minus
its uncertainty-weighted mean (SURVEY.md Appendix A; pins the reference's libstempo
golden vector to <= 4e-4 rms).  PINT itself, fitting, ``to_enterprise`` and par
writing are out of scope (SURVEY.md section 8f, row f3).
"""
from __future__ import annotations

import glob
import os
from dataclasses import dataclass

import numpy as np

from . import partim

_UNIT_IN_SECONDS = {"s": 1.0, "us": 1e-6, "ms": 1e-3, "ns": 1e-9, "day": 86400.0, "d": 86400.0}


class TimeArray(np.ndarray):
    """float64 ndarray tagged with a time unit; the slice of astropy's Quantity API
    that reference user code touches on ledger entries and residuals
    (``.value``, ``.to(unit)``, ``.to_value(unit)``)."""

    def __new__(cls, values, unit="s"):
        obj = np.asarray(values, dtype=float).view(cls)
        obj.unit = str(unit)
        return obj

    def __array_finalize__(self, obj):
        self.unit = getattr(obj, "unit", "s")

    @property
    def value(self):
        return np.asarray(self)

    def to(self, unit):
        unit = str(unit)
        fac = _UNIT_IN_SECONDS[self.unit] / _UNIT_IN_SECONDS[unit]
        return TimeArray(np.asarray(self) * fac, unit)

    def to_value(self, unit):
        return self.to(unit).value


class _FlagColumn(list):
    """List of per-TOA flag dicts; ``.data`` as in an astropy table column."""

    @property
    def data(self):
        return self


class _Scalar:
    def __init__(self, value):
        self.value = value


class TOAs:
    """Per-TOA arrays with the accessor names the reference calls on ``pint.toa.TOAs``.

    ``table['tdbld']`` is long-double MJD (``red_noise.py:123`` casts it to f64 seconds),
    ``table['flags']`` a list of dicts (``white_noise.py:98-99``), ``get_mjds().value``
    f64 MJD, ``get_errors()`` microseconds with ``.to('s')``, ``first_MJD`` / ``last_MJD``
    (``red_noise.py:182-183``), ``adjust_TOAs`` (``white_noise.py:124``).
    """

    def __init__(self, mjd, err_us, freq=None, site=None, flags=None, names=None):
        mjd = np.asarray(mjd, dtype=np.longdouble)
        n = len(mjd)
        self.ntoas = n
        self.err_us = np.broadcast_to(np.asarray(err_us, dtype=float), (n,)).copy()
        self.freq = np.broadcast_to(np.asarray(1440.0 if freq is None else freq, dtype=float), (n,)).copy()
        self.site = list(site) if site is not None else ["AXIS"] * n
        self.names = list(names) if names is not None else ["fake"] * n
        fl = _FlagColumn(dict(f) for f in flags) if flags is not None else _FlagColumn({} for _ in range(n))
        self.table = {"tdbld": mjd.copy(), "mjd_float": np.asarray(mjd, dtype=float), "flags": fl, "freq": self.freq}
        self.delay_s = np.zeros(n)  # accumulated injected delay [s]

    def __len__(self):
        return self.ntoas

    def get_mjds(self):
        return TimeArray(np.asarray(self.table["tdbld"], dtype=float), "day")

    def get_errors(self):
        return TimeArray(self.err_us, "us")

    def get_flag_value(self, flagid):
        return [f.get(flagid) for f in self.table["flags"]]

    # PINT reports first/last MJD from its own (clock-corrected) columns; a caller that needs to
    # reproduce a PINT-made data set's GWB grid exactly can pin them here (SURVEY.md 0.5).
    first_MJD_override = None
    last_MJD_override = None

    @property
    def first_MJD(self):
        v = self.first_MJD_override
        return _Scalar(float(np.min(self.table["tdbld"])) if v is None else float(v))

    @property
    def last_MJD(self):
        v = self.last_MJD_override
        return _Scalar(float(np.max(self.table["tdbld"])) if v is None else float(v))

    def adjust_TOAs(self, delta):
        """Shift the TOAs by ``delta`` (TimeArray, or plain array of days)."""
        sec = delta.to("s").value if isinstance(delta, TimeArray) else np.asarray(delta, float) * 86400.0
        self.delay_s = self.delay_s + sec
        self.table["tdbld"] = self.table["tdbld"] + np.asarray(sec, dtype=np.longdouble) / np.longdouble(86400)
        self.table["mjd_float"] = np.asarray(self.table["tdbld"], dtype=float)


class Residuals:
    """Injected delay minus its weighted mean; the fields user code reads off
    ``pint.residuals.Residuals`` (``time_resids``, ``resids_value``, ``get_data_error``)."""

    def __init__(self, toas: TOAs, model=None):
        w = 1.0 / np.square(toas.err_us)
        d = toas.delay_s
        mean = float(np.sum(w * d) / np.sum(w)) if toas.ntoas else 0.0
        self.time_resids = TimeArray(d - mean, "s")
        self._err = toas.get_errors()

    @property
    def resids_value(self):
        return self.time_resids.value

    def get_data_error(self):
        return self._err


@dataclass
class SimulatedPulsar:
    """Holds one pulsar's TOAs, residuals, position and the injected-signal ledgers."""

    ephem: str = "DE440"
    model: dict = None
    toas: TOAs = None
    residuals: Residuals = None
    name: str = None
    loc: dict = None
    added_signals: dict = None
    added_signals_time: dict = None

    def __repr__(self):
        return f"SimulatedPulsar({self.name})"

    def _is_pint(self):
        return not isinstance(self.toas, TOAs)

    def update_residuals(self):
        if self._is_pint():     # PINT-backed pulsar (pint_bridge.load_pulsar_pint): simulate.py:40-42
            from pint.residuals import Residuals as PintResiduals
            self.residuals = PintResiduals(self.toas, self.model)
        else:
            self.residuals = Residuals(self.toas, self.model)

    def update_added_signals(self, signal_name, param_dict, dt=None):
        # simulate.py:83-89: ledgers are None until make_ideal(); names are unique
        if self.added_signals is None:
            raise ValueError("make_ideal() must be called on SimulatedPulsar before adding new signals.")
        if signal_name in self.added_signals:
            raise ValueError(f"{signal_name} already exists in the model.")
        self.added_signals[signal_name] = param_dict
        if dt is not None:
            self.added_signals_time[signal_name] = dt

    def fit(self, fitter="auto", **fitter_kwargs):
        """Refit the timing model (simulate.py:44-69): delegated to PINT for PINT-backed pulsars."""
        from . import pint_bridge
        if not self._is_pint():
            raise pint_bridge.PintUnavailable("fit() needs a PINT timing model: load the pulsar with pint_bridge.load_pulsar_pint")
        pint_bridge.fit(self, fitter, **fitter_kwargs)

    def to_enterprise(self, ephem="DE440"):
        """enterprise ``Pulsar`` (simulate.py:91-95): delegated to enterprise for PINT-backed pulsars."""
        from . import pint_bridge
        if not self._is_pint():
            raise pint_bridge.PintUnavailable("to_enterprise() needs PINT TOAs and a PINT model: load the pulsar with "
                                              "pint_bridge.load_pulsar_pint")
        return pint_bridge.to_enterprise(self, ephem)

    def write_partim(self, outpar: str, outtim: str, tempo2: bool = False):
        """Write the current (signal-shifted) TOAs and the par file (simulate.py:71-77).  PINT-backed pulsars go through
        PINT's writers; the PINT-free container writes Tempo2 ``FORMAT 1`` lines itself (MJD with 19 decimals, all flags;
        ``partim.read_tim`` reads them back exactly) and copies the par file through."""
        if self._is_pint():
            from . import pint_bridge
            return pint_bridge.write_partim(self, outpar, outtim, tempo2)
        cols = {"name": self.toas.names, "freq": self.toas.freq, "mjd": self.toas.table["tdbld"],
                "err_us": self.toas.err_us, "site": self.toas.site, "flags": self.toas.table["flags"]}
        partim.write_tim(outtim, cols)
        src = (self.model or {}).get("_path")
        if src and os.path.isfile(src):
            with open(src) as fi, open(outpar, "w") as fo:
                fo.write(fi.read())


def _location(par: dict) -> dict:
    return dict(par["_loc"])


def simulate_pulsar(parfile: str, obstimes, toaerr, freq=1440.0, observatory="AXIS", flags=None,
                    ephem: str = "DE440") -> SimulatedPulsar:
    """Fake TOAs at ``obstimes`` [MJD] with errors ``toaerr`` [us] for the pulsar in ``parfile``."""
    if not os.path.isfile(parfile):
        raise FileNotFoundError("par file does not exist.")
    par = partim.read_par(parfile)
    par["_path"] = parfile
    obstimes = np.asarray(obstimes, dtype=np.longdouble)
    n = len(obstimes)
    if flags is None:
        fl = None
    elif isinstance(flags, dict):
        fl = [dict(flags) for _ in range(n)]
    else:
        fl = list(flags)
    toas = TOAs(obstimes, toaerr, freq=freq, site=[observatory] * n, flags=fl)
    psr = SimulatedPulsar(ephem=ephem, model=par, toas=toas, name=par["_name"], loc=_location(par))
    psr.update_residuals()
    return psr


def load_pulsar(parfile: str, timfile: str, ephem: str = "DE440") -> SimulatedPulsar:
    """Load one pulsar from a par and a tim file."""
    if not os.path.isfile(parfile):
        raise FileNotFoundError("par file does not exist.")
    if not os.path.isfile(timfile):
        raise FileNotFoundError("tim file does not exist.")
    par = partim.read_par(parfile)
    par["_path"] = parfile
    cols = partim.read_tim(timfile)
    toas = TOAs(cols["mjd"], cols["err_us"], freq=cols["freq"], site=cols["site"], flags=cols["flags"],
                names=cols["name"])
    psr = SimulatedPulsar(ephem=ephem, model=par, toas=toas, name=par["_name"], loc=_location(par))
    psr.update_residuals()
    return psr


def load_from_directories(pardir: str, timdir: str, ephem: str = "DE440", num_psrs: int = None,
                          debug=False) -> list:
    """Pair sorted ``*.par`` (minus ``.t2`` variants) with sorted ``*.tim`` and load them."""
    if not os.path.isdir(pardir):
        raise FileNotFoundError("par directory does not exist.")
    if not os.path.isdir(timdir):
        raise FileNotFoundError("tim directory does not exist.")
    pars = [p for p in sorted(glob.glob(os.path.join(pardir, "*.par"))) if ".t2" not in p]
    tims = sorted(glob.glob(os.path.join(timdir, "*.tim")))
    out = []
    for par, tim in zip(pars, tims):
        if num_psrs and len(out) >= num_psrs:
            break
        if debug:
            print(f"loading {par=}, {tim=}")
        out.append(load_pulsar(par, tim, ephem=ephem))
    return out


def make_ideal(psr: SimulatedPulsar, iterations: int = 2):
    """Zero the residuals and open the signal ledgers (required before any ``add_*``)."""
    for _ in range(max(int(iterations), 1)):
        psr.toas.table["tdbld"] = psr.toas.table["tdbld"] - np.asarray(psr.toas.delay_s, np.longdouble) / np.longdouble(86400)
        psr.toas.delay_s = np.zeros(psr.toas.ntoas)
    psr.toas.table["mjd_float"] = np.asarray(psr.toas.table["tdbld"], dtype=float)
    psr.added_signals = {}
    psr.added_signals_time = {}
    psr.update_residuals()


def pulsar_from_arrays(name, loc, mjd, err_us, flags=None, freq=1440.0, site="AXIS") -> SimulatedPulsar:
    """Build a pulsar from in-memory arrays (synthetic data sets; no files)."""
    n = len(mjd)
    toas = TOAs(mjd, err_us, freq=freq, site=[site] * n, flags=flags)
    psr = SimulatedPulsar(model={"_name": name, "_loc": dict(loc)}, toas=toas, name=name, loc=dict(loc))
    psr.update_residuals()
    return psr

"""Parse NANOGrav-style noise dictionaries (``noise_dicts/ng15_dict.json`` of the reference) into the
per-backend arrays the injection functions take -- the logic of ``examples/add_noise.ipynb`` cells 5-6
(substring match on the pulsar name, suffix stripping), with the one key asymmetry of the 15-yr
dictionary handled (a backend that has equad/ecorr but no efac gets efac = 1).

``data/ng15_noise_dict.json`` is the reference's data file re-serialised (data, not source).
"""
from __future__ import annotations

import json
import os

import numpy as np

NG15_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "ng15_noise_dict.json")


def load_noise_dict(path: str = NG15_PATH) -> dict:
    with open(path) as fh:
        return {k: float(v) for k, v in json.load(fh).items()}


def pulsar_names(noise_params: dict, require_red: bool = True) -> list:
    """Sorted pulsar names that appear in the dictionary (those with a red-noise entry by default)."""
    suf = "_red_noise_gamma"
    if require_red:
        return sorted(k[:-len(suf)] for k in noise_params if k.endswith(suf))
    names = set()
    for k in noise_params:
        for s in ("_efac", "_log10_t2equad", "_log10_ecorr", suf, "_red_noise_log10_A"):
            if k.endswith(s):
                names.add(k.split("_")[0])
    return sorted(names)


def per_pulsar(noise_params: dict, name: str) -> dict:
    """``{'backends': [...], 'efac': arr, 'log10_equad': arr, 'log10_ecorr': arr, 'rn_log10_A', 'rn_gamma', 'dm_log10_A',
    'dm_gamma', 'chrom_log10_A', 'chrom_gamma', 'chrom_idx'}``; each process's values are None when its keys are absent."""
    pre = name + "_"
    be = {}
    out = {"rn_log10_A": None, "rn_gamma": None}
    # chromatic processes (enterprise_extensions' dm_gp / chrom_gp names); chrom_idx defaults to 4 when absent
    chrom = {"dm_gp_log10_A": "dm_log10_A", "dm_gp_gamma": "dm_gamma", "chrom_gp_log10_A": "chrom_log10_A",
             "chrom_gp_gamma": "chrom_gamma", "chrom_gp_idx": "chrom_idx"}
    out.update({v: None for v in chrom.values()})
    for k, v in noise_params.items():
        if not k.startswith(pre):
            continue
        rest = k[len(pre):]
        if rest in chrom:
            out[chrom[rest]] = v
        elif rest == "red_noise_gamma":
            out["rn_gamma"] = v
        elif rest == "red_noise_log10_A":
            out["rn_log10_A"] = v
        elif rest.endswith("_efac"):
            be.setdefault(rest[:-5], {})["efac"] = v
        elif rest.endswith("_log10_t2equad"):
            be.setdefault(rest[:-14], {})["equad"] = v
        elif rest.endswith("_log10_tnequad"):
            be.setdefault(rest[:-14], {})["equad"] = v
        elif rest.endswith("_log10_ecorr"):
            be.setdefault(rest[:-12], {})["ecorr"] = v
    names = sorted(be)
    out["backends"] = names
    out["efac"] = np.array([be[b].get("efac", 1.0) for b in names])
    out["log10_equad"] = np.array([be[b].get("equad", -300.0) for b in names])
    out["log10_ecorr"] = np.array([be[b].get("ecorr", -300.0) for b in names])
    if out["chrom_log10_A"] is not None and out["chrom_idx"] is None:
        out["chrom_idx"] = 4.0
    return out

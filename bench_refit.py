#!/usr/bin/env python
"""Benchmark of the free spectrum's spectral refit: the workload of bench_fs.py (bench.py's config 2: 67-pulsar ng15-full
EFAC/EQUAD + ECORR + red noise + HD GWB, with ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar, and
``set_free_spectrum(orf="hd")`` at its defaults: K = 14 bins, 121 log10 rho points, uncorrelated and HD models) plus
``set_spectral_refit({"powerlaw": spectra.powerlaw(), "turnover": spectra.turnover()})`` at their default grids (97 x 57
and 97 x 41 templates).  Prints one JSON line.

    python bench_refit.py --steps K --warmup W [--nreal R]

A step = ``free_spectrum(R)``: R realizations generated (pre-fit) and reduced to the free spectrum's per-bin summaries
and every refit model's summaries, both free-spectrum models.  ``value`` = realizations/s of the whole step;
``kernels_ms_per_step`` = per-kernel ms per step from CUDA events around every launch in a second pass of the same
steps; ``fs_refit`` = the algorithmic flop of the refit GEMMs, 2 R T K n summed over the (free-spectrum model, refit
model) pairs with n = 2 n_psr, the flop fs_refit_kernel executes (64-realization and 64-template blocks, depth K np) and
the achieved TFLOP/s of both against the data-sheet 67 TFLOP/s of fp64 tensor cores; ``refit_statics_s`` = the refit's
host statics, ``fs_statics_s`` the free spectrum's.  The card name and power limit are read with a read-only nvidia-smi
query in the same run.  Writes nothing into the tree.
"""
from __future__ import annotations

import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True   # the tree may be read-only

import bench  # noqa: E402  (the metric workload)
from bench_postfit import card, parse, parser, timed_statistic, timing_model_batch  # noqa: E402


def main():
    from pta_replicator_b200 import spectra
    args = parse(parser())
    b, kind, t0 = timing_model_batch(args)
    b.set_free_spectrum(orf="hd")
    b.set_spectral_refit({"powerlaw": spectra.powerlaw(), "turnover": spectra.turnover()})
    b.compile()
    setup_s = time.perf_counter() - t0
    R = args.nreal
    ms, kms = timed_statistic(b.free_spectrum, R, args.steps, args.warmup)
    st = b.compile()["fs"]
    m = st["fs"]
    n, K, npad = 2 * b.n_psr, m.n_bin, m.np
    n_fs = 1 + ("hd" in st)
    tmpl = {rf["name"]: rf["shape"][0] * rf["shape"][1] for rf in st["refit"]}
    flop = sum(2.0 * R * T * K * n for T in tmpl.values()) * n_fs
    exe = sum(2.0 * (-(-R // 64) * 64) * (-(-T // 64) * 64) * K * npad for T in tmpl.values()) * n_fs
    sec = (kms["fs_refit"] + kms.get("hd_fs_refit", 0.0)) * 1e-3
    line = {"metric": "realizations/sec of free_spectrum with a power-law and a turnover refit (67-psr ng15 "
                      "GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"free spectrum (K={K} bins, {m.n_amp} log10 rho, uncorrelated + HD) + refit "
                        + ", ".join(f"{k} ({T} templates)" for k, T in tmpl.items()),
            "kernels_ms_per_step": kms,
            "fs_refit": {"kernel": "fs_refit_kernel (Y^2 W GEMM on DMMA, W formed on the fly), all models",
                         "ms_per_step": sec * 1e3, "algorithmic_flop": flop, "executed_flop": exe,
                         "TFLOPs_algorithmic": flop / sec / 1e12, "TFLOPs_executed": exe / sec / 1e12,
                         "frac_of_67_TFLOPs_executed": exe / sec / 1e12 / 67.0},
            "setup_s": setup_s, "refit_statics_s": st["refit_setup_s"], "fs_statics_s": st["setup_s"],
            "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

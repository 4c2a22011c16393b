#!/usr/bin/env python
"""Benchmark of the factorised free-spectrum likelihood: the workload of bench_curn.py (bench.py's config 2: 67-pulsar
ng15-full EFAC/EQUAD + ECORR + red noise + HD GWB, with ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar) with
``set_free_spectrum(orf="hd")`` at its defaults (K = 14 bins, 121 log10 rho points, uncorrelated and HD models).  Prints
one JSON line.

    python bench_fs.py --steps K --warmup W [--nreal R]

A step = ``free_spectrum(R)``: R realizations generated (pre-fit; the marginalised timing model needs no fit) and
reduced to the per-realization, per-bin likelihood summaries of both models on the device.  ``value`` = realizations/s
of the whole step; ``kernels_ms_per_step`` = per-kernel ms per step from CUDA events around every launch in a second
pass of the same steps; ``fs_grid`` = the algorithmic flop of one model, 2 R K n (n + NR) with n = 2 n_psr, the flop
fs_grid_kernel executes (padded to 64-realization blocks, n2p gathered columns, np eigen-rows and 64-point amplitude
blocks), and the achieved TFLOP/s of both against the data-sheet 67 TFLOP/s of fp64 tensor cores; ``setup_s`` = batch +
recipe + plan + compile, of which ``fs_statics_s`` is the free spectrum's host statics; ``V_bytes`` = the device bytes
of V of both models.  The card name and power limit are read with a read-only nvidia-smi query in the same run.  Writes
nothing into the tree.
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
    args = parse(parser())
    b, kind, t0 = timing_model_batch(args)
    b.set_free_spectrum(orf="hd")
    b.compile()
    setup_s = time.perf_counter() - t0
    R = args.nreal
    ms, kms = timed_statistic(b.free_spectrum, R, args.steps, args.warmup)
    st = b.compile()["fs"]
    m = st["fs"]
    n, K, NR = 2 * b.n_psr, m.n_bin, m.n_amp
    flop = 2.0 * R * K * n * (n + NR)                                         # one model
    n_ab = -(-NR // 64)
    exe = 2.0 * (-(-R // 64) * 64) * K * n_ab * m.np * (m.n2p + 64)            # one model, as executed
    sec = (kms["fs_grid"] + kms["hd_fs_grid"]) * 1e-3 / 2                      # per model
    line = {"metric": "realizations/sec of free_spectrum (67-psr ng15 GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"free spectrum (K={K} bins, {NR} log10 rho, uncorrelated + HD)",
            "kernels_ms_per_step": kms,
            "fs_grid": {"kernel": "fs_grid_kernel (gathered two-GEMM chain on DMMA), per model",
                        "ms_per_step": sec * 1e3, "algorithmic_flop": flop, "executed_flop": exe,
                        "TFLOPs_algorithmic": flop / sec / 1e12, "TFLOPs_executed": exe / sec / 1e12,
                        "frac_of_67_TFLOPs_executed": exe / sec / 1e12 / 67.0},
            "setup_s": setup_s, "fs_statics_s": st["setup_s"], "V_bytes": st["nbytes"], "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

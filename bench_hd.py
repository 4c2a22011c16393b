#!/usr/bin/env python
"""Benchmark of the HD likelihood: the workload of bench_curn.py (bench.py's config 2: 67-pulsar ng15-full EFAC/EQUAD +
ECORR + red noise + HD GWB, ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar, ``set_curn_likelihood()`` at
its defaults: K = 14, 97 log10 A x 57 gamma points) plus ``set_hd_likelihood()``.  Prints one JSON line.

    python bench_hd.py --steps K --warmup W [--nreal R]

A step = ``curn_likelihood(R)``: R realizations generated (pre-fit) and reduced to the CURN and HD likelihood summaries
on the device.  ``value`` = realizations/s of the whole step; ``kernels_ms_per_step`` = per-kernel ms per step from
CUDA events around every launch in a second pass of the same steps; ``hd_grid`` = the achieved TFLOP/s of the two-GEMM
chain at the algorithmic 2 R Ng N (N + NA) flop (N = n_psr 2K) and at the executed 2 R Ng np (n_psr ncp + NAp) flop (the
kernel's padded shapes), and their fraction of the data-sheet 67 TFLOP/s of fp64 tensor cores; ``hd_statics_s`` = the
HD likelihood's host statics, ``hd_V_bytes`` = the device bytes of V.  The card name and power limit are read with a
read-only nvidia-smi query in the same run.  Writes nothing into the tree.
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
    b.set_curn_likelihood()
    b.set_hd_likelihood()
    b.compile()
    setup_s = time.perf_counter() - t0
    R = args.nreal
    ms, kms = timed_statistic(b.curn_likelihood, R, args.steps, args.warmup)
    st = b.compile()["curn"]
    m, hm = st["curn"], st["hd"]["model"]
    nap = 64 if m.n_amp <= 64 else 128 if m.n_amp <= 128 else 256
    flop = 2.0 * R * m.n_gamma * hm.n * (hm.n + m.n_amp)
    flop_x = 2.0 * R * m.n_gamma * hm.np * (b.n_psr * m.ncp + nap)
    sec = kms["hd_grid"] * 1e-3
    line = {"metric": "realizations/sec of curn_likelihood with the HD likelihood (67-psr ng15 GWB+RN+ECORR, spin + "
                      "JUMPs marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"CURN and HD likelihood (K={m.nc // 2}, N={hm.n}, {m.n_amp} log10 A x {m.n_gamma} gamma)",
            "kernels_ms_per_step": kms,
            "hd_grid": {"kernel": "hd_grid_kernel (two-GEMM chain on DMMA)", "ms_per_step": kms["hd_grid"],
                        "algorithmic_flop": flop, "TFLOPs": flop / sec / 1e12, "frac_of_67_TFLOPs": flop / sec / 67e12,
                        "executed_flop": flop_x, "executed_TFLOPs": flop_x / sec / 1e12,
                        "executed_frac_of_67_TFLOPs": flop_x / sec / 67e12},
            "setup_s": setup_s, "curn_statics_s": st["setup_s"], "hd_statics_s": st["hd"]["out"]["hd_setup_s"],
            "hd_V_bytes": int(st["hd"]["arrays"]["V"].numel() * 8), "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

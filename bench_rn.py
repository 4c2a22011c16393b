#!/usr/bin/env python
"""Benchmark of the single-pulsar red-noise likelihood: the workload of bench_curn.py (bench.py's config 2: 67-pulsar
ng15-full EFAC/EQUAD + ECORR + red noise + HD GWB, with ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar) with
``set_red_noise_likelihood()`` at its defaults (K = 30 on each pulsar's span, 97 log10 A x 57 gamma points).  Prints one
JSON line.

    python bench_rn.py --steps K --warmup W [--nreal R]

A step = ``red_noise_likelihood(R)``: R realizations generated (pre-fit; the marginalised timing model needs no fit) and
reduced to the per-realization, per-pulsar likelihood summaries on the device.  ``value`` = realizations/s of the whole
step; ``kernels_ms_per_step`` = per-kernel ms per step from CUDA events around every launch in a second pass of the same
steps; ``rn_grid`` = the achieved TFLOP/s of the two-GEMM chain at the algorithmic 2 R Ng P nc (nc + NA) flop and its
fraction of the data-sheet 67 TFLOP/s of fp64 tensor cores; ``setup_s`` = batch + recipe + plan + compile, of which
``rn_statics_s`` is the red-noise likelihood's host statics.  The card name and power limit are read with a read-only
nvidia-smi query in the same run.  Writes nothing into the tree.
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
    b.set_red_noise_likelihood()
    b.compile()
    setup_s = time.perf_counter() - t0
    R = args.nreal
    ms, kms = timed_statistic(b.red_noise_likelihood, R, args.steps, args.warmup)
    st = b.compile()["rn"]
    m = st["rn"]
    flop = 2.0 * R * m.n_gamma * b.n_psr * m.nc * (m.nc + m.n_amp)
    tflops = flop / (kms["rn_grid"] * 1e-3) / 1e12
    line = {"metric": "realizations/sec of red_noise_likelihood (67-psr ng15 GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"red-noise likelihood (K={m.nc // 2} per pulsar, {m.n_amp} log10 A x {m.n_gamma} gamma)",
            "kernels_ms_per_step": kms,
            "rn_grid": {"kernel": "rn_grid_kernel (two-GEMM chain on DMMA)", "ms_per_step": kms["rn_grid"],
                        "algorithmic_flop": flop, "TFLOPs": tflops, "frac_of_67_TFLOPs": tflops / 67.0},
            "setup_s": setup_s, "rn_statics_s": st["setup_s"], "rn_statics_share": st["setup_s"] / setup_s,
            "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Benchmark of the anisotropy statistics of the optimal statistic: the ``bench_os.py`` workload (bench.py's config 2,
67-pulsar ng15-full, timing model marginalised, ``set_optimal_statistic()`` at its defaults) with
``set_os_anisotropy(lmax=L, nside=N)`` (default lmax 6, nside 8).  Prints one JSON line.

    python bench_aniso.py --steps K --warmup W [--nreal R] [--lmax L] [--nside N]

A step = ``optimal_statistic(R)``: R realizations generated and reduced on the device to the optimal statistic, the
fitted c_lm, the anisotropy chi^2 and the radiometer map's max and argmax (the map itself is not kept).  ``value`` =
realizations/s of the whole step; ``kernels_ms_per_step`` = per-kernel ms per step from CUDA events around every launch
in a second pass of the same steps; ``os_aniso`` = the GEMM's achieved TFLOP/s at the algorithmic 2 R n_pairs n_col
flop against the data-sheet 67 TFLOP/s of fp64 tensor cores, the bytes of V and the anisotropy statics' host time.
The card name and power limit are read with a read-only nvidia-smi query in the same run.  Writes nothing into the tree.
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
    ap = parser()
    ap.add_argument("--lmax", type=int, default=6)
    ap.add_argument("--nside", type=int, default=8)
    args = parse(ap)

    b, kind, t0 = timing_model_batch(args)
    b.set_optimal_statistic()
    b.set_os_anisotropy(lmax=args.lmax, nside=args.nside)
    b.compile()
    setup_s = time.perf_counter() - t0
    R = args.nreal
    ms, kms = timed_statistic(b.optimal_statistic, R, args.steps, args.warmup)
    st = b.compile()["os"]
    an = st["aniso"]
    kd, ncol = int(an["model"].kd), an["n_col"]
    flop = 2.0 * R * kd * ncol
    tflops = flop / (kms["os_aniso_gemm"] * 1e-3) / 1e12
    line = {"metric": "realizations/sec of optimal_statistic + anisotropy (67-psr ng15 GWB+RN+ECORR, spin + JUMPs "
                      "marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"optimal statistic (K=14, templates {st['names']}, {st['n_pairs']} pairs) + anisotropy "
                        f"(lmax {args.lmax}: {an['n_lm']} c_lm + {an['n_z']} z; nside {args.nside}: {an['n_sky']} pixels)",
            "kernels_ms_per_step": kms,
            "os_aniso": {"kernels": "os_null_prepare_kernel + os_null_gemm_kernel (DMMA) + os_aniso_reduce_kernel",
                         "kd": kd, "n_col": ncol, "ms_per_step": kms["os_aniso_prepare"] + kms["os_aniso_gemm"] +
                         kms["os_aniso_reduce"], "gemm_ms_per_step": kms["os_aniso_gemm"], "gemm_flop": flop,
                         "gemm_TFLOPs": tflops, "frac_of_67_TFLOPs": tflops / 67.0,
                         "V_bytes": int(an["dev"]["V"].numel()) * 8, "aniso_statics_s": an["out"]["aniso_setup_s"]},
            "setup_s": setup_s, "os_statics_s": st["setup_s"], "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Benchmark of the optimal statistic: bench.py's metric workload (config 2: 67-pulsar ng15-full EFAC/EQUAD + ECORR +
red noise + HD GWB) with ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar and ``set_optimal_statistic()`` at
its defaults (K = 14, HD + monopole + dipole).  Prints one JSON line.

    python bench_os.py --steps K --warmup W [--nreal R]

A step = ``optimal_statistic(R)``: R realizations generated (pre-fit; the marginalised timing model needs no fit) and
reduced to A2 / S/N / A2_mc on the device.  ``value`` = realizations/s of the whole step; ``kernels_ms_per_step`` =
per-kernel ms per step from CUDA events around every launch in a second pass of the same steps; ``os_project`` = the
achieved bandwidth of the tile GEMM at the algorithmic 8 B per output (one fp64 residual read per TOA and
realization) and its fraction of the data-sheet 3.35 TB/s; ``setup_s`` = batch + recipe + plan + compile, of which
``os_statics_s`` is the optimal statistic's host statics.  The card name and power limit are read with a read-only
nvidia-smi query in the same run.  Writes nothing into the tree.

    python bench_os.py --null {phase_shift,sky_scramble} [--n-null N]

adds ``set_os_null(method, n=N)`` (default 1024; HD template) to the same workload: the step then also returns each
realization's null count and p-value, and the line gains ``os_null``: the GEMM's achieved TFLOP/s at the algorithmic
2 R (N + 1) Kd flop against the data-sheet 67 TFLOP/s of fp64 tensor cores, V's bytes and the null statics' host time.
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
    ap.add_argument("--null", default=None, choices=["phase_shift", "sky_scramble"])
    ap.add_argument("--n-null", type=int, default=1024)
    args = parse(ap)

    hbm, how = bench.peaks()
    b, kind, t0 = timing_model_batch(args)
    b.set_optimal_statistic()
    if args.null:
        b.set_os_null(args.null, n=args.n_null)
    b.compile()
    setup_s = time.perf_counter() - t0
    R = args.nreal
    ms, kms = timed_statistic(b.optimal_statistic, R, args.steps, args.warmup)
    gbps = 8.0 * b.n_toa_total * R / (kms["os_project"] * 1e-3) / 1e9
    st = b.compile()["os"]
    line = {"metric": "realizations/sec of optimal_statistic (67-psr ng15 GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"optimal statistic (K=14, templates {st['names']}, {st['n_pairs']} pairs)",
            "kernels_ms_per_step": kms,
            "os_project": {"kernel": "os_project_kernel (tile GEMM on DMMA)", "ms_per_step": kms["os_project"],
                           "algorithmic_bytes_per_output": 8, "algorithmic_GBps": gbps, "frac": gbps / hbm, "peak": hbm,
                           "peak_source": how},
            "setup_s": setup_s, "os_statics_s": st["setup_s"], "card": card()}
    if args.null:
        nl = st["null"]
        kd, ncol = int(nl["model"].kd), nl["n_col"]
        tflops = 2.0 * R * ncol * kd / (kms["os_null_gemm"] * 1e-3) / 1e12
        line["metric"] = line["metric"].replace("optimal_statistic", f"optimal_statistic + {args.null} null")
        line["workload"] += f" + {args.null} null of the HD S/N ({args.n_null} columns + the template, Kd = {kd})"
        line["os_null"] = {"method": args.null, "n": args.n_null, "kd": kd, "kernel": "os_null_gemm_kernel (DMMA)",
                           "gemm_ms_per_step": kms["os_null_gemm"], "gemm_flop": 2.0 * R * ncol * kd,
                           "gemm_TFLOPs": tflops, "frac_of_67_TFLOPs": tflops / 67.0,
                           "V_bytes": int(nl["dev"]["V"].numel()) * 8, "U_bytes_per_chunk": int(b._scratch_bufs["os_null_U"].numel()) * 8,
                           "null_statics_s": nl["setup_s"]}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

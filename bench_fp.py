#!/usr/bin/env python
"""Benchmark of the Fp-statistic: bench.py's metric workload (config 2: 67-pulsar ng15-full EFAC/EQUAD + ECORR + red
noise + HD GWB) with ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar and
``set_fp_statistic(n_freqs=N, log10_A_common=<the injected GWB amplitude>)`` (the background modelled as noise, as a
continuous-wave search does).  Prints one JSON line.

    python bench_fp.py --steps K --warmup W [--nreal R] [--n-freqs N]

A step = ``fp_statistic(R)``: R realizations generated (pre-fit; the marginalised timing model needs no fit) and reduced
to Fp, max_f Fp, its argmax and the single-frequency false-alarm probabilities on the device.  ``value`` =
realizations/s of the whole step; ``kernels_ms_per_step`` = per-kernel ms per step from CUDA events around every launch
in a second pass of the same steps; ``fp_project`` = the GEMM's achieved TFLOP/s at the algorithmic 2 R (sum_a n_a) 2 Nf
flop against the data-sheet 67 TFLOP/s of fp64 tensor cores; ``Ct_bytes`` = the device bytes of the whitened basis;
``setup_s`` = batch + recipe + plan + compile, of which ``fp_statics_s`` is the Fp-statistic's host statics.  The card
name and power limit are read with a read-only nvidia-smi query in the same run.  Writes nothing into the tree.
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

FP64_TC_PEAK = 67.0   # TFLOP/s, H100 SXM data sheet (not measured)


def main():
    ap = parser()
    ap.add_argument("--n-freqs", type=int, default=100)
    args = parse(ap)

    b, kind, t0 = timing_model_batch(args)
    gw_log10_A = -14.6733                                   # the GWB amplitude config 2 injects (synthetic.ng15_recipe)
    b.set_fp_statistic(n_freqs=args.n_freqs, log10_A_common=gw_log10_A)
    st = b.compile()["fp"]
    setup_s = time.perf_counter() - t0
    R = args.nreal
    ms, kms = timed_statistic(b.fp_statistic, R, args.steps, args.warmup)
    flop = 2.0 * R * b.n_toa_total * 2 * args.n_freqs
    tflops = flop / (kms["fp_project"] * 1e-3) / 1e12
    line = {"metric": "realizations/sec of fp_statistic (67-psr ng15 GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"Fp-statistic (Nf={args.n_freqs} at k/Tspan, common process log10_A={gw_log10_A} as noise)",
            "kernels_ms_per_step": kms,
            "fp_project": {"kernel": "fp_project_kernel (DMMA, one CTA per pulsar x 64 realizations x 64 columns)",
                           "ms_per_step": kms["fp_project"], "flop": flop, "TFLOPs": tflops,
                           "frac_of_67_TFLOPs": tflops / FP64_TC_PEAK, "peak_source": "H100 SXM data sheet (not measured)"},
            "Ct_bytes": int(st["Ct"].numel()) * 8, "setup_s": setup_s, "fp_statics_s": st["setup_s"], "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

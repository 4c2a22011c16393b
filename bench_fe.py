#!/usr/bin/env python
"""Benchmark of the Fe-statistic: the ``bench_fp.py`` step (config 2 of bench.py, 67-pulsar ng15-full EFAC/EQUAD + ECORR +
red noise + HD GWB, ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar, ``set_fp_statistic(n_freqs=N,
log10_A_common=<the injected GWB amplitude>)``) plus ``set_fe_statistic(nside=NSIDE)``.  Prints one JSON line.

    python bench_fe.py --steps K --warmup W [--nreal R] [--n-freqs N] [--nside 8|16]

A step = ``fp_statistic(R)`` without maps: R realizations generated and reduced to Fp and to the Fe sky maxima
(``Fe_fmax``, ``Fe_max`` and their argmaxes) on the device.  ``value`` = realizations/s of the whole step;
``kernels_ms_per_step`` = per-kernel ms per step from CUDA events around every launch in a second pass of the same steps;
``fe_sky`` = the sky GEMM's achieved TFLOP/s at the algorithmic 8 R Nf S P flop (4 outputs per (r, f, s), P
multiply-adds each) against the data-sheet 67 TFLOP/s of fp64 tensor cores; ``fe_statics_bytes`` = the device bytes of
L_a(f), the antenna layout and L4^-1; ``fe_statics_s`` = the host time of the Fe statics.  The card name and power limit
are read with a read-only nvidia-smi query in the same run.  Writes nothing into the tree.
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
    ap.add_argument("--nside", type=int, default=8, choices=[1, 2, 4, 8, 16, 32])
    args = parse(ap)

    b, kind, t0 = timing_model_batch(args)
    gw_log10_A = -14.6733                                   # the GWB amplitude config 2 injects (synthetic.ng15_recipe)
    b.set_fp_statistic(n_freqs=args.n_freqs, log10_A_common=gw_log10_A)
    b.set_fe_statistic(nside=args.nside)
    st = b.compile()["fp"]
    setup_s = time.perf_counter() - t0
    R, S = args.nreal, st["fe"]["n_sky"]
    ms, kms = timed_statistic(b.fp_statistic, R, args.steps, args.warmup)
    flop = 8.0 * R * args.n_freqs * S * b.n_psr
    tflops = flop / (kms["fe_sky"] * 1e-3) / 1e12
    line = {"metric": "realizations/sec of fp_statistic with the Fe sky search (67-psr ng15 GWB+RN+ECORR, spin + JUMPs "
                      "marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"Fp-statistic (Nf={args.n_freqs} at k/Tspan, common process log10_A={gw_log10_A} as noise) + "
                        f"Fe-statistic (HEALPix nside {args.nside}, S={S})",
            "kernels_ms_per_step": kms,
            "fe_sky": {"kernel": "fe_sky_kernel (DMMA, one CTA per 32 realizations x frequency walking the sky, fused "
                                 "1/2 |L4^-1 N4|^2 and max epilogue)",
                       "ms_per_step": kms["fe_sky"], "flop": flop, "TFLOPs": tflops,
                       "frac_of_67_TFLOPs": tflops / FP64_TC_PEAK, "peak_source": "H100 SXM data sheet (not measured)"},
            "fe_statics_bytes": int(st["fe"]["nbytes"]), "fe_statics_s": st["fe"]["setup_s"],
            "fp_statics_s": st["setup_s"], "setup_s": setup_s, "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

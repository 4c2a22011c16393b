#!/usr/bin/env python
"""Benchmark of the burst-with-memory search: config 2 of bench.py (67-pulsar ng15-full EFAC/EQUAD + ECORR + red noise +
HD GWB), ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar and ``set_bwm_statistic(n_epochs=T, nside=NSIDE,
log10_A_common=<the injected GWB amplitude>)``.  Prints one JSON line.

    python bench_bwm.py --steps K --warmup W [--nreal R] [--n-epochs T] [--nside 8|16]

A step = ``bwm_statistic(R)`` without maps: R realizations generated and reduced to the epoch x sky maxima, the strain
and polarisation at the maximum and the pulsar-term maxima on the device.  ``value`` = realizations/s of the whole step;
``kernels_ms_per_step`` = per-kernel ms per step from CUDA events around every launch in a second pass of the same
steps; ``bwm_sky`` = the sky GEMM's achieved TFLOP/s at the algorithmic 4 R T S P flop (2 outputs per (r, t, s), P
multiply-adds each) and ``bwm_project`` the projection's at 2 R sum(N_toa) T, both against the data-sheet 67 TFLOP/s of
fp64 tensor cores; ``bwm_statics_bytes`` = the device bytes of the whitened ramps, sqrt(m), the seen mask, the antenna
layouts and L2^-1; ``bwm_statics_s`` = the host time of the statics.  The card name and power limit are read with a
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

FP64_TC_PEAK = 67.0   # TFLOP/s, H100 SXM data sheet (not measured)


def main():
    ap = parser()
    ap.add_argument("--n-epochs", type=int, default=100)
    ap.add_argument("--nside", type=int, default=8, choices=[1, 2, 4, 8, 16, 32])
    args = parse(ap)

    b, kind, t0 = timing_model_batch(args)
    gw_log10_A = -14.6733                                   # the GWB amplitude config 2 injects (synthetic.ng15_recipe)
    b.set_bwm_statistic(n_epochs=args.n_epochs, nside=args.nside, log10_A_common=gw_log10_A)
    st = b.compile()["bwm"]
    setup_s = time.perf_counter() - t0
    R, S, T = args.nreal, st["n_sky"], st["n_t0"]
    ms, kms = timed_statistic(b.bwm_statistic, R, args.steps, args.warmup)
    flop_sky = 4.0 * R * T * S * b.n_psr
    flop_proj = 2.0 * R * b.n_toa_total * T
    tf_sky = flop_sky / (kms["bwm_sky"] * 1e-3) / 1e12
    tf_proj = flop_proj / (kms["bwm_project"] * 1e-3) / 1e12
    line = {"metric": "realizations/sec of bwm_statistic (67-psr ng15 GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"BWM search (T={T} epochs, HEALPix nside {args.nside}, S={S}, common process "
                        f"log10_A={gw_log10_A} as noise)",
            "kernels_ms_per_step": kms,
            "bwm_sky": {"kernel": "bwm_sky_kernel (DMMA, one CTA per 32 realizations x epoch pair walking the sky, fused "
                                  "1/2 |L2^-1 N2|^2 and max epilogue)",
                        "ms_per_step": kms["bwm_sky"], "flop": flop_sky, "TFLOPs": tf_sky,
                        "frac_of_67_TFLOPs": tf_sky / FP64_TC_PEAK, "peak_source": "H100 SXM data sheet (not measured)"},
            "bwm_project": {"kernel": "fp_project_kernel on the whitened ramps (DMMA, column j = epoch j)",
                            "ms_per_step": kms["bwm_project"], "flop": flop_proj, "TFLOPs": tf_proj,
                            "frac_of_67_TFLOPs": tf_proj / FP64_TC_PEAK,
                            "peak_source": "H100 SXM data sheet (not measured)"},
            "bwm_statics_bytes": int(st["nbytes"]), "bwm_statics_s": st["setup_s"], "setup_s": setup_s, "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

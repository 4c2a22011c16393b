#!/usr/bin/env python
"""Benchmark of the sine-Gaussian burst search: config 2 of bench.py (67-pulsar ng15-full EFAC/EQUAD + ECORR + red noise +
HD GWB), ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar and ``set_burst_statistic(nside=NSIDE,
log10_A_common=<the injected GWB amplitude>)`` with the default bank.  Prints one JSON line.

    python bench_burst.py --steps K --warmup W [--nreal R] [--nside 8|16]

A step = ``burst_statistic(R)`` without maps: R realizations generated and reduced to the template x sky maxima, the
amplitudes at the maximum and the per-pulsar transient maxima on the device.  ``value`` = realizations/s of the whole
step; ``kernels_ms_per_step`` = per-kernel ms per step from CUDA events around every launch in a second pass of the same
steps (``burst_project.g`` and ``burst_sky.g`` per template group g, and their sums); ``burst_project`` = its achieved
TFLOP/s at the algorithmic 2 R sum(window) 2 flop (two columns per template over the TOAs of its window) against the
data-sheet 67 TFLOP/s of fp64 tensor cores; ``burst_statics_bytes`` / ``burst_statics_s`` = the device bytes and host
seconds of the statics; ``burst_scratch_bytes`` = the per-pass scratch (N^-1 r, z, amplitudes, per-template maxima of
``PulsarBatch.BURST_ROWS`` realizations); ``dense_ct`` = what the dense alternative (whitened columns P_a^-1 W_j stored
as ``Ct`` and projected by ``ptar_fp_project``) would need, computed from shapes and not built.  The card name and power limit are read with a
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
    ap.add_argument("--nside", type=int, default=8, choices=[1, 2, 4, 8, 16, 32])
    args = parse(ap)

    b, kind, t0 = timing_model_batch(args)
    gw_log10_A = -14.6733                                   # the GWB amplitude config 2 injects (synthetic.ng15_recipe)
    b.set_burst_statistic(nside=args.nside, log10_A_common=gw_log10_A)
    pb = b.plan()["burst"]
    st = b.compile()["burst"]
    setup_s = time.perf_counter() - t0
    R, S, J = args.nreal, st["n_sky"], st["n_tmpl"]
    ms, kms = timed_statistic(b.burst_statistic, R, args.steps, args.warmup)
    for k in ("burst_project", "burst_sky"):
        kms[k] = sum(v for name, v in kms.items() if name.startswith(k + "."))
    win = int((pb["win"][..., 1] - pb["win"][..., 0]).sum())
    flop_proj = 2.0 * R * win * 2
    flop_dense = 2.0 * R * b.n_toa_total * 2 * J
    rank = pb["rank"].astype(float)
    ntoa = [float(n) for n in b.ntoa]
    tf_proj = flop_proj / (kms["burst_project"] * 1e-3) / 1e12
    line = {"metric": "realizations/sec of burst_statistic (67-psr ng15 GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"burst search (default bank: J={J} templates, HEALPix nside {args.nside}, S={S}, common process "
                        f"log10_A={gw_log10_A} as noise)",
            "kernels_ms_per_step": kms,
            "burst_project": {"kernel": "burst_project_kernel (W generated per 64-TOA chunk, DMMA over each 16-template "
                                        "block's window union, H^T z and L^-1 epilogue)",
                              "ms_per_step": kms["burst_project"], "flop": flop_proj, "TFLOPs": tf_proj,
                              "frac_of_67_TFLOPs": tf_proj / FP64_TC_PEAK, "sum_window_toas": win,
                              "windowed_over_dense_flop": flop_proj / flop_dense,
                              "peak_source": "H100 SXM data sheet (not measured)"},
            "burst_statics_bytes": int(st["nbytes"]), "burst_statics_s": st["setup_s"],
            "burst_scratch_bytes": int(st["scratch_bytes"]), "burst_device_bytes": int(st["nbytes"] + st["scratch_bytes"]),
            "dense_ct": {"built": False, "bytes": int(pb["dense_ct_bytes"]), "projection_flop": flop_dense,
                         "host_flop": float(sum(2 * r * n * 2 * J for r, n in zip(rank, ntoa)))},
            "setup_s": setup_s, "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

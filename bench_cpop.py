#!/usr/bin/env python
"""Benchmark of per-realization common-process populations: the ``bench_curn.py`` step (config 2 of bench.py, 67-pulsar
ng15-full EFAC/EQUAD + ECORR + red noise + HD GWB, ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar,
``set_curn_likelihood()`` at its defaults) with ``set_hd_likelihood()``, with and without ``set_common_population()`` at
its defaults (HD power law, K = 14, the CURN grid's ranges as priors).  Prints one JSON line.

    python bench_cpop.py --steps K --warmup W [--nreal R] [--components K]

A step = ``curn_likelihood(R)``.  The batch without a population and the batch with one are timed alternately in the
same run, ``rounds`` times each (best round kept); ``value`` = realizations/s of the step with the population, ``plain``
the same without it, and ``kernels_ms_per_step`` the per-kernel ms per step of each from CUDA events around every
launch.  ``cpop_add`` reports the add kernel's achieved bytes/s at its algorithmic 16 B per (TOA, realization) -- one
read and one write of every row element -- against the data-sheet 3.35 TB/s of HBM3, and which bound applies: memory
when that share is at least a half, otherwise the fp64 work (2K sincos per slot per 32 realizations, 2K FMA per
element).  The card name and power limit are read with a read-only nvidia-smi query in the same run.  Writes nothing
into the tree.
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

HBM_PEAK = 3.35e12   # B/s, H100 SXM data sheet (not measured)


def main():
    ap = parser()
    ap.add_argument("--components", type=int, default=14)
    ap.add_argument("--rounds", type=int, default=3)
    args = parse(ap)
    batches = {}
    for name in ("plain", "cpop"):
        b, kind, t0 = timing_model_batch(args)
        b.set_curn_likelihood()
        b.set_hd_likelihood()
        if name == "cpop":
            b.set_common_population(components=args.components)
        b.compile()
        batches[name] = (b, time.perf_counter() - t0)
    R = args.nreal
    best = {}
    for _ in range(args.rounds):    # alternate the two batches in the same run
        for name, (b, _) in batches.items():
            ms, kms = timed_statistic(b.curn_likelihood, R, args.steps, args.warmup)
            if name not in best or ms < best[name][0]:
                best[name] = (ms, kms)
    b = batches["cpop"][0]
    kms = best["cpop"][1]
    nbytes = 16.0 * b.n_toa_total * R
    bps = nbytes / (kms["cpop_add"] * 1e-3)
    frac = bps / HBM_PEAK
    K = args.components
    line = {"metric": f"realizations/sec of curn_likelihood with the HD likelihood and a common-process population (HD "
                      f"power law, K={K}) per realization (67-psr ng15 GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (best["cpop"][0] * 1e-3), "unit": "realizations/s",
            "ms_per_step": best["cpop"][0] / args.steps,
            "plain": {"value": R * args.steps / (best["plain"][0] * 1e-3), "ms_per_step": best["plain"][0] / args.steps},
            "cpop_over_plain": best["cpop"][0] / best["plain"][0],
            "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "realizations_per_step": R,
            "components": K, "sum_n_toa": b.n_toa_total,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        "CURN likelihood (defaults) + HD likelihood + "
                        f"set_common_population(components={K}) at its default priors",
            "kernels_ms_per_step": {"plain": best["plain"][1], "cpop": kms},
            "cpop_add": {"kernel": "cpop_add_kernel (thread per TOA slot, 2K basis values in registers, 32 realizations "
                                   "per CTA, coefficient records in shared memory, one read-modify-write per row element)",
                         "ms_per_step": kms["cpop_add"], "bytes": nbytes, "bytes_per_s": bps,
                         "frac_of_3.35_TBs": frac, "bound": "memory" if frac >= 0.5 else "compute (fp64)",
                         "algorithmic_fma": 2.0 * K * b.n_toa_total * R,
                         "peak_source": "H100 SXM data sheet (not measured)"},
            "cpop_draw_ms_per_step": kms["cpop_draw"],
            "setup_s": {k: v[1] for k, v in batches.items()}, "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Benchmark of per-realization continuous-wave populations: the ``bench_fe.py`` step (config 2 of bench.py, 67-pulsar
ng15-full EFAC/EQUAD + ECORR + red noise + HD GWB, ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar,
``set_fp_statistic(n_freqs=100, log10_A_common=<the injected GWB amplitude>)``, ``set_fe_statistic(nside=8)``) with and
without ``set_cw_population(n_sources=N)`` at its default priors.  Prints one JSON line.

    python bench_cwpop.py --steps K --warmup W [--nreal R] [--n-sources N] [--mode mono|evolve]

A step = ``fp_statistic(R)`` without maps.  The batch without a population and the batch with one are timed alternately
in the same run, ``rounds`` times each (best round kept); ``value`` = realizations/s of the step with the population,
``plain`` the same without it, and ``kernels_ms_per_step`` the per-kernel ms per step of each from CUDA events around
every launch.  ``cwpop_add`` reports the add kernel's achieved bytes/s at its algorithmic 16 B per (TOA, realization) --
one read and one write of every row element -- against the data-sheet 3.35 TB/s of HBM3, and which bound applies: memory
when that share is at least a half, otherwise the fp64 transcendentals per (TOA, realization, source).  The card name
and power limit are read with a read-only nvidia-smi query in the same run.  Writes nothing into the tree.
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
    ap.add_argument("--n-sources", type=int, default=1)
    ap.add_argument("--mode", default="mono", choices=["mono", "evolve"])
    ap.add_argument("--rounds", type=int, default=3)
    args = parse(ap)
    gw_log10_A = -14.6733                                   # the GWB amplitude config 2 injects (synthetic.ng15_recipe)
    batches = {}
    for name in ("plain", "cwpop"):
        b, kind, t0 = timing_model_batch(args)
        b.set_fp_statistic(n_freqs=100, log10_A_common=gw_log10_A)
        b.set_fe_statistic(nside=8)
        if name == "cwpop":
            b.set_cw_population(n_sources=args.n_sources, evolve=args.mode == "evolve")
        b.compile()
        batches[name] = (b, time.perf_counter() - t0)
    R = args.nreal
    best = {}
    for _ in range(args.rounds):    # alternate the two batches in the same run
        for name, (b, _) in batches.items():
            ms, kms = timed_statistic(b.fp_statistic, R, args.steps, args.warmup)
            if name not in best or ms < best[name][0]:
                best[name] = (ms, kms)
    b = batches["cwpop"][0]
    kms = best["cwpop"][1]
    nbytes = 16.0 * b.n_toa_total * R
    bps = nbytes / (kms["cwpop_add"] * 1e-3)
    frac = bps / HBM_PEAK
    line = {"metric": f"realizations/sec of fp_statistic with the Fe sky search and a {args.n_sources}-source CW population "
                      f"({args.mode}) per realization (67-psr ng15 GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (best["cwpop"][0] * 1e-3), "unit": "realizations/s",
            "ms_per_step": best["cwpop"][0] / args.steps,
            "plain": {"value": R * args.steps / (best["plain"][0] * 1e-3), "ms_per_step": best["plain"][0] / args.steps},
            "cwpop_over_plain": best["cwpop"][0] / best["plain"][0],
            "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "realizations_per_step": R,
            "n_sources": args.n_sources, "mode": args.mode, "sum_n_toa": b.n_toa_total,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"Fp-statistic (Nf=100, common process log10_A={gw_log10_A} as noise) + Fe-statistic (nside 8) + "
                        f"set_cw_population(n_sources={args.n_sources}, evolve={args.mode == 'evolve'}) at its default priors",
            "kernels_ms_per_step": {"plain": best["plain"][1], "cwpop": kms},
            "cwpop_add": {"kernel": "cwpop_add_kernel (thread per TOA slot, 16 realizations per CTA, (r, s) records in "
                                    "shared memory, one read-modify-write per row element)",
                          "ms_per_step": kms["cwpop_add"], "bytes": nbytes, "bytes_per_s": bps,
                          "frac_of_3.35_TBs": frac, "bound": "memory" if frac >= 0.5 else "compute (fp64 transcendentals)",
                          "peak_source": "H100 SXM data sheet (not measured)"},
            "cwpop_draw_ms_per_step": kms["cwpop_draw"],
            "setup_s": {k: v[1] for k, v in batches.items()}, "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

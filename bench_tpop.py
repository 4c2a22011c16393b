#!/usr/bin/env python
"""Benchmark of per-realization transient populations: the ``bench_bwm.py`` or ``bench_burst.py`` step (config 2 of
bench.py, 67-pulsar ng15-full EFAC/EQUAD + ECORR + red noise + HD GWB, ``set_timing_model(i, poly=2, jumps="f")`` on every
pulsar, the search at its default grid with ``log10_A_common=<the injected GWB amplitude>``) with and without
``set_bwm_population`` / ``set_burst_population(n_sources=N)`` at its default priors.  Prints one JSON line.

    python bench_tpop.py --family bwm|burst --steps K --warmup W [--nreal R] [--n-sources N]

A step = ``bwm_statistic(R)`` / ``burst_statistic(R)`` without maps.  The batch without a population and the batch with
one are timed alternately in the same run, ``rounds`` times each (best round kept); ``value`` = realizations/s of the
step with the population, ``plain`` the same without it, and ``kernels_ms_per_step`` the per-kernel ms per step of each
from CUDA events around every launch.  ``add`` reports the add kernel's achieved bytes/s at its algorithmic 16 B per
(TOA, realization) -- one read and one write of every row element, although the kernel skips the elements whose terms
are all 0 -- against the data-sheet 3.35 TB/s of HBM3; ``draw_ms_per_step`` is the draw kernel's time.  ``detection``
(one source per realization) splits the population's amplitude prior into quarters and gives, per quarter, the share of
realizations whose search maximum exceeds the 99th percentile of the plain batch's: the prior's span from undetectable
to loud.  The card name and power limit are read with a read-only nvidia-smi query in the same run.  Writes nothing into
the tree.
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
    import numpy as np
    ap = parser()
    ap.add_argument("--family", default="bwm", choices=["bwm", "burst"])
    ap.add_argument("--n-sources", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    args = parse(ap)
    gw_log10_A = -14.6733                                   # the GWB amplitude config 2 injects (synthetic.ng15_recipe)
    fam, key = args.family, args.family + "pop"
    batches = {}
    for name in ("plain", key):
        b, kind, t0 = timing_model_batch(args)
        if fam == "bwm":
            b.set_bwm_statistic(log10_A_common=gw_log10_A)
        else:
            b.set_burst_statistic(log10_A_common=gw_log10_A)
        if name == key:
            (b.set_bwm_population if fam == "bwm" else b.set_burst_population)(n_sources=args.n_sources)
        b.compile()
        batches[name] = (b, time.perf_counter() - t0)
    stat = {n: (b.bwm_statistic if fam == "bwm" else b.burst_statistic) for n, (b, _) in batches.items()}
    R = args.nreal
    best = {}
    for _ in range(args.rounds):    # alternate the two batches in the same run
        for name in batches:
            ms, kms = timed_statistic(stat[name], R, args.steps, args.warmup)
            if fam == "burst":
                for k in ("burst_project", "burst_sky"):
                    kms[k] = sum(v for n, v in kms.items() if n.startswith(k + "."))
            if name not in best or ms < best[name][0]:
                best[name] = (ms, kms)
    b = batches[key][0]
    kms = best[key][1]
    nbytes = 16.0 * b.n_toa_total * R
    bps = nbytes / (kms[key + "_add"] * 1e-3)
    line = {"metric": f"realizations/sec of {fam}_statistic with a {args.n_sources}-source {fam} population per "
                      "realization (67-psr ng15 GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (best[key][0] * 1e-3), "unit": "realizations/s",
            "ms_per_step": best[key][0] / args.steps,
            "plain": {"value": R * args.steps / (best["plain"][0] * 1e-3), "ms_per_step": best["plain"][0] / args.steps},
            "pop_over_plain": best[key][0] / best["plain"][0],
            "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "realizations_per_step": R,
            "family": fam, "n_sources": args.n_sources, "sum_n_toa": b.n_toa_total,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"{fam} search at its default grid (common process log10_A={gw_log10_A} as noise) + "
                        f"set_{fam}_population(n_sources={args.n_sources}) at its default priors",
            "kernels_ms_per_step": {"plain": best["plain"][1], key: kms},
            "add": {"kernel": f"tpop_add_kernel<{fam.upper()}> (thread per TOA slot, 16 realizations per CTA, (r, s) "
                              "records in shared memory, one read-modify-write per row element with a non-zero term)",
                    "ms_per_step": kms[key + "_add"], "bytes": nbytes, "bytes_per_s": bps,
                    "frac_of_3.35_TBs": bps / HBM_PEAK, "peak_source": "H100 SXM data sheet (not measured)"},
            "draw_ms_per_step": kms[key + "_draw"],
            "setup_s": {k: v[1] for k, v in batches.items()}, "card": card()}
    if args.n_sources == 1:
        mx = "bwm_max" if fam == "bwm" else "B_max"
        seed = bench.SEED + 1
        noise = stat["plain"](R, seed=seed)[mx].cpu().numpy()
        got = stat[key](R, seed=seed)[mx].cpu().numpy()
        prm = (b.bwm_population_params if fam == "bwm" else b.burst_population_params)(R, seed=seed)
        la = prm["log10_strain" if fam == "bwm" else "log10_amp"][:, 0].cpu().numpy()
        thr = float(np.quantile(noise, 0.99))
        edges = np.quantile(la, [0, 0.25, 0.5, 0.75, 1.0])
        q = np.clip(np.searchsorted(edges, la, side="right") - 1, 0, 3)
        line["detection"] = {"threshold_B": thr, "threshold": "99th percentile of the plain batch's maximum",
                             "log10_amp_quarters": [[float(edges[i]), float(edges[i + 1])] for i in range(4)],
                             "frac_above": [float(np.mean(got[q == i] > thr)) for i in range(4)]}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Benchmark of the per-frequency optimal statistic: the ``bench_os.py`` workload (bench.py's config 2, 67-pulsar
ng15-full, timing model marginalised, ``set_optimal_statistic()`` at its defaults) with ``set_os_per_frequency()``.
Prints one JSON line.

    python bench_pfos.py --steps K --warmup W [--nreal R]

A step = ``optimal_statistic(R)``: R realizations generated and reduced on the device to the broadband optimal
statistic and, per GW frequency, phi_ok, its S/N and the multiple-component estimate (pair values are not kept).
``value`` = realizations/s of the whole step; ``kernels_ms_per_step`` = per-kernel ms per step from CUDA events around
every launch in a second pass of the same steps; ``os_pf`` = the kernel's algorithmic bytes (the projections X read,
R P nc 8 B) and flop (R K n_pairs (3 + 2 n_orf)), its achieved GB/s and that rate's share of the data-sheet
3.35 TB/s.  The card name and power limit are read with a read-only nvidia-smi query in the same run.  Writes nothing
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

HBM_GBS = 3350.0   # H100 SXM data sheet


def main():
    args = parse(parser())

    b, kind, t0 = timing_model_batch(args)
    b.set_optimal_statistic()
    b.set_os_per_frequency()
    b.compile()
    setup_s = time.perf_counter() - t0
    R = args.nreal
    ms, kms = timed_statistic(b.optimal_statistic, R, args.steps, args.warmup)
    st = b.compile()["os"]
    K, n_pairs, n_orf, P = st["pf"]["K"], st["n_pairs"], st["n_orf"], b.n_psr
    nbytes = 8.0 * R * P * 2 * K
    flop = float(R) * K * n_pairs * (3 + 2 * n_orf)
    gbps = nbytes / (kms["os_pf"] * 1e-3) / 1e9
    line = {"metric": "realizations/sec of optimal_statistic + per-frequency optimal statistic (67-psr ng15 "
                      "GWB+RN+ECORR, spin + JUMPs marginalised)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing model per pulsar (poly=2 + JUMPs of flag f) + "
                        f"optimal statistic (K={K}, templates {st['names']}, {n_pairs} pairs) + per-frequency optimal "
                        "statistic",
            "kernels_ms_per_step": kms,
            "os_pf": {"kernel": "os_pf_kernel", "ms_per_step": kms["os_pf"], "algorithmic_bytes": nbytes,
                      "algorithmic_flop": flop, "achieved_GBps": gbps, "frac_of_3350_GBps": gbps / HBM_GBS,
                      "GFLOPs": flop / (kms["os_pf"] * 1e-3) / 1e9, "pf_statics_s": st["pf"]["out"]["pf_setup_s"]},
            "setup_s": setup_s, "os_statics_s": st["setup_s"], "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

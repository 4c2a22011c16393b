#!/usr/bin/env python
"""Benchmark of chromatic noise in the generator: bench.py's config 2 (67-pulsar ng15-full EFAC/EQUAD + ECORR + red noise
+ HD GWB) with each epoch's sub-band TOAs spread evenly over the receiver band its backend flag names (430 MHz,
Rcvr_800, L-wide / Rcvr1_2, S-wide), a DM process (30 components) on every pulsar and a scattering process (idx 4,
30 components) on every third pulsar.  Prints one JSON line.

    python bench_chrom.py --steps K --warmup W [--nreal R]

A step = ``generate(R)``.  The plain batch (config 2 on the same TOAs) and the chromatic batch are timed alternately in
the same run, ``rounds`` times each; ``value`` = realizations/s of the chromatic step (best round), ``plain`` the same for
the plain step, and ``kernels_ms_per_step`` the per-kernel ms per step of each from CUDA events around every launch.
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
from bench_postfit import card, parse, parser  # noqa: E402


def main():
    import numpy as np
    import torch
    from pta_replicator_b200 import synthetic
    ap = parser()
    ap.add_argument("--rounds", type=int, default=3)
    args = parse(ap)
    torch.cuda.set_device(0)
    psrs, noise = synthetic.make_ng15_like(args.kind)
    synthetic.spread_subband_frequencies(psrs)
    t0 = time.perf_counter()
    plain = bench.make_batch("2", args, psrs_noise=(psrs, noise))[0]
    chrom = bench.make_batch("2", args, psrs_noise=(psrs, noise))[0]
    for i in range(chrom.n_psr):
        chrom.set_dm_noise(i, -13.5, 2.5, components=30)
        if i % 3 == 0:
            chrom.set_chromatic_noise(i, -14.0, 3.0, idx=4.0, components=30)
    chrom.compile()
    setup_s = time.perf_counter() - t0
    R = args.nreal
    best = {}
    for _ in range(args.rounds):    # alternate the two batches in the same run
        for name, b in (("plain", plain), ("chrom", chrom)):
            ms, kern, _ = bench.timed_steps(b, R, args.steps, args.warmup, 0)
            if name not in best or ms < best[name][0]:
                best[name] = (ms, {k: v["total_ms"] / args.steps for k, v in kern.items()})
    rate = {k: R * args.steps / (v[0] * 1e-3) for k, v in best.items()}
    st = chrom.compile()
    line = {"metric": "realizations/sec of generate with DM + scattering noise (67-psr ng15 GWB+RN+ECORR)",
            "value": rate["chrom"], "unit": "realizations/s", "ms_per_step": best["chrom"][0] / args.steps,
            "plain": {"value": rate["plain"], "ms_per_step": best["plain"][0] / args.steps},
            "chrom_over_plain": best["chrom"][0] / best["plain"][0],
            "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "realizations_per_step": R,
            "workload": bench.workload_name("2", args.kind, chrom) + " + sub-band frequencies over each backend's band, "
                        f"DM (30 comp) on {chrom.n_psr} psr + scattering (idx 4, 30 comp) on "
                        f"{int(sum(c is not None for c in chrom._chrom[1]['f']))} psr",
            "epochs": {"plain": int(plain.compile()["n_epochs"]), "chrom": int(st["n_epochs"])},
            "kernels_ms_per_step": {"plain": best["plain"][1], "chrom": best["chrom"][1]},
            "freq_MHz_range": [float(min(np.min(f) for f in chrom.freq)), float(max(np.max(f) for f in chrom.freq))],
            "setup_s": setup_s, "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

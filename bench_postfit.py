#!/usr/bin/env python
"""Benchmark of the post-fit path: bench.py's metric workload (config 2: 67-pulsar ng15-full EFAC/EQUAD + ECORR + red
noise + HD GWB) with ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar (phase offset + F0 + F1 and one JUMP
per backend flag), so every residual is post-fit.  Prints one JSON line.

    python bench_postfit.py --steps K --warmup W [--nreal R]

``value`` = realizations/s of the whole post-fit step; ``kernels`` = per-kernel ms per step from CUDA events around
every launch (``timing_reduce`` and ``timing_apply`` are the fit); ``projection`` = achieved bandwidth of the fit at
the algorithmic 16 B per fitted output (one read, one write; the two-kernel form moves 24 B) and its fraction of the
peak bench.py uses.  The card name and power limit are read with a read-only nvidia-smi query in the same run.
Writes nothing into the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True   # the tree may be read-only

import bench  # noqa: E402  (the metric workload and its timing helpers)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=10)
        name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception:  # noqa: BLE001
        return None


def parser():
    """The options of every benchmark on the timing-model workload (this one and the statistic benchmarks)."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--nreal", type=int, default=1000)
    ap.add_argument("--kind", default="full", choices=["full", "epoch"])
    ap.add_argument("--taylor-tol", type=float, default=1e-13)
    return ap


def parse(ap):
    """``ap``'s arguments; bench.make_batch's split, chunk and rc are off unless ``ap`` has an option for them."""
    return ap.parse_args(namespace=argparse.Namespace(split=False, chunk=0, rc=0))


def timing_model_batch(args):
    """bench.py's config-2 batch on device 0 with ``set_timing_model(i, poly=2, jumps="f")`` on every pulsar.  Returns
    (batch, kind, t0) with t0 the perf_counter reading after the pulsars are made and before the batch is built: the
    caller's setup clock, stopped after its own registrations and ``compile()``."""
    import torch
    from pta_replicator_b200 import synthetic
    torch.cuda.set_device(0)
    psrs_noise = synthetic.make_ng15_like(args.kind)
    t0 = time.perf_counter()
    b, _psrs, _noise, _s, kind = bench.make_batch("2", args, psrs_noise=psrs_noise)
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    return b, kind, t0


def timed_statistic(fn, R, steps, warmup):
    """Time ``fn(R, seed, real0, timers)`` (a statistic of R generated realizations): ``warmup`` untimed calls, ``steps``
    calls between two CUDA events, then ``steps`` more with per-launch timers.  Every call draws fresh realizations.
    Returns (ms of the event-timed calls, {kernel: ms per step} of the timed-launch pass)."""
    import numpy as np
    import torch

    def step(k, timers=None):
        fn(R, seed=bench.SEED, real0=4 * k * R, timers=timers)

    for k in range(warmup):
        step(k)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(steps):
        step(warmup + k)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    timers = {}
    for k in range(steps):
        step(warmup + steps + k, timers)
    torch.cuda.synchronize()
    per = {}
    for name, a, z in timers["events"]:
        per.setdefault(name, []).append(a.elapsed_time(z))
    return ms, {k: float(np.sum(v)) / steps for k, v in per.items()}


def main():
    ap = parser()
    ap.add_argument("--rc", type=int, default=0)
    ap.add_argument("--chunk", type=int, default=0)
    args = parse(ap)

    hbm, how = bench.peaks()
    b, kind, t0 = timing_model_batch(args)
    tm = b.plan()["tm"]
    b.compile()
    setup_s = time.perf_counter() - t0
    R = args.nreal
    ms, kern, _step = bench.timed_steps(b, R, args.steps, args.warmup, args.rc)
    kms = {k: v["total_ms"] / args.steps for k, v in kern.items()}
    proj_ms = kms["timing_reduce"] + kms["timing_apply"]
    n_fit = int(sum(b.ntoa[i] for i in range(b.n_psr) if tm["k"][i] > 0))
    gbps = 16.0 * n_fit * R / (proj_ms * 1e-3) / 1e9
    line = {"metric": "realizations/sec (67-psr ng15 GWB+RN+ECORR, post-fit: spin + JUMPs)",
            "value": R * args.steps / (ms * 1e-3), "unit": "realizations/s", "ms_per_step": ms / args.steps,
            "steps": args.steps, "warmup": args.warmup, "realizations_per_step": R,
            "workload": bench.workload_name("2", kind, b) + " + timing-model fit per pulsar (poly=2 + JUMPs of flag f)",
            "columns_per_pulsar": {"max": int(tm["k"].max()), "sum": int(tm["k"].sum())},
            "kernels_ms_per_step": kms,
            "projection": {"kernels": "timing_reduce + timing_apply", "ms_per_step": proj_ms,
                           "algorithmic_bytes_per_output": 16, "algorithmic_GBps": gbps, "frac": gbps / hbm, "peak": hbm,
                           "peak_source": how, "moved_bytes_per_output": 24},
            "setup_s": setup_s, "card": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

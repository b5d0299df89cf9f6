"""Cost of the on-device timeline (gs_set_timeline): gs_summarize with the timeline off and on.

Workloads, each on one handle of replicas generated with gs_boot_traces (Philox key (seed, replica)) on 4x32x8:
  fifo      bench.py's fifo step: 3696 replicas x 100k jobs, span budget 1.5
  sjf       2640 replicas x 10k jobs (bench.py's sjf extra)
  dlas-gpu  2640 replicas x 100k jobs, 4 queues (bench.py's dlas-gpu extra)
Every step is gs_boot_traces -> gs_run -> gs_summarize (-> gs_fetch_timeline), with the timeline off, on at B = 128 or
on at B = 1024; the three alternate step by step after warm-up (the order rotates).  The bin width is the run's
largest makespan over B - 1, so the bins span the runs.  Reports per setting the median device time of gs_summarize's
kernels, the extra over "off", and the bytes and wall time of reading the bins back.  A seeded sample of replicas is
checked against the numpy binning of their fetched rows (tests/test_timeline_cpu.py).  The GPU's name and power limit
are read in the same run.  Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tools"))

from bench import BASE_SEED, fast_table, make_policy  # noqa: E402  (the benchmark's own trace generator and policies)
from summary_bench import gpu_info  # noqa: E402

WORKLOADS = (("fifo", 3696, 100000), ("sjf", 2640, 10000), ("dlas-gpu", 2640, 100000))
ROWS_CAP = {"fifo": 0, "sjf": 1 << 16, "dlas-gpu": 1 << 16}     # the policies run in windows, summarised after each
SETTINGS = (0, 128, 1024)


def step(eng, params, W, B, rows_cap, sample=()):
    """one boot -> run -> summarise step with the timeline at (W, B) (B = 0: off), gs_summarize after every gs_run
    window; (summary kernel ms over the windows, fetch s, bins, summaries, rows of the `sample` replicas)"""
    eng.boot_traces(params)
    eng.set_timeline(W, B)
    ms, parts = 0.0, {i: [] for i in sample}
    while True:
        eng.run(0, rows_cap)
        out, m = eng.summarize(with_time=True)
        ms += m
        for i in sample:
            w = eng.window(i)
            if w.ticks > w.row_first:
                parts[i].append(eng.fetch_rows(i, w.row_first, w.ticks - w.row_first))
        if out["done"].all():
            break
    bins, fetch_s = None, 0.0
    if B:
        t0 = time.perf_counter()
        bins = eng.timeline()
        fetch_s = time.perf_counter() - t0
    return ms, fetch_s, bins, out, {i: np.concatenate(p) for i, p in parts.items()}


def measure(name, R, n, args, cluster):
    from gpuschedule_b200 import capi
    from test_timeline_cpu import assert_bins, reference_bins
    population = fast_table(n, BASE_SEED)
    params = np.zeros(R, dtype=capi.BOOT_PARAMS_DTYPE)
    params["seed"], params["stream"], params["n"], params["gap_num"], params["gap_den"] = args.seed, np.arange(R), n, 1, 1
    res = {B: [] for B in SETTINGS}
    with capi.Engine(device=0, nsims=R) as eng:
        eng.set_async(True)
        pol = make_policy(name, population)
        for i in range(R):
            eng.config(i, cluster, pol)
        eng.set_span_budget(1.5)
        eng.boot_population(population)
        cap = ROWS_CAP[name]
        _, _, _, out, _ = step(eng, params, 0, 0, cap)
        makespan = int(out["makespan"].max())
        width = {B: max(1, math.ceil(makespan / max(B - 1, 1))) for B in SETTINGS}
        for s in range(args.warmup + args.steps):
            order = SETTINGS[s % 3:] + SETTINGS[:s % 3]
            for B in order:
                ms, fetch_s, _, _, _ = step(eng, params, width[B] if B else 0, B, cap)
                if s >= args.warmup:
                    res[B].append((ms, fetch_s))
        B = 128
        rng = np.random.default_rng(7)
        sample = sorted(rng.choice(R, size=min(args.sample, R), replace=False).tolist())
        _, _, bins, out, rows = step(eng, params, width[B], B, cap, sample)
        for i in sample:
            assert_bins(bins[i], reference_bins(rows[i], width[B], B), f"{name} replica {i}")
        events = sum(int(eng.stats(i).events) for i in range(R))
    med = {B: float(np.median([r[0] for r in res[B]])) for B in SETTINGS}
    block = {"replicas": R, "jobs": n, "events_per_step": events, "max_makespan": makespan,
             "summarize_kernel_ms_off": med[0], "checked_replicas": len(sample)}
    for B in SETTINGS[1:]:
        block[f"B{B}"] = {"bin_width": width[B], "summarize_kernel_ms": med[B], "extra_kernel_ms": med[B] - med[0],
                          "fetch_bytes": 128 * R * B, "fetch_ms": 1e3 * float(np.median([r[1] for r in res[B]]))}
    return block


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=3, help="timed steps of each setting")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=1, help="Philox seed of the generated replicas")
    ap.add_argument("--sample", type=int, default=3, help="replicas checked against the numpy binning of their rows")
    ap.add_argument("--workloads", nargs="+", default=[w[0] for w in WORKLOADS], choices=[w[0] for w in WORKLOADS])
    args = ap.parse_args()
    from gpuschedule_b200 import capi
    out = {"gpu": gpu_info(), "cluster": "4x32x8", "steps": args.steps, "warmup": args.warmup}
    cluster = capi.make_cluster(4, 32, 8)
    for name, R, n in WORKLOADS:
        if name in args.workloads:
            out[name] = measure(name, R, n, args, cluster)
    out["gpu_after"] = gpu_info()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

"""Cost of the on-device time-weighted occupancy (gs_set_occupancy): gs_summarize's kernel time with it off and on.

Workloads, each on one handle of replicas generated with gs_boot_traces (Philox key (seed, replica)) on 4x32x8:
  fifo      bench.py's fifo step: 3696 replicas x 100k jobs, span budget 1.5, one gs_run window
  dlas-gpu  2640 replicas x 100k jobs, 4 queues (bench.py's dlas-gpu extra), run in windows of 65536 rows
A run is summarised after every gs_run window, as a sweep does; the setting cannot change once rows are folded, so
every step runs the workload twice from gs_reset, once off and once on (the queue edges 0, 1, 2, 4, ... 2^30), in an
order that rotates step by step.  Reports per setting the median over steps of the summed device time of
gs_summarize's kernels over the run's windows, the extra of "on", and the bytes and wall time of gs_fetch_occupancy.
The summaries of both settings must be byte-equal, and three replicas per workload are checked against
tests/test_occupancy_cpu.reference over their fetched rows.  The GPU's name and power limit are read in the same run.
Prints one JSON line."""
from __future__ import annotations

import argparse
import json
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

WORKLOADS = (("fifo", 3696, 100000), ("dlas-gpu", 2640, 100000))
ROWS_CAP = {"fifo": 0, "dlas-gpu": 1 << 16}
EDGES = (0,) + tuple(2 ** i for i in range(31))


def run_once(eng, name, on):
    """reset, run to the end summarising after every window -> (summed kernel ms, windows, last summaries)"""
    eng.reset()
    eng.set_occupancy(EDGES if on else None)
    total, windows = 0.0, 0
    while True:
        eng.run(0, ROWS_CAP[name])
        out, ms = eng.summarize(with_time=True)
        total += ms
        windows += 1
        if out["done"].all():
            return total, windows, out


def measure(name, R, n, args, cluster):
    from gpuschedule_b200 import capi
    from test_occupancy_cpu import assert_occ, reference
    population = fast_table(n, BASE_SEED)
    params = np.zeros(R, dtype=capi.BOOT_PARAMS_DTYPE)
    params["seed"], params["stream"], params["n"], params["gap_num"], params["gap_den"] = args.seed, np.arange(R), n, 1, 1
    res = {"off": [], "on": []}
    fetch = []
    with capi.Engine(device=0, nsims=R) as eng:
        eng.set_async(True)
        pol = make_policy(name, population)
        for i in range(R):
            eng.config(i, cluster, pol)
        eng.set_span_budget(1.5)
        eng.boot_population(population)
        eng.boot_traces(params)
        ref_out = None
        for s in range(args.warmup + args.steps):
            for on in ((False, True) if s % 2 == 0 else (True, False)):
                ms, windows, out = run_once(eng, name, on)
                if ref_out is None:
                    ref_out = out
                assert out.tobytes() == ref_out.tobytes()
                if on:
                    t0 = time.perf_counter()
                    rec, busy, queue = eng.occupancy()
                    f_s = time.perf_counter() - t0
                if s >= args.warmup:
                    res["on" if on else "off"].append(ms)
                    if on:
                        fetch.append(f_s)
        rng = np.random.default_rng(7)
        sample = sorted(rng.choice(R, size=min(args.sample, R), replace=False).tolist())
        eng.reset()
        eng.set_occupancy(EDGES)
        parts = {i: [] for i in sample}
        while True:
            eng.run(0, ROWS_CAP[name])
            out = eng.summarize()
            for i in sample:
                w = eng.window(i)
                if w.ticks > w.row_first:
                    parts[i].append(eng.fetch_rows(i, w.row_first, w.ticks - w.row_first))
            if out["done"].all():
                break
        rec, busy, queue = eng.occupancy()
        for i in sample:
            assert_occ(rec[i], busy[i], queue[i], reference(np.concatenate(parts[i]), 1024, EDGES, True, per_tick=name == "fifo"),
                       f"{name} replica {i}")
    med = {k: float(np.median(v)) for k, v in res.items()}
    return {"replicas": R, "jobs": n, "windows": windows, "rows": int(out["rows"].sum()), "checked_replicas": sample,
            "summarize_kernel_ms_off": med["off"], "summarize_kernel_ms_on": med["on"], "extra_kernel_ms": med["on"] - med["off"],
            "runs_ms_off": res["off"], "runs_ms_on": res["on"],
            "fetch_bytes": R * (capi.OCC_DTYPE.itemsize + 8 * (2 * 1025 + len(EDGES) + 1)),
            "fetch_ms": 1e3 * float(np.median(fetch))}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=4, help="timed runs of each setting")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=1, help="Philox seed of the generated replicas")
    ap.add_argument("--sample", type=int, default=3, help="replicas checked against the restatement")
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

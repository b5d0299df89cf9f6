"""Cost of the on-device job statistics by key with bounded slowdown (gs_set_slowdown): gs_summarize with them off and on.

Workloads, each on one handle of replicas generated with gs_boot_traces (Philox key (seed, replica)) on 4x32x8:
  fifo      bench.py's fifo step: 3696 replicas x 100k jobs, span budget 1.5
  dlas-gpu  2640 replicas x 100k jobs, 4 queues (bench.py's dlas-gpu extra)
Each handle runs its replicas to the end once (gs_summarize after every gs_run window); the settings are then compared
on the finished run, where the job part is largest: off and "C4" (length classes 60 / 720 / 2880, tau 1, the sweep's
default edges: 31 for wait / turnaround / jct and 21 for sd) alternate call by call after warm-up (the order
rotates).  Reports per setting the median device time of gs_summarize's kernels, the extra over "off", and the bytes
and wall time of gs_fetch_slowdown.  Three replicas per workload are checked against reference_slowdown
(tests/test_slowdown_cpu.py) over their fetched job records and traces.  The GPU's name and power limit are read in
the same run.  Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import types

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tools"))

from bench import BASE_SEED, fast_table, make_policy  # noqa: E402  (the benchmark's own trace generator and policies)
from summary_bench import gpu_info  # noqa: E402

WORKLOADS = (("fifo", 3696, 100000), ("dlas-gpu", 2640, 100000))
ROWS_CAP = {"fifo": 0, "dlas-gpu": 1 << 16}       # the policy runs in windows, summarised after each
SETTINGS = {"off": None,
            "C4": ("length", (60, 720, 2880), 1, tuple(2 ** i for i in range(31)), tuple(1024 * 2 ** i for i in range(21)))}


def measure(name, R, n, args, cluster):
    from gpuschedule_b200 import capi
    from test_slowdown_cpu import assert_slowdown, reference_slowdown
    from test_summary_cpu import job_columns
    population = fast_table(n, BASE_SEED)
    params = np.zeros(R, dtype=capi.BOOT_PARAMS_DTYPE)
    params["seed"], params["stream"], params["n"], params["gap_num"], params["gap_den"] = args.seed, np.arange(R), n, 1, 1
    res = {k: [] for k in SETTINGS}
    fetch = []
    with capi.Engine(device=0, nsims=R) as eng:
        eng.set_async(True)
        pol = make_policy(name, population)
        for i in range(R):
            eng.config(i, cluster, pol)
        eng.set_span_budget(1.5)
        eng.boot_population(population)
        eng.boot_traces(params)
        t0 = time.perf_counter()
        while True:
            eng.run(0, ROWS_CAP[name])
            out = eng.summarize()
            if out["done"].all():
                break
        run_s = time.perf_counter() - t0
        names = list(SETTINGS)
        for s in range(args.warmup + args.steps):
            for key in names[s % 2:] + names[:s % 2]:
                eng.set_slowdown(*(SETTINGS[key] or (None,)))
                out2, ms = eng.summarize(with_time=True)
                assert out2.tobytes() == out.tobytes()
                if SETTINGS[key]:
                    t0 = time.perf_counter()
                    eng.slowdown()
                    f_s = time.perf_counter() - t0
                if s >= args.warmup:
                    res[key].append(ms)
                    if SETTINGS[key]:
                        fetch.append(f_s)
        rng = np.random.default_rng(7)
        sample = sorted(rng.choice(R, size=min(args.sample, R), replace=False).tolist())
        setting = SETTINGS["C4"]
        eng.set_slowdown(*setting)
        eng.summarize()
        recs, hist = eng.slowdown()
        for i in sample:
            tr = eng.fetch_trace(i)
            table = types.SimpleNamespace(arrive_tick=tr["arrive_tick"].astype(np.int64), gpus=tr["gpus"].astype(np.int64))
            jobs = job_columns(table, *eng.fetch_jobs(i))
            assert_slowdown(recs[i], hist[i], reference_slowdown(*jobs, *setting), f"{name} replica {i}")
        finished = int(out["finished"].sum())
    med = {k: float(np.median(v)) for k, v in res.items()}
    C, E, Es = len(setting[1]) + 1, len(setting[3]), len(setting[4])
    return {"replicas": R, "jobs": n, "finished_jobs": finished, "run_s": run_s, "summarize_kernel_ms_off": med["off"],
            "checked_replicas": sample,
            "C4": {"summarize_kernel_ms": med["C4"], "extra_kernel_ms": med["C4"] - med["off"],
                   "fetch_bytes": R * C * (capi.SDCLASS_DTYPE.itemsize + 4 * (3 * (E + 1) + Es + 1)),
                   "fetch_ms": 1e3 * float(np.median(fetch))}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5, help="timed gs_summarize calls of each setting")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1, help="Philox seed of the generated replicas")
    ap.add_argument("--sample", type=int, default=3, help="replicas checked against reference_slowdown")
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

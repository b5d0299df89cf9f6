"""Cost of the on-device job statistics by arrival time (gs_set_arrivals): gs_summarize with them off and on.

Workloads, each on one handle of replicas generated with gs_boot_traces (Philox key (seed, replica)) on 4x32x8:
  fifo      bench.py's fifo step: 3696 replicas x 100k jobs, span budget 1.5
  dlas-gpu  2640 replicas x 100k jobs, 4 queues (bench.py's dlas-gpu extra)
Each handle runs its replicas to the end once (gs_summarize after every gs_run window); the settings are then compared
on the finished run, where the job part is largest: off, B = 128 and B = 1024 bins alternate call by call after warm-up
(the order rotates).  The bin width W is chosen so that B bins span the base trace's arrivals: about 780 finished jobs
per bin at B = 128 (the block path of gs_arr_jobs_kernel) and about 100 at B = 1024 (the warp path).  Reports per
setting the median device time of gs_summarize's kernels, the extra over "off", the bytes and wall time of
gs_fetch_arrivals, and the device's free memory with the 1024-bin records allocated.  One replica per workload and
setting is checked against reference_arrivals (tests/test_arrivals_cpu.py) over its fetched job records and trace.  The
GPU's name and power limit are read in the same run.  Prints one JSON line."""
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
BINS = {"off": 0, "B128": 128, "B1024": 1024}


def measure(name, R, n, args, cluster):
    import torch
    from gpuschedule_b200 import capi
    from test_arrivals_cpu import assert_arrivals, reference_arrivals
    from test_summary_cpu import job_columns
    population = fast_table(n, BASE_SEED)
    last = int(population.arrive_tick.max())
    params = np.zeros(R, dtype=capi.BOOT_PARAMS_DTYPE)
    params["seed"], params["stream"], params["n"], params["gap_num"], params["gap_den"] = args.seed, np.arange(R), n, 1, 1
    res = {k: [] for k in BINS}
    fetch = {k: [] for k in BINS if BINS[k]}
    width = {k: last // B + 1 for k, B in BINS.items() if B}
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
        eng.set_arrivals(width["B1024"], 1024)
        free_b, total_b = torch.cuda.mem_get_info(0)
        names = list(BINS)
        for s in range(args.warmup + args.steps):
            k = s % len(names)
            for key in names[k:] + names[:k]:
                eng.set_arrivals(width.get(key, 0), BINS[key])
                out2, ms = eng.summarize(with_time=True)
                assert out2.tobytes() == out.tobytes()
                if BINS[key]:
                    t0 = time.perf_counter()
                    eng.arrivals()
                    f_s = time.perf_counter() - t0
                if s >= args.warmup:
                    res[key].append(ms)
                    if BINS[key]:
                        fetch[key].append(f_s)
        i = int(np.random.default_rng(7).integers(R))
        tr = eng.fetch_trace(i)
        table = types.SimpleNamespace(arrive_tick=tr["arrive_tick"].astype(np.int64), gpus=tr["gpus"].astype(np.int64))
        jobs = job_columns(table, *eng.fetch_jobs(i))
        checked = {}
        for key, B in BINS.items():
            if B:
                eng.set_arrivals(width[key], B)
                eng.summarize()
                recs = eng.arrivals(first=i, count=1)[0]
                assert_arrivals(recs, reference_arrivals(*jobs, table.arrive_tick, width[key], B, 1), f"{name} {key} replica {i}")
                sizes = recs["s"]["jc"]["jobs"]
                checked[key] = {"replica": i, "max_bin_jobs": int(sizes.max()), "median_bin_jobs": float(np.median(sizes))}
        finished = int(out["finished"].sum())
    med = {k: float(np.median(v)) for k, v in res.items()}
    return {"replicas": R, "jobs": n, "finished_jobs": finished, "run_s": run_s, "summarize_kernel_ms_off": med["off"],
            "free_bytes_with_1024_bins": int(free_b), "total_bytes": int(total_b),
            **{key: {"bins": BINS[key], "width": width[key], "summarize_kernel_ms": med[key], "extra_kernel_ms": med[key] - med["off"],
                     "fetch_bytes": R * BINS[key] * capi.ABIN_DTYPE.itemsize, "fetch_ms": 1e3 * float(np.median(fetch[key])),
                     "checked": checked[key]} for key in BINS if BINS[key]}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5, help="timed gs_summarize calls of each setting")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1, help="Philox seed of the generated replicas")
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

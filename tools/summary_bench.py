"""Cost of on-device run summaries (gs_summarize) on one GPU, next to the engine they summarise.

Workloads (the same traces, seeds and cluster as bench.py):
  fifo      bench.py's headline step: replicas x 100k-job synthetic traces on 4x32x8, one trace per replica; every step
            is "packed upload -> gs_run -> gs_summarize" and reads back one 256-byte record per replica
  policies  the sjf (10k jobs) / dlas-gpu / gittins (100k jobs) batches of bench.py's secondary measurements

Reports, per workload: the summary kernels' device time per step and its ratio to the engine's kernel time, the
bytes read back per step, and for fifo the wall-clock events/s of the per-step loop.  A fixed, seeded sample of
replicas is checked against the numpy summary of their fetched rows and job records (tests/test_summary_cpu.py).
The GPU's name and power limit are read in the same run.  Prints one JSON line."""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

from bench import BASE_SEED, fast_table, make_policy  # noqa: E402  (the benchmark's own trace generator and policies)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip()
    except OSError:
        q = ""
    return q or "nvidia-smi unavailable"


def check_sample(eng, tables, sample):
    """summaries of `sample` replicas == the numpy summary of their fetched rows and job records"""
    from test_summary_cpu import assert_summary, job_columns, reference_summary
    out = eng.summarize()
    for i in sample:
        st = eng.stats(i)
        rows = eng.fetch_rows(i, 0, st.ticks)
        recs, order = eng.fetch_jobs(i)
        assert_summary(out[i], reference_summary(rows, *job_columns(tables[i], recs, order)), f"replica {i}")
    return len(sample)


def fifo(args, cluster):
    from gpuschedule_b200 import capi
    R, n = args.replicas, args.jobs
    rng = np.random.default_rng(7)
    sample = sorted(rng.choice(R, size=min(args.sample, R), replace=False).tolist())
    pitch = capi.JOBIN_DTYPE.itemsize * n
    buf = capi.PinnedBuffer(pitch * R)
    block = buf.view(capi.JOBIN_DTYPE, R * n)
    tables = {}

    def make(r):                                   # only the checked replicas keep their table
        t = fast_table(n, BASE_SEED + r, rate=0.5)
        block[r * n:(r + 1) * n] = t.packed()
        if r in sample:
            tables[r] = t
    with cf.ThreadPoolExecutor(min(32, len(os.sched_getaffinity(0)))) as ex:
        list(ex.map(make, range(R)))
    n_each = np.full(R, n, dtype=np.int64)
    with capi.Engine(device=0, nsims=R) as eng:
        eng.set_async(True)
        for i in range(R):
            eng.config(i, cluster)
        eng.set_span_budget(1.5)
        steps = []
        for step in range(args.warmup + args.steps):
            k0 = eng.stats(0).kernel_ms
            t0 = time.perf_counter()
            eng.load_traces_packed(block, pitch, n_each)
            eng.run(0, 0)
            out, sum_ms = eng.summarize(with_time=True)
            wall = time.perf_counter() - t0
            assert out["done"].all()
            eng_ms = eng.stats(0).kernel_ms - k0
            events = sum(int(eng.stats(i).events) for i in range(R))
            if step >= args.warmup:
                steps.append((wall, sum_ms, eng_ms, events))
        checked = check_sample(eng, tables, sample)
    buf.free()
    wall, sum_ms, eng_ms, events = (float(np.median([s[k] for s in steps])) for k in range(4))
    return {"workload": f"{n}-job synthetic traces x {R} replicas, 4x32x8, fifo+yarn (bench.py's step)",
            "summary_kernel_ms_per_step": sum_ms, "engine_kernel_ms_per_step": eng_ms, "summary_over_engine": sum_ms / eng_ms,
            "bytes_read_back_per_step": 256 * R, "wall_ms_per_step": wall * 1e3, "events_per_step": events,
            "e2e_events_per_s": events / wall, "steps": args.steps, "checked_replicas": checked}


def policy(args, cluster, name, njobs):
    from gpuschedule_b200 import capi
    R = args.policy_replicas
    with cf.ThreadPoolExecutor(min(32, len(os.sched_getaffinity(0)))) as ex:
        tables = list(ex.map(lambda sd: fast_table(njobs, sd, rate=0.5), [BASE_SEED + r for r in range(R)]))
    rng = np.random.default_rng(11)
    sample = sorted(rng.choice(R, size=min(args.sample, R), replace=False).tolist())
    with capi.Engine(device=0, nsims=R) as eng:
        for i, t in enumerate(tables):
            eng.config(i, cluster, make_policy(name, t))
            eng.load_trace_packed(i, t.packed())
        sum_ms, launches = 0.0, 0
        while True:
            eng.run(0, 0)
            out, ms = eng.summarize(with_time=True)
            sum_ms += ms
            launches += 1
            if out["done"].all():
                break
        eng_ms = eng.stats(0).kernel_ms
        checked = check_sample(eng, tables, sample)
    return {"workload": f"{njobs}-job synthetic traces x {R} replicas, 4x32x8, {name}", "launches": launches,
            "summary_kernel_ms": sum_ms, "engine_kernel_ms": eng_ms, "summary_over_engine": sum_ms / eng_ms,
            "bytes_read_back": 256 * R * launches, "checked_replicas": checked}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replicas", type=int, default=3696, help="fifo replicas: the H100's 132 SMs x 28 resident warps, as bench.py")
    ap.add_argument("--jobs", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--policy-replicas", type=int, default=2640, help="as bench.py: 132 SMs x 20 resident warps")
    ap.add_argument("--no-policies", action="store_true")
    ap.add_argument("--sample", type=int, default=4, help="replicas per workload checked against the numpy summary")
    args = ap.parse_args()
    from gpuschedule_b200 import capi
    cluster = capi.make_cluster(4, 32, 8)
    res = {"gpu": gpu_info(), "fifo": fifo(args, cluster)}
    if not args.no_policies:
        for name, njobs in (("sjf", 10000), ("dlas-gpu", 100000), ("gittins", 100000)):
            res[name] = policy(args, cluster, name, njobs)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

"""Cost of the paired per-job comparison (gs_compare) on a finished bootstrap handle.

Workload: bench.py's 100k-job trace on 4x32x8, generated with gs_boot_traces into one handle as 1320 fifo and 1320
dlas-gpu replicas on the same Philox streams (key (seed, replica)), run to the end (gs_summarize after every gs_run
window).  Then, alternating call by call after warm-up (the order rotates): gs_compare over the 1320 (fifo, dlas-gpu)
pairs at (C, E) = (1, 0), (4, 63) and (8, 255), and gs_summarize with jobdist (C = 4, E = 32) on the same handle for
scale.  Reports the median device time of each call's kernels, and the bytes read back.  Three pairs are checked
against the numpy restatement (tests/test_compare_cpu.py) over their fetched job records.  The GPU's name and power
limit are read in the same run.  Prints one JSON line."""
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

PAIRS, JOBS = 1320, 100000
DIFF_EDGES = tuple(-2 ** i for i in range(30, -1, -1)) + (0,) + tuple(2 ** i for i in range(31))
SETTINGS = {"C1_E0": ((), ()),
            "C4_E63": ((5, 17, 65), DIFF_EDGES),
            "C8_E255": ((2, 3, 5, 9, 17, 33, 65), tuple(range(-127 * 4096, 128 * 4096, 4096)))}
JD_SETTING = ((5, 17, 65), tuple(2 ** i for i in range(31)) + (2 ** 31 - 1,))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5, help="timed calls of each setting")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1, help="Philox seed of the generated replicas")
    ap.add_argument("--sample", type=int, default=3, help="pairs checked against the numpy restatement")
    args = ap.parse_args()
    from gpuschedule_b200 import capi, tracegen
    from test_compare_cpu import assert_pair, reference_pair, run_cols
    out = {"gpu": gpu_info(), "cluster": "4x32x8", "pairs": PAIRS, "jobs": JOBS, "steps": args.steps, "warmup": args.warmup}
    cluster = capi.make_cluster(4, 32, 8)
    population = fast_table(JOBS, BASE_SEED)
    R = 2 * PAIRS
    params = np.zeros(R, dtype=capi.BOOT_PARAMS_DTYPE)
    params["seed"], params["stream"], params["n"], params["gap_num"], params["gap_den"] = args.seed, np.arange(R) % PAIRS, JOBS, 1, 1
    pa, pb = np.arange(PAIRS), np.arange(PAIRS) + PAIRS
    times = {k: [] for k in list(SETTINGS) + ["summarize_jd_C4_E32"]}
    with capi.Engine(device=0, nsims=R) as eng:
        eng.set_async(True)
        fifo, dlas = make_policy("fifo", population), make_policy("dlas-gpu", population)
        for i in range(R):
            eng.config(i, cluster, fifo if i < PAIRS else dlas)
        eng.set_span_budget(1.5)
        eng.boot_population(population)
        eng.boot_traces(params)
        t0 = time.perf_counter()
        while True:
            eng.run(0, 1 << 16)
            summ = eng.summarize()
            if summ["done"].all():
                break
        out["run_s"] = time.perf_counter() - t0
        out["finished_jobs"] = int(summ["finished"].sum())
        eng.set_jobdist(*JD_SETTING)
        names = list(times)
        results = {}
        for s in range(args.warmup + args.steps):
            for key in names[s % len(names):] + names[:s % len(names)]:
                if key in SETTINGS:
                    recs, hist, ms = eng.compare(pa, pb, *SETTINGS[key], with_time=True)
                    if key in results:
                        assert recs.tobytes() == results[key][0].tobytes() and hist.tobytes() == results[key][1].tobytes()
                    results[key] = (recs, hist)
                else:
                    _, ms = eng.summarize(with_time=True)
                if s >= args.warmup:
                    times[key].append(ms)
        rng = np.random.default_rng(7)
        sample = sorted(rng.choice(PAIRS, size=min(args.sample, PAIRS), replace=False).tolist())
        for i in sample:
            table = tracegen.bootstrap_table(population, args.seed, i, JOBS, 1, 1)
            (ra, fa), (rb, fb) = eng.fetch_jobs(int(pa[i])), eng.fetch_jobs(int(pb[i]))
            for key, (bounds, edges) in SETTINGS.items():
                recs, hist = results[key]
                assert_pair(recs[i], hist[i], reference_pair(table.arrive_tick, table.gpus, run_cols(ra), fa, run_cols(rb), fb, bounds, edges),
                            f"{key} pair {i}")
        out["checked_pairs"] = sample
        out["jobs_in_both"] = int(results["C1_E0"][0]["jobs"].sum())
    for key, v in times.items():
        block = {"kernel_ms_median": float(np.median(v)), "kernel_ms_min": float(np.min(v)), "kernel_ms_max": float(np.max(v))}
        if key in SETTINGS:
            C, E = len(SETTINGS[key][0]) + 1, len(SETTINGS[key][1])
            block["readback_bytes"] = PAIRS * C * (288 + 3 * (E + 1) * 4)
        out[key] = block
    out["gpu_after"] = gpu_info()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

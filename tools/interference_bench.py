"""Cost of the on-device interference statistics (gs_horus_set_interference): gs_horus_summarize with them off and on.

Workload: bench.py's horus line, 8448 replicas of 60-job traces (bench.fast_table) on a 2x4x8 cluster, horus schedule
and placement, one shared standard-normal stream (seed 0).  The handle runs its replicas to the end once; the settings
are then compared on the finished run: off, "C1" (one class) and "C4" (num_gpu classes 1, 2-3, 4-7, 8+) alternate call
by call after warm-up (the order rotates).  Reports per setting the median device time of gs_horus_summarize's kernels
(kernel_ms), the extra over "off", and the bytes and wall time of gs_horus_fetch_interference.  Three replicas are
checked against reference_interference (tests/test_interference_cpu.py) over their fetched job records.  The GPU's name
and power limit are read in the same run.  Prints one JSON line."""
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

from bench import BASE_SEED, fast_table  # noqa: E402  (the benchmark's own trace generator)
from summary_bench import gpu_info  # noqa: E402

SETTINGS = {"off": None, "C1": (), "C4": (2, 4, 8)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replicas", type=int, default=8448)
    ap.add_argument("--jobs", type=int, default=60)
    ap.add_argument("--stream", type=int, default=4000000, help="standard-normal samples shared by the replicas")
    ap.add_argument("--rows", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=20, help="timed gs_horus_summarize calls of each setting")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=3, help="replicas checked against reference_interference")
    args = ap.parse_args()
    from gpuschedule_b200 import capi
    from test_interference_cpu import assert_interference, job_columns_if, reference_interference
    out = {"gpu": gpu_info(), "cluster": "2x4x8", "replicas": args.replicas, "jobs": args.jobs, "steps": args.steps,
           "warmup": args.warmup}
    R, n = args.replicas, args.jobs
    cluster = capi.make_cluster(num_switch=2, num_node_p_switch=4, num_gpu_p_node=8)
    tables = [fast_table(n, BASE_SEED + 1000 + r, rate=1.0) for r in range(R)]
    np.random.seed(0)
    stream = np.random.standard_normal(args.stream)
    hp = capi.make_horus_params("horus", "horus", 5)
    res = {k: [] for k in SETTINGS}
    fetch = {k: [] for k in SETTINGS if SETTINGS[k] is not None}
    with capi.HorusEngine(device=0, nsims=R) as eng:
        for r in range(R):
            eng.config(r, cluster, hp)
            eng.load_trace(r, tables[r])
        eng.load_stream(-1, stream)
        t0 = time.perf_counter()
        eng.run(rows_cap=args.rows)
        out["run_s"] = time.perf_counter() - t0
        base = eng.summarize()
        assert base["done"].all()
        names = list(SETTINGS)
        for s in range(args.warmup + args.steps):
            k0 = s % len(names)
            for key in names[k0:] + names[:k0]:
                eng.set_interference(SETTINGS[key])
                rec, ms = eng.summarize(with_time=True)
                assert rec.tobytes() == base.tobytes()
                if SETTINGS[key] is not None:
                    t0 = time.perf_counter()
                    eng.interference()
                    f_s = time.perf_counter() - t0
                if s >= args.warmup:
                    res[key].append(ms)
                    if SETTINGS[key] is not None:
                        fetch[key].append(f_s)
        rng = np.random.default_rng(7)
        sample = sorted(rng.choice(R, size=min(args.sample, R), replace=False).tolist())
        eng.set_interference(SETTINGS["C4"])
        eng.summarize()
        recs = eng.interference()
        for i in sample:
            _, _, _, hrecs, order = eng.fetch(i)
            assert_interference(recs[i], reference_interference(*job_columns_if(tables[i], hrecs, order), SETTINGS["C4"]), f"replica {i}")
        out["degraded_jobs"] = int(recs["degraded"]["jobs"].sum())
        out["finished_jobs"] = int(base["finished"].sum())
    med = {k: float(np.median(v)) for k, v in res.items()}
    out["summarize_kernel_ms_off"] = med["off"]
    out["checked_replicas"] = sample
    for key in fetch:
        C = len(SETTINGS[key]) + 1
        out[key] = {"summarize_kernel_ms": med[key], "extra_kernel_ms": med[key] - med["off"],
                    "fetch_bytes": R * C * capi.IFCLASS_DTYPE.itemsize, "fetch_ms": 1e3 * float(np.median(fetch[key]))}
    out["gpu_after"] = gpu_info()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

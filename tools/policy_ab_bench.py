"""Rates of the event-driven policy kernels, optionally of two builds of libgsched.so alternated in one process.

Workload: bench.py's secondary policy measurements -- sjf on 10k-job traces, dlas-gpu and gittins on 100k-job traces,
2640 replicas on 4x32x8, with bench.py's trace generator, seeds and policy settings.  A round loads every replica into a
fresh handle, runs it once to size the row window (as bench.py does) and then times `--steps` full runs with the
engine's device timer; the rate is events / kernel seconds, bench.py's figure.  With `--other PATH` every round is run
once with this tree's library and once with the library at PATH, the order swapped every round, and the two must give
the same events and the same rows for replica 0.  Prints one JSON line: every round's rate per build and policy, their
medians and min / max, and the GPU's name and power limit read in the same run.

    python tools/policy_ab_bench.py [--other OTHER/libgsched.so] [--rounds 4] [--steps 3]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

from bench import BASE_SEED, fast_table, make_policy, run_to_done  # noqa: E402  (the benchmark's own workload)
from summary_bench import gpu_info  # noqa: E402

WORKLOADS = (("sjf", 10000), ("dlas-gpu", 100000), ("gittins", 100000))


def load_build(path):
    """the ctypes library at `path` with the package's prototypes (capi.load_library on another file)"""
    from gpuschedule_b200 import capi
    keep_lib, keep_path = capi._lib, capi.LIB_PATH
    capi._lib, capi.LIB_PATH = None, path
    try:
        return capi.load_library()
    finally:
        capi._lib, capi.LIB_PATH = keep_lib, keep_path


def one_round(lib, cluster, tables, pols, steps):
    """(events / kernel second, events, rows of replica 0) of `steps` timed runs of every replica under `lib`"""
    from gpuschedule_b200 import capi
    keep = capi._lib
    capi._lib = lib
    try:
        with capi.Engine(device=0, nsims=len(tables)) as eng:
            for i, t in enumerate(tables):
                eng.config(i, cluster, pols[i])
                eng.load_trace_packed(i, t.packed())
            run_to_done(eng, 0)
            cap = max(eng.stats(i).ticks for i in range(len(tables))) + 64
            ms = 0.0
            for _ in range(steps):
                eng.reset()
                run_to_done(eng, cap)
                ms += eng.stats(0).kernel_ms
            events = sum(eng.stats(i).events for i in range(len(tables)))
            return events * steps / (ms / 1e3), events, eng.fetch_rows(0)
    finally:
        capi._lib = keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", default=None, help="another build of libgsched.so, timed alternately with this tree's")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3, help="timed full runs per round")
    ap.add_argument("--replicas", type=int, default=2640)
    args = ap.parse_args()
    from gpuschedule_b200 import capi, dist as gdist
    builds = {"this": load_build(capi.LIB_PATH)}
    if args.other:
        builds["other"] = load_build(os.path.abspath(args.other))
    cluster = capi.make_cluster(4, 32, 8)
    seeds = gdist.replica_seeds(0, 1, args.replicas, base=BASE_SEED)
    out = {"gpu": gpu_info(), "replicas": args.replicas, "rounds": args.rounds, "steps": args.steps,
           "unit": "events/s (device-timed)", "policies": {}}
    cache = {}
    for name, n in WORKLOADS:
        if n not in cache:
            cache = {n: [fast_table(n, sd, rate=0.5) for sd in seeds]}
        tables = cache[n]
        pols = [make_policy(name, t) for t in tables]
        rates = {b: [] for b in builds}
        ref = None
        for r in range(args.rounds):
            order = list(builds) if r % 2 == 0 else list(builds)[::-1]
            for b in order:
                rate, events, rows = one_round(builds[b], cluster, tables, pols, args.steps)
                rates[b].append(rate)
                if ref is None:
                    ref = (events, rows.tobytes())
                assert (events, rows.tobytes()) == ref, f"{name}: build {b} computes something else"
        out["policies"][name] = {"jobs": n, **{b: {"rates": v, "median": float(np.median(v)), "min": min(v), "max": max(v)}
                                               for b, v in rates.items()}}
        if args.other:
            out["policies"][name]["median_ratio_this_over_other"] = float(np.median(rates["this"]) / np.median(rates["other"]))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

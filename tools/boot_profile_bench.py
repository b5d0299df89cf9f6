"""Cost of profiled bootstrap replicas (gs_boot_traces_profiled) against unprofiled replicas at load 1.

Workload: bench.py's fifo step -- replicas x 100k jobs on 4x32x8, span budget 1.5 (--span-budget) -- on one handle,
the population one fast_table trace of 100k jobs (bench.py's generator), replica r drawn with Philox key (seed, r).
Three loops, each generate -> gs_run -> gs_summarize, alternated step by step after warm-up (the order rotates every
step):
  plain     gs_boot_traces at load 1 (gap scale 1 / 1), no profile
  surge     gs_boot_traces_profiled, every replica under 0:1,20000:3,22000:1 (a 3x surge for 2000 ticks)
  periodic  gs_boot_traces_profiled, every replica under a 24-segment daily cycle of period 1440 ticks, load factors
            1 + 0.4 sin(2 pi (k + 0.5) / 24) for k = 0 .. 23
Reports per loop the medians (and min / max) of the generator's, the engine's and the summary's kernel times, the
wall-clock time per step, the engine's events and the mean wait over all replicas: a profile changes the workload the
engine sees, so the number to compare is the generator's.  Also the host time of gs_boot_profiles.  A seeded sample
of replicas of every loop is compared with tracegen.bootstrap_packed record for record.  The GPU's name and power
limit are read in the same run.  Prints one JSON line."""
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
sys.path.insert(0, os.path.join(REPO, "tools"))

from bench import BASE_SEED, fast_table  # noqa: E402  (the benchmark's own trace generator)
from summary_bench import gpu_info  # noqa: E402

SURGE = (((0, 1.0), (20000, 3.0), (22000, 1.0)), 0)
DAILY = (tuple((60 * k, 1.0 + 0.4 * math.sin(2 * math.pi * (k + 0.5) / 24)) for k in range(24)), 1440)
LOOPS = (("plain", None), ("surge", 0), ("periodic", 1))


def step(eng, R, params, prof):
    """generate -> gs_run -> gs_summarize; (wall s, generator ms, engine ms, summary ms, events, wait sum, finished)"""
    k0 = eng.stats(0).kernel_ms
    t0 = time.perf_counter()
    gen_ms = eng.boot_traces(params, with_time=True, profile=prof)
    eng.run(0, 0)
    out, sum_ms = eng.summarize(with_time=True)
    wall = time.perf_counter() - t0
    assert out["done"].all()
    eng_ms = eng.stats(0).kernel_ms - k0
    events = sum(int(eng.stats(i).events) for i in range(R))
    return wall, gen_ms, eng_ms, sum_ms, events, int(out["wait_sum"].sum()), int(out["finished"].sum())


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replicas", type=int, default=3696, help="as bench.py: the H100's 132 SMs x 28 resident warps")
    ap.add_argument("--jobs", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=5, help="timed steps of each loop")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=1, help="Philox seed of the generated replicas")
    ap.add_argument("--sample", type=int, default=4, help="replicas of each loop compared with the numpy mirror")
    ap.add_argument("--span-budget", type=float, default=1.5, help="span records per job (bench.py's step: 1.5)")
    args = ap.parse_args()
    from gpuschedule_b200 import capi, sweep, tracegen
    R, n = args.replicas, args.jobs
    gpu = gpu_info()
    cluster = capi.make_cluster(4, 32, 8)
    population = fast_table(n, BASE_SEED).packed()
    profiles = [sweep.profile_segments(points, period, 1.0) for points, period in (SURGE, DAILY)]
    params = np.zeros(R, dtype=capi.BOOT_PARAMS_DTYPE)
    params["seed"], params["stream"], params["n"], params["gap_num"], params["gap_den"] = args.seed, np.arange(R), n, 1, 1

    res = {name: [] for name, _ in LOOPS}
    checked = 0
    rng = np.random.default_rng(7)
    with capi.Engine(device=0, nsims=R) as eng:
        eng.set_async(True)
        for i in range(R):
            eng.config(i, cluster)
        eng.set_span_budget(args.span_budget)
        eng.boot_population(population)
        t0 = time.perf_counter()
        eng.boot_profiles(profiles)
        profiles_ms = (time.perf_counter() - t0) * 1e3
        for s in range(args.warmup + args.steps):
            for k in range(len(LOOPS)):
                name, m = LOOPS[(s + k) % len(LOOPS)]
                r = step(eng, R, params, m)
                if s >= args.warmup:
                    res[name].append(r)
        sample = sorted(rng.choice(R, size=min(args.sample, R), replace=False).tolist())
        for name, m in LOOPS:
            eng.boot_traces(params, profile=m)
            for i in sample:
                want = tracegen.bootstrap_packed(population, args.seed, i, n, profile=None if m is None else profiles[m])[0]
                assert eng.fetch_trace(i).tobytes() == want.tobytes(), f"{name}: replica {i} differs from tracegen.bootstrap_packed"
                checked += 1

    def stat(name, k):
        v = [r[k] for r in res[name]]
        return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
    out = {"gpu": gpu, "workload": f"{n}-job traces x {R} replicas, 4x32x8, fifo+yarn (bench.py's step), span budget {args.span_budget}",
           "steps": args.steps, "warmup": args.warmup}
    out["boot_profiles_host_ms"] = profiles_ms
    out["base_last_arrival"] = int(population["arrive_tick"][-1])
    out["profiles"] = {"surge": profiles[0], "periodic": profiles[1]}
    for name, m in LOOPS:
        last = res[name][-1]
        out[name] = {"profile": m, "generator_kernel_ms": stat(name, 1), "engine_kernel_ms": stat(name, 2),
                     "summary_kernel_ms": stat(name, 3), "wall_ms_per_step": float(np.median([r[0] for r in res[name]]) * 1e3),
                     "events_per_step": last[4], "mean_wait_ticks": last[5] / max(last[6], 1)}
    out["checked_replicas"] = checked
    out["gpu_after"] = gpu_info()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

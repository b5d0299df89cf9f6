"""Cost of bootstrap replicas generated on the GPU (gs_boot_traces) against the packed upload of host-made traces.

Workload: bench.py's fifo step -- replicas x 100k jobs on 4x32x8, span budget 1.5 -- timed as two loops on one handle,
alternated step by step after warm-up (which one goes first alternates too):
  boot    gs_boot_traces -> gs_run -> gs_summarize; the population is one fast_table trace of 100k jobs (bench.py's
          generator), replica r draws with Philox key (seed, r) at the base trace's arrival rate
  packed  the loop of tools/summary_bench.py: gs_load_traces_packed of one fast_table trace per replica from a
          page-locked block -> gs_run -> gs_summarize
Reports per loop: the median wall-clock time per step and events/s, the engine and summary kernel times, and for the
boot loop the generator's kernel time and the bytes it writes (32 per job).  A seeded sample of generated replicas is
compared with tracegen.bootstrap_packed record for record.  The GPU's name and power limit are read in the same run.
Prints one JSON line."""
from __future__ import annotations

import argparse
import concurrent.futures as cf
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


def step(eng, R, upload):
    """upload() then gs_run -> gs_summarize; (wall s, upload kernel ms or None, engine ms, summary ms, events)"""
    k0 = eng.stats(0).kernel_ms
    t0 = time.perf_counter()
    gen_ms = upload()
    eng.run(0, 0)
    out, sum_ms = eng.summarize(with_time=True)
    wall = time.perf_counter() - t0
    assert out["done"].all()
    eng_ms = eng.stats(0).kernel_ms - k0
    events = sum(int(eng.stats(i).events) for i in range(R))
    return wall, gen_ms, eng_ms, sum_ms, events


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replicas", type=int, default=3696, help="as bench.py: the H100's 132 SMs x 28 resident warps")
    ap.add_argument("--jobs", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=3, help="timed steps of each loop")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=1, help="Philox seed of the generated replicas")
    ap.add_argument("--sample", type=int, default=8, help="generated replicas compared with the numpy mirror")
    args = ap.parse_args()
    from gpuschedule_b200 import capi, tracegen
    R, n = args.replicas, args.jobs
    gpu = gpu_info()
    cluster = capi.make_cluster(4, 32, 8)
    population = fast_table(n, BASE_SEED).packed()
    params = np.zeros(R, dtype=capi.BOOT_PARAMS_DTYPE)
    params["seed"], params["stream"], params["n"], params["gap_num"], params["gap_den"] = args.seed, np.arange(R), n, 1, 1

    pitch = capi.JOBIN_DTYPE.itemsize * n
    buf = capi.PinnedBuffer(pitch * R)
    block = buf.view(capi.JOBIN_DTYPE, R * n)

    def make(r):
        block[r * n:(r + 1) * n] = fast_table(n, BASE_SEED + r, rate=0.5).packed()
    with cf.ThreadPoolExecutor(min(32, len(os.sched_getaffinity(0)))) as ex:
        list(ex.map(make, range(R)))
    n_each = np.full(R, n, dtype=np.int64)

    res = {"boot": [], "packed": []}
    with capi.Engine(device=0, nsims=R) as eng:
        eng.set_async(True)
        for i in range(R):
            eng.config(i, cluster)
        eng.set_span_budget(1.5)
        eng.boot_population(population)
        loops = {"boot": lambda: eng.boot_traces(params, with_time=True),
                 "packed": lambda: eng.load_traces_packed(block, pitch, n_each)}
        for s in range(args.warmup + args.steps):
            for name in (("boot", "packed") if s % 2 == 0 else ("packed", "boot")):
                r = step(eng, R, loops[name])
                if s >= args.warmup:
                    res[name].append(r)
        eng.boot_traces(params)
        rng = np.random.default_rng(7)
        sample = sorted(rng.choice(R, size=min(args.sample, R), replace=False).tolist())
        for i in sample:
            want = tracegen.bootstrap_packed(population, args.seed, i, n)[0]
            assert eng.fetch_trace(i).tobytes() == want.tobytes(), f"replica {i} differs from tracegen.bootstrap_packed"
    buf.free()

    def med(name, k):
        return float(np.median([r[k] for r in res[name]]))
    out = {"gpu": gpu, "workload": f"{n}-job traces x {R} replicas, 4x32x8, fifo+yarn (bench.py's step), span budget 1.5",
           "steps": args.steps, "warmup": args.warmup}
    for name in ("boot", "packed"):
        wall, events = med(name, 0), med(name, 4)
        out[name] = {"wall_ms_per_step": wall * 1e3, "engine_kernel_ms_per_step": med(name, 2), "summary_kernel_ms_per_step": med(name, 3),
                     "events_per_step": events, "e2e_events_per_s": events / wall}
    gen_ms = med("boot", 1)
    out["boot"].update(generator_kernel_ms_per_step=gen_ms, generator_bytes_written=32 * R * n,
                       generator_write_gb_per_s=32 * R * n / (gen_ms * 1e-3) / 1e9)
    out["packed"]["trace_bytes_uploaded"] = 32 * R * n
    out["checked_replicas"] = len(sample)
    out["gpu_after"] = gpu_info()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

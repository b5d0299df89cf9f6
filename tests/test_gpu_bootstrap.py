"""Bootstrap replicas generated on the H100 (gs_boot_population / gs_boot_traces / gs_fetch_trace, sweep.summarize_bootstrap).

Every generated trace is compared byte for byte with the numpy mirror tracegen.bootstrap_packed; a handle that
generates its traces must then compute exactly what a handle computes when it is given the mirror's traces through
gs_load_traces_packed; the error codes leave the handle working; and the sweep's bootstrap path must return the
records of the ordinary path run on bootstrap_table's replicas."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

RC = 1 << 16                       # explicit rows_cap: both handles of a comparison get the same result layout


@pytest.fixture(scope="module")
def pop():
    from gpuschedule_b200 import ingest, tracegen
    return ingest.table_from_columns(tracegen.synth_columns(3000, seed=3))


def clusters():
    from gpuschedule_b200 import capi
    return capi.make_cluster(4, 32, 8), capi.make_cluster(2, 16, 4, num_cpu_p_node=64, mem_p_node=256)


def policy(name, table):
    from gpuschedule_b200 import capi, policies
    if name == "gittins":
        return capi.make_policy(name, gittins_table=policies.build_gittins_table(policies.gittins_samples(table), 3250.0))
    if name == "dlas-gpu":
        return capi.make_policy(name, num_queue=3, queue_limit=(3600.0, 7200.0))
    return capi.make_policy(name)


def mirror(pop_table, p):
    from gpuschedule_b200 import tracegen
    return tracegen.bootstrap_packed(pop_table.packed(), int(p["seed"]), int(p["stream"]), int(p["n"]), int(p["gap_num"]), int(p["gap_den"]))[0]


def make_params(R, ns, scales, seed=11, stream0=0):
    from gpuschedule_b200 import capi
    p = np.zeros(R, dtype=capi.BOOT_PARAMS_DTYPE)
    for i in range(R):
        num, den = scales[i % len(scales)]
        p[i] = (seed, stream0 + i, ns[i % len(ns)], num, den)
    return p


def packed_block(traces):
    from gpuschedule_b200 import capi
    nmax = max(max(len(t) for t in traces), 1)
    block = np.zeros(len(traces) * nmax, dtype=capi.JOBIN_DTYPE)
    for i, t in enumerate(traces):
        block[i * nmax:i * nmax + len(t)] = t
    return block, nmax * capi.JOBIN_DTYPE.itemsize, np.array([len(t) for t in traces], dtype=np.int64)


def test_fetch_trace_equals_mirror_heterogeneous(pop):
    from gpuschedule_b200 import capi
    R = 72
    params = make_params(R, ns=(0, 1, 255, 256, 257, 1000, 3000, 2999), scales=((1, 1), (1, 2), (2, 1), (7, 3), (0, 1)))
    shapes = clusters()
    max_need = int(max(1.0, float(pop.duration.max()))) + 2
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, shapes[i % 2])
        eng.boot_population(pop)
        ms = eng.boot_traces(params, with_time=True)
        assert ms > 0
        want = [mirror(pop, params[i]) for i in range(R)]
        for i in range(R):
            assert eng.fetch_trace(i).tobytes() == want[i].tobytes(), i
        eng.run(max_ticks=1, rows_cap=0)              # one tick: enough to read the layout the load-time bounds gave
        for i in range(R):
            lay, w, M = eng.result_layout(i), want[i], shapes[i % 2].n_nodes
            last = int(w["arrive_tick"][-1]) if len(w) else 0
            assert lay.cap_ev == last + 2 * max_need + 4096, i                # last arrival tick from the kernel
            spans = int(np.minimum(w["gpus"] // w["gpu_per_task"], M).sum())
            assert lay.cap_spans == max(spans, 1), i                          # span-pool bound from the kernel


def compare_handles(gen, ref, name, R):
    """identical results of two handles after their runs (fifo: result blocks; others: rows, job records, finish order)"""
    a, b = gen.run_summarized(rows_cap=RC), ref.run_summarized(rows_cap=RC)
    assert a.tobytes() == b.tobytes()
    assert a["done"].all() and (a["finished"] > 0).any()
    if name == "fifo":
        la, lb = gen.result_layout(0), ref.result_layout(0)
        pitch = int(la.block_bytes)
        for i in range(R):
            assert bytes(gen.result_layout(i)) == bytes(ref.result_layout(i)), i
            pitch = max(pitch, int(gen.result_layout(i).block_bytes))
        ba, bb = np.zeros(pitch * R, dtype=np.uint8), np.zeros(pitch * R, dtype=np.uint8)
        gen.fetch_results(ba, pitch)
        ref.fetch_results(bb, pitch)
        gen.sync()
        ref.sync()
        for i in range(R):
            wa, wb = gen.window(i), ref.window(i)
            assert bytes(wa) == bytes(wb), i
            va = gen.result_views(ba, pitch, i, gen.result_layout(i), wa)
            vb = ref.result_views(bb, pitch, i, ref.result_layout(i), wb)
            for x, y in zip(va, vb):
                assert x.tobytes() == y.tobytes(), i
    else:
        for i in range(R):
            wa = gen.window(i)
            assert bytes(wa) == bytes(ref.window(i)), i
            cnt = int(wa.ticks - wa.row_first)
            assert gen.fetch_rows(i, int(wa.row_first), cnt).tobytes() == ref.fetch_rows(i, int(wa.row_first), cnt).tobytes(), i
            ra, oa = gen.fetch_jobs(i)
            rb, ob = ref.fetch_jobs(i)
            assert ra.tobytes() == rb.tobytes() and oa.tobytes() == ob.tobytes(), i
    return a


@pytest.mark.parametrize("name", ["fifo", "sjf", "dlas-gpu", "gittins"])
def test_generated_handle_runs_like_packed_upload(pop, name):
    from gpuschedule_b200 import capi
    R = 24
    params = make_params(R, ns=(1500, 700, 2000, 1), scales=((1, 1), (1, 2), (3, 2)), seed=5)
    traces = [mirror(pop, params[i]) for i in range(R)]
    shapes = clusters()
    pol = policy(name, pop)
    with capi.Engine(device=0, nsims=R) as gen, capi.Engine(device=0, nsims=R) as ref:
        for i in range(R):
            gen.config(i, shapes[i % 2], pol)
            ref.config(i, shapes[i % 2], pol)
        gen.boot_population(pop)
        gen.boot_traces(params)
        block, pitch, n_each = packed_block(traces)
        ref.load_traces_packed(block, pitch, n_each)
        first = compare_handles(gen, ref, name, R)
        gen.reset()
        ref.reset()
        second = compare_handles(gen, ref, name, R)
        assert first.tobytes() == second.tobytes()


def test_regenerate_and_replace(pop):
    from gpuschedule_b200 import capi
    R = 8
    params = make_params(R, ns=(500, 800), scales=((1, 1), (1, 3)), seed=21)
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, clusters()[0])
        eng.boot_population(pop)
        eng.boot_traces(params)
        first = [eng.fetch_trace(i).tobytes() for i in range(R)]
        eng.run_summarized()
        eng.boot_traces(params)
        assert [eng.fetch_trace(i).tobytes() for i in range(R)] == first
        other = params.copy()
        other["stream"][3] += 1000
        eng.boot_traces(other)
        got = [eng.fetch_trace(i).tobytes() for i in range(R)]
        assert got[3] != first[3] and got[3] == mirror(pop, other[3]).tobytes()
        assert got[:3] + got[4:] == first[:3] + first[4:]
        traces = [pop.packed()[i * 10:i * 10 + 100 + i] for i in range(R)]
        block, pitch, n_each = packed_block(traces)
        eng.load_traces_packed(block, pitch, n_each)
        assert [eng.fetch_trace(i).tobytes() for i in range(R)] == [t.tobytes() for t in traces]
        out = eng.run_summarized()
        assert out["n"].tolist() == n_each.tolist() and out["done"].all()


def test_error_codes_leave_the_handle_working(pop):
    from gpuschedule_b200 import capi
    lib = capi.load_library()
    R = 3
    good = make_params(R, ns=(400,), scales=((1, 1),), seed=2)

    def code(fn, *a):
        with pytest.raises(capi.GsError) as e:
            fn(*a)
        return e.value.code

    with capi.Engine(device=0, nsims=R) as eng:
        assert code(eng.boot_traces, good) == capi.GS_ERR_STATE                 # no population
        assert code(eng.boot_population, pop.packed()[:0]) == capi.GS_ERR_ARG    # k < 1
        assert lib.gs_boot_population(eng.h, None, 10) == capi.GS_ERR_ARG
        bad = pop.packed()[:50].copy()
        bad["arrive_tick"][20] = bad["arrive_tick"][19] - 1
        assert code(eng.boot_population, bad) == capi.GS_ERR_ARG                 # arrivals must not decrease
        bad = pop.packed()[:50].copy()
        bad["gpus"][7] = 3
        bad["gpu_per_task"][7] = 2
        assert code(eng.boot_population, bad) == capi.GS_ERR_ARG                 # gpus a multiple of gpu_per_task
        bad = pop.packed()[:50].copy()
        bad["duration"][3] = float(1 << 27)
        assert code(eng.boot_population, bad) == capi.GS_ERR_ARG                 # duration above 2^26 ticks
        eng.boot_population(pop)
        eng.config(0, clusters()[0])
        eng.config(1, clusters()[1])
        assert code(eng.boot_traces, good) == capi.GS_ERR_STATE                 # replica 2 not configured
        assert code(eng.fetch_trace, 0) == capi.GS_ERR_STATE                    # no trace yet
        assert lib.gs_fetch_trace(eng.h, R, None) == capi.GS_ERR_ARG
        eng.config(2, capi.make_cluster(4, 32, 8, enable_network_costs=True))
        assert code(eng.boot_traces, good) == capi.GS_ERR_ARG                   # network costs
        eng.config(2, clusters()[0])
        eng.boot_traces(good)
        before = [eng.fetch_trace(i).tobytes() for i in range(R)]
        for field, value in (("n", -1), ("n", 1 << 31), ("gap_num", -1), ("gap_den", 0)):
            p = good.copy()
            p[field][1] = value
            assert code(eng.boot_traces, p) == capi.GS_ERR_ARG, field
        assert lib.gs_boot_traces(eng.h, None, None) == capi.GS_ERR_ARG
        with pytest.raises(ValueError):
            eng.boot_traces(good[:2])
        assert [eng.fetch_trace(i).tobytes() for i in range(R)] == before   # refused calls changed nothing
        wide = pop.packed()[:100].copy()
        wide["arrive_tick"][50:] += 10 ** 6                                  # one gap of 10^6 ticks
        eng.boot_population(wide)
        p = good.copy()
        p["n"] = 2200                                                         # 2199 * 10^6 >= 2^31 - 1
        assert code(eng.boot_traces, p) == capi.GS_ERR_ARG
        p["n"], p["gap_num"], p["gap_den"] = 2200, 1, 2                       # 1.0995e9: allowed
        eng.boot_traces(p)
        assert eng.fetch_trace(1).tobytes() == mirror_packed(wide, p[1]).tobytes()
        eng.boot_population(pop)                  # (a run over a 10^9-tick horizon would size its rows by it)
        eng.boot_traces(good)
        assert [eng.fetch_trace(i).tobytes() for i in range(R)] == before
        out = eng.run_summarized()
        assert out["done"].all() and out["n"].tolist() == [400] * R


def mirror_packed(packed, p):
    from gpuschedule_b200 import tracegen
    return tracegen.bootstrap_packed(packed, int(p["seed"]), int(p["stream"]), int(p["n"]), int(p["gap_num"]), int(p["gap_den"]))[0]


@pytest.mark.parametrize("n", [None, 150])
def test_summarize_bootstrap_equals_the_ordinary_path(n):
    from gpuschedule_b200 import capi, sweep, tracegen
    trace = os.path.join(GOLDEN, "n64", "trace.csv")
    flag_sets = [sweep.make_flags(trace_file=trace, schedule=s, num_queue=2) for s in ("fifo", "sjf", "dlas-gpu", "gittins")]
    loads, R, seed = (1.0, 2.0, 0.5), 3, 7
    recs = sweep.summarize_bootstrap(flag_sets, R, loads, seed=seed, n=n)
    assert recs.shape == (len(flag_sets), len(loads), R)
    for c, (fl, infra, jm, pol) in enumerate(sweep._plain_setup(flag_sets)):
        for li, L in enumerate(loads):
            num, den = sweep.load_gap_scale(L)
            for r in range(R):
                table = tracegen.bootstrap_table(jm.table, seed, r, jm.table.n if n is None else n, num, den)
                with capi.Engine(device=0, nsims=1) as eng:
                    eng.config(0, infra.gs_cluster(), pol)
                    eng.load_trace(0, table)
                    want = eng.run_summarized()
                assert recs[c, li, r].tobytes() == want[0].tobytes(), (fl.schedule, L, r)
    assert (recs["finished"] > 0).all()


def test_sweep_cli_bootstrap(tmp_path):
    import csv
    from gpuschedule_b200 import summary, sweep
    trace = os.path.join(GOLDEN, "n64", "trace.csv")
    out, ci = str(tmp_path / "s.csv"), str(tmp_path / "ci.csv")
    sweep.main(["--trace", trace, "--schedule", "fifo", "sjf", "--bootstrap", "5", "--load", "1", "1.5", "--jobs", "80",
                "--seed", "3", "--summary", out, "--summary-ci", ci])
    with open(out) as f:
        rows = list(csv.DictReader(f))
    assert len(rows) == 2 * 2 * 5
    assert [r["replica"] for r in rows[:5]] == ["0", "1", "2", "3", "4"] and {r["n"] for r in rows} == {"80"}
    with open(ci) as f:
        lines = list(csv.DictReader(f))
    assert len(lines) == 4 and set(summary.spread_columns()) <= set(lines[0])
    assert all(float(x["makespan_lo"]) <= float(x["makespan_mean"]) <= float(x["makespan_hi"]) for x in lines)

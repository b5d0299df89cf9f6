"""The statistics kernels of gs_summary.cuh on the H100, past the regimes the feature tests reach.

* More replicas (pairs) than blocks: handles of more than 8 blocks x SMs replicas, so that every block of
  gs_sum_jobs_kernel / gs_jd_jobs_kernel / gs_cmp_pairs_kernel folds several replicas of different sizes with the
  same scratch slice, shared histograms, edges and class cursors -- fifo, the event-driven policies and the horus
  engine, with the summary, the timeline (1024 bins) and the job statistics (8 classes, 255 edges) on together.
* Four-pass selects: the long traces of test_stats_edges_cpu (waits spanning more than 2^27 ticks) under fifo, sjf and
  dlas-gpu and their compares in both orders, and designed jct multisets (ties, two values, ranks that share their
  top digits, values at 1 and 2^26) for k around the rank boundaries.
* 128-bit sums: memory near 2^45 per device, so mem_busy_sum, the timeline bins' memory and the sums of squares of
  jobdist and compare leave their low words, within one launch and across many windows.
* One bench-shaped step: bench.py's fifo replica count with the timeline and job statistics on.

Every integer field is compared bit for bit with the Python references over what the same handle hands out (rows,
job records, or the fifo engine's compact records where the rows are too many to expand), and every test first
asserts on the device's own output that its regime was reached."""
import math

import numpy as np
import pytest

from test_compare_cpu import assert_pair, reference_pair, run_cols
from test_gpu_summary import _engine_run
from test_jobdist_cpu import assert_jobdist, reference_jobdist
from test_stats_edges_cpu import (CMP_EDGES, JCT_KS, JD_BOUNDS, JD_EDGES, JOB_KINDS, LONG_B, LONG_PAIRS, LONG_W, ROW_FIELDS,
                                  fifo_configs, grid_bound, horus_configs, jct_trace, jct_values, long_cluster, long_policies,
                                  long_trace, policy_configs, records_bins, records_summary, select_passes, small_table)
from test_summary_cpu import assert_summary, job_columns, reference_summary
from test_timeline_cpu import assert_bins, reference_bins

pytestmark = pytest.mark.gpu

COUNT = 1100
TL_W, TL_B = 64, 1024


@pytest.fixture(scope="module")
def bound():
    """an upper bound on the grid any of the three job kernels launches on this device"""
    import torch
    b = grid_bound(torch.cuda.get_device_properties(0).multi_processor_count)
    assert COUNT > b, (COUNT, b)
    return b


def _sizes_precondition(tables, bound, big):
    n = np.array([t.n for t in tables])
    assert len(n) > bound and (n == 0).any() and (n == 1).any() and n.max() >= big
    for g in range(1, bound + 1):                     # replicas r and r + grid differ in size, whatever the grid
        assert (n[:-g] != n[g:]).any(), g


def _check_replica(i, table, summ, rows, jobs, tl, classes, hist, util=None):
    tag = f"replica {i} (n={table.n})"
    ref = reference_summary(rows, *jobs, util=util)
    assert_summary(summ, ref, tag, skip=() if util is not None else ("util_sum",))
    assert_bins(tl, reference_bins(rows, TL_W, TL_B, util=util), tag)
    assert_jobdist(classes, hist, reference_jobdist(*jobs, JD_BOUNDS, JD_EDGES), tag)


def _engine_handle(capi, configs):
    eng = capi.Engine(device=0, nsims=len(configs))
    for i, (cl, table, pol) in enumerate(configs):
        eng.config(i, cl, pol)
        eng.load_trace(i, table)
    eng.set_timeline(TL_W, TL_B)
    eng.set_jobdist(JD_BOUNDS, JD_EDGES)
    return eng


# ---------------------------------------------------------------- 1. more replicas than blocks
@pytest.mark.parametrize("kind", ["fifo", "policies"])
def test_engine_handle_of_more_replicas_than_blocks(bound, kind):
    from gpuschedule_b200 import capi
    configs = fifo_configs(COUNT) if kind == "fifo" else policy_configs(COUNT)
    tables = [t for _, t, _ in configs]
    _sizes_precondition(tables, bound, 100000)
    with _engine_handle(capi, configs) as eng:
        out, rows, _ = _engine_run(eng)
        tl = eng.timeline()
        classes, hist = eng.jobdist()
        fin = out["finished"]
        assert (fin == 0).any() and (fin == 1).any() and fin.max() >= 10000 and (out["status"] == 0).all()
        for i, (_, table, _) in enumerate(configs):
            recs, order = eng.fetch_jobs(i)
            assert out[i]["n"] == table.n and out[i]["done"] == 1
            _check_replica(i, table, out[i], rows[i], job_columns(table, recs, order), tl[i], classes[i], hist[i])
        # a sub-range with first > 0 and more replicas than blocks: the job part again, the same bits
        first, count = 5, COUNT - 9
        assert count > bound
        part = eng.summarize(first, count)
        assert part.tobytes() == out[first:first + count].tobytes()
        pc, ph = eng.jobdist(first, count)
        assert pc.tobytes() == classes[first:first + count].tobytes() and ph.tobytes() == hist[first:first + count].tobytes()


def test_horus_handle_of_more_replicas_than_blocks(bound):
    from gpuschedule_b200 import capi
    configs = horus_configs(COUNT)
    tables = [t for _, t, _ in configs]
    _sizes_precondition(tables, bound, 300)
    np.random.seed(3)
    words = np.random.randint(0, 2 ** 32, size=64 << 20, dtype=np.uint32)      # one stream, read by every replica
    with capi.HorusEngine(device=0, nsims=COUNT) as eng:
        for i, (cl, table, params) in enumerate(configs):
            eng.config(i, cl, params)
            eng.load_trace(i, table)
        eng.load_words(-1, words)
        eng.set_timeline(TL_W, TL_B)
        eng.set_jobdist(JD_BOUNDS, JD_EDGES)
        for _ in range(1000):
            eng.run(rows_cap=1 << 16)
            if all(eng.stats(i).done for i in range(COUNT)):
                break
        out = eng.summarize()
        tl = eng.timeline()
        classes, hist = eng.jobdist()
        fin = out["finished"]
        assert (fin == 0).any() and (fin == 1).any() and fin.max() >= 250 and (out["status"] == 0).all()
        for i, table in enumerate(tables):
            rows, util, _, recs, order = eng.fetch(i)
            _check_replica(i, table, out[i], rows, job_columns(table, recs, order), tl[i], classes[i], hist[i], util=util)
        first, count = 3, COUNT - 4
        assert eng.summarize(first, count).tobytes() == out[first:first + count].tobytes()


def _pairs(n_traces, n_self):
    """(a, b) pairs over replicas 3t (fifo / horus), 3t + 1 (sjf / gandiva), 3t + 2 (dlas-gpu / horus): both orders, and
    self-pairs"""
    pa, pb = [], []
    for t in range(n_traces):
        for x, y in ((0, 1), (1, 0), (0, 2), (2, 0)):
            pa.append(3 * t + x)
            pb.append(3 * t + y)
    for t in range(n_self):
        pa.append(3 * t + 1)
        pb.append(3 * t + 1)
    return pa, pb


def _check_pairs(recs, hist, pa, pb, tables, jobs_of, bound):
    assert len(pa) > bound
    selfs = 0
    for p, (a, b) in enumerate(zip(pa, pb)):
        t = tables[a // 3]
        (ra, fa), (rb, fb) = jobs_of(a), jobs_of(b)
        assert_pair(recs[p], hist[p], reference_pair(t.arrive_tick, t.gpus, run_cols(ra), fa, run_cols(rb), fb, JD_BOUNDS, CMP_EDGES), f"pair {p} ({a}, {b})")
        if a == b:
            selfs += 1
            assert (recs[p]["eq"] == recs[p]["jobs"][:, None]).all() and not recs[p]["q_hi"].any()
    assert selfs > 0


def test_engine_compare_of_more_pairs_than_blocks(bound):
    from gpuschedule_b200 import capi
    n_traces = 300
    sizes = [int(x) for x in np.random.default_rng(21).integers(2, 200, n_traces)]
    sizes[2], sizes[4], sizes[6] = 0, 1, 20000
    tables = [small_table(n, 2100 + i) for i, n in enumerate(sizes)]
    configs = []
    for i, t in enumerate(tables):
        cl = capi.make_cluster(1, 4, 8) if t.n < 1000 else capi.make_cluster(4, 32, 8)
        configs += [(cl, t, None), (cl, t, capi.make_policy("sjf")), (cl, t, capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,)))]
    pa, pb = _pairs(n_traces, 100)
    with capi.Engine(device=0, nsims=len(configs)) as eng:
        for i, (cl, t, pol) in enumerate(configs):
            eng.config(i, cl, pol)
            eng.load_trace(i, t)
        out = eng.run_summarized()
        assert (out["status"] == 0).all() and (out["finished"] == 0).any()
        recs, hist = eng.compare(pa, pb, JD_BOUNDS, CMP_EDGES)
        jobs = {}
        _check_pairs(recs, hist, pa, pb, tables, lambda r: jobs.setdefault(r, eng.fetch_jobs(r)), bound)


def test_horus_compare_of_more_pairs_than_blocks(bound):
    from gpuschedule_b200 import capi
    n_traces = 280
    sizes = [int(x) for x in np.random.default_rng(22).integers(2, 120, n_traces)]
    sizes[2], sizes[4], sizes[6] = 0, 1, 300
    tables = [small_table(n, 2200 + i) for i, n in enumerate(sizes)]
    kinds = (("horus", "horus", 5, 1), ("gandiva", "gandiva", 5, 1), ("horus+", "horus+", 5, 3))
    np.random.seed(4)
    words = np.random.randint(0, 2 ** 32, size=64 << 20, dtype=np.uint32)
    pa, pb = _pairs(n_traces, 100)
    with capi.HorusEngine(device=0, nsims=3 * n_traces) as eng:
        for i, t in enumerate(tables):
            for k, (scheme, sched, nbuf, nq) in enumerate(kinds):
                eng.config(3 * i + k, capi.make_cluster(1, 3 + i % 3, 8), capi.make_horus_params(scheme, sched, nbuf, nq))
                eng.load_trace(3 * i + k, t)
        eng.load_words(-1, words)
        for _ in range(1000):
            eng.run(rows_cap=1 << 16)
            if all(eng.stats(i).done for i in range(3 * n_traces)):
                break
        recs, hist = eng.compare(pa, pb, JD_BOUNDS, CMP_EDGES)
        fetched = {}

        def jobs_of(r):
            if r not in fetched:
                _, _, _, hr, fo = eng.fetch(r)
                fetched[r] = (hr, fo)
            return fetched[r]
        _check_pairs(recs, hist, pa, pb, tables, jobs_of, bound)


# ---------------------------------------------------------------- 2 + 3. long runs: four passes, 128-bit sums
def _run_long(eng, fifo, rows_cap):
    """run to the end, summarising after every launch: (summaries, per replica the windows [(ev, qr, ticks, wm)] of the
    fifo engine's compact records, per replica the rows of the event-driven policies); fifo[s]: replica s runs fifo"""
    from gpuschedule_b200.log_manager import ROW_DTYPE
    nsims = len(fifo)
    wins = [[] for _ in range(nsims)]
    rows = [[] for _ in range(nsims)]
    wm = [0] * nsims
    for _ in range(100000):
        eng.run(0, rows_cap)
        out = eng.summarize()
        for s in range(nsims):
            w = eng.window(s)
            if eng.stats(s).ticks == 0:
                continue
            if fifo[s]:
                ww, ev, qr, _, _, _, _, _ = eng.fetch_compact(s)
                wins[s].append((ev.copy(), qr.copy(), int(ww.ticks), wm[s]))
                wm[s] = int(ww.ticks)
            elif w.ticks > w.row_first:
                rows[s].append(eng.fetch_rows(s, w.row_first, w.ticks - w.row_first))
        if out["done"].all():
            return out, wins, [np.concatenate(r) if r else np.zeros(0, dtype=ROW_DTYPE) for r in rows]
    raise AssertionError("the run did not end")


@pytest.fixture(scope="module")
def long_handle():
    """the long trace as fifo on 2 and 32 nodes and as sjf / dlas-gpu on 2 nodes, summarised with the timeline and the
    job statistics, one launch per 4096 records; and fifo on 2 nodes again in 8-record windows"""
    from gpuschedule_b200 import capi
    table = long_trace()
    names = ["fifo", "fifo32", "sjf", "dlas-gpu"]
    pols = dict(long_policies())
    res = {}
    for tag, nm, cap in (("one", names, 4096), ("many", ["fifo"], 8)):
        eng = capi.Engine(device=0, nsims=len(nm))
        for i, name in enumerate(nm):
            eng.config(i, long_cluster(32 if name == "fifo32" else 2), pols.get(name))
            eng.load_trace(i, table)
        eng.set_timeline(LONG_W, LONG_B)
        eng.set_jobdist(JD_BOUNDS, JD_EDGES)
        out, wins, rows = _run_long(eng, [name.startswith("fifo") for name in nm], cap)
        jobs = [eng.fetch_jobs(i) for i in range(len(nm))]
        res[tag] = dict(eng=eng, names=nm, out=out, wins=wins, rows=rows, jobs=jobs, tl=eng.timeline(), jd=eng.jobdist())
    yield table, res
    for r in res.values():
        r["eng"].close()


def test_long_runs_four_pass_summaries_and_high_words(long_handle):
    table, res = long_handle
    for tag, r in res.items():
        for i, name in enumerate(r["names"]):
            s, (recs, order) = r["out"][i], r["jobs"][i]
            jobs = job_columns(table, recs, order)
            assert s["finished"] == table.n and s["status"] == 0, (tag, name)
            # the regime, from the device's own output: the range of the waits or turnarounds (at least max - median)
            # needs four passes, and fifo's memory (a row per tick; the policies write a row per event) leaves 64 bits
            if name != "fifo32":
                assert select_passes(max(int(s[f][4]) - int(s[f][0]) for f in ("wait_q", "turnaround_q"))) == 4, (tag, name)
            if name.startswith("fifo"):
                assert int(s["mem_busy_hi"]) > 0, (tag, name)
            if name.startswith("fifo"):
                want = records_summary(r["wins"][i])
                want.update({k: v for k, v in reference_summary(r["rows"][i][:0], *jobs).items() if k not in ROW_FIELDS})
                bins = records_bins(r["wins"][i], LONG_W, LONG_B)
            else:
                want = reference_summary(r["rows"][i], *jobs)
                bins = reference_bins(r["rows"][i], LONG_W, LONG_B)
            assert_summary(s, want, f"{tag} {name}", skip=("util_sum",))
            assert_bins(r["tl"][i], bins, f"{tag} {name}", rel=1e-9)
            if name == "fifo":
                assert int(r["tl"][i]["mem_busy_hi"].max()) > 0, (tag, name)
            classes, hist = r["jd"][0][i], r["jd"][1][i]
            assert_jobdist(classes, hist, reference_jobdist(*jobs, JD_BOUNDS, JD_EDGES), f"{tag} {name}")
            if name == "fifo":
                assert int(classes["wait_sq_hi"].max()) > 0 and int(classes["turnaround_sq_hi"].max()) > 0, (tag, name)
    assert len(res["many"]["wins"][0]) > 8
    one, many = res["one"]["out"][0], res["many"]["out"][0]
    assert all(np.array_equal(one[f], many[f]) for f in one.dtype.names if f not in ("avg_pending_sum", "util_sum"))
    assert math.isclose(one["avg_pending_sum"], many["avg_pending_sum"], rel_tol=1e-12)


def test_long_compares_four_passes_both_ways(long_handle):
    table, res = long_handle
    r = res["one"]
    idx = {name: i for i, name in enumerate(r["names"])}
    pa = [idx[a] for a, _ in LONG_PAIRS]
    pb = [idx[b] for _, b in LONG_PAIRS]
    for bounds, edges in (((), ()), (JD_BOUNDS, CMP_EDGES)):
        recs, hist = r["eng"].compare(pa, pb, bounds, edges)
        for p, (a, b) in enumerate(LONG_PAIRS):
            (ra, fa), (rb, fb) = r["jobs"][idx[a]], r["jobs"][idx[b]]
            assert_pair(recs[p], hist[p], reference_pair(table.arrive_tick, table.gpus, run_cols(ra), fa, run_cols(rb), fb, bounds, edges),
                        f"{a},{b} {bounds}")
            if bounds or a == b:
                continue
            q = recs[p][0]
            # device precondition: the wait differences span more than 2^27, so q_hi and q_lo each took four passes
            assert select_passes(int(q["q_hi"][0][4]) - int(q["q_lo"][0][4])) == 4, (a, b)
            if {a, b} <= {"fifo", "sjf", "dlas-gpu"}:
                assert q["lt"][0] > 0 and q["gt"][0] > 0, (a, b)
            if {a, b} == {"fifo", "fifo32"}:
                assert int(q["d_sq_hi"][0]) > 0 and int(q["d_sq_hi"][1]) > 0, (a, b)


def test_designed_jct_multisets():
    """ties, two values, ranks sharing their top digits, values at 1 and 2^26, for k at the rank boundaries"""
    from gpuschedule_b200 import capi
    cases = [(kind, k) for kind in JOB_KINDS for k in JCT_KS]
    with capi.Engine(device=0, nsims=len(cases)) as eng:
        tables = []
        for i, (kind, k) in enumerate(cases):
            tables.append(jct_trace(kind, k))
            eng.config(i, long_cluster(1))
            eng.load_trace(i, tables[-1])
        eng.set_jobdist(JD_BOUNDS, JD_EDGES)
        out, wins, _ = _run_long(eng, [True] * len(cases), 1 << 14)
        classes, hist = eng.jobdist()
        for i, ((kind, k), table) in enumerate(zip(cases, tables)):
            s = out[i]
            tag = f"{kind} k={k}"
            v = np.sort(jct_values(kind, k))
            ranks = [(q * k + 999) // 1000 - 1 for q in (500, 900, 950, 990, 1000)]
            assert s["finished"] == k and s["jct_q"].tolist() == v[ranks].tolist(), tag     # the designed multiset went through
            if kind == "extremes":
                assert s["jct_q"][4] == 2 ** 26 and (k == 1 or s["jct_q"][0] == 1), tag
            if kind == "shared" and k >= 255:
                u = s["jct_q"][:3].astype(np.int64) - 1
                assert len(set((u >> 9).tolist())) == 1 and len(set(u.tolist())) == 3, tag
            recs, order = eng.fetch_jobs(i)
            jobs = job_columns(table, recs, order)
            want = records_summary(wins[i])
            want.update({key: val for key, val in reference_summary(np.zeros(0, dtype=_rows_dtype()), *jobs).items() if key not in ROW_FIELDS})
            assert_summary(s, want, tag, skip=("util_sum",))
            assert_jobdist(classes[i], hist[i], reference_jobdist(*jobs, JD_BOUNDS, JD_EDGES), tag)


def _rows_dtype():
    from gpuschedule_b200.log_manager import ROW_DTYPE
    return ROW_DTYPE


# ---------------------------------------------------------------- 4. one bench-shaped step
def test_bench_shaped_step():
    """bench.py's fifo replica count and cluster, traces shrunk to 2000 jobs, summary + timeline + job statistics;
    every replica's finished / n / status, and a seeded sample of 40 replicas in full"""
    import bench
    from gpuschedule_b200 import capi
    R, n = bench.CONFIGS["c1"]["replicas"], 2000
    cluster = capi.make_cluster(4, 32, 8)
    tables = [bench.fast_table(n, bench.BASE_SEED + r) for r in range(R)]
    with capi.Engine(device=0, nsims=R) as eng:
        for r in range(R):
            eng.config(r, cluster)
            eng.load_trace_packed(r, tables[r].packed())
        eng.set_timeline(TL_W, TL_B)
        eng.set_jobdist(JD_BOUNDS, JD_EDGES)
        out, rows, _ = _engine_run(eng)
        assert (out["n"] == n).all() and (out["finished"] == n).all() and (out["status"] == 0).all() and (out["done"] == 1).all()
        tl = eng.timeline()
        classes, hist = eng.jobdist()
        for i in sorted(np.random.default_rng(2026).choice(R, 40, replace=False).tolist()):
            recs, order = eng.fetch_jobs(i)
            _check_replica(i, tables[i], out[i], rows[i], job_columns(tables[i], recs, order), tl[i], classes[i], hist[i])

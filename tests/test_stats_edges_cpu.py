"""Inputs that drive the statistics kernels of gs_summary.cuh into their rare regimes, and proof on the CPU that they do.

Three pieces of the kernels only run on the device, so their host builds never meet them: the grid-stride loops of
gs_sum_jobs_kernel / gs_jd_jobs_kernel / gs_cmp_pairs_kernel (a block that folds a second replica or pair), the radix
select's fourth pass (value ranges of 2^27 and more), and the high words of the 128-bit sums.  The builders below make
traces that reach each regime; test_gpu_stats_edges.py runs them on the device.  Here every builder is checked to
reach its regime -- 28-bit value ranges, both select directions of a compare at four passes, totals above 2^64, more
replicas than any grid -- so that a change to a builder cannot quietly weaken the GPU tests, and the same inputs run
through the host builds (summary_emu, timeline_emu, jobdist_emu, compare_emu) against the numpy / Python-int
references of test_summary_cpu, test_timeline_cpu, test_jobdist_cpu and test_compare_cpu.

The long fifo runs last about 2^30 ticks, too many rows to expand, so their row part is judged by
`records_summary` / `records_bins`: the rows of the fifo engine's compact records (include/gsched.h, gs_evrow) summed
in closed form with Python integers.  That fold is itself checked against the expanded rows of the fixtures."""
import ctypes as C
import math

import numpy as np
import pytest

from conftest import golden_cases, load_golden
from test_compare_cpu import DIFF_EDGES, assert_pair, emu_pair, reference_pair, run_cols
from test_jobdist_cpu import assert_jobdist, emu_jobdist, reference_jobdist
from test_summary_cpu import FLOAT_FIELDS, add_jobs, assert_summary, job_columns, reference_summary
from test_timeline_cpu import INT_FIELDS, assert_bins, reference_bins

TWO64 = 1 << 64
CAP_GIB = 2 ** 16                 # gpu_memory_capacity of the big-memory clusters: 2^46-byte devices
BIG_MEM = 2 ** 45                 # memory_max near this counts in full (below the cap minus 500 MiB)
JD_BOUNDS = (1, 2, 3, 4, 8, 16, 32)                           # eight classes, the most gs_set_jobdist takes
JD_EDGES = tuple(int(x) for x in np.unique(np.round(np.geomspace(1, 2 ** 31 - 1, 255))).tolist())
CMP_EDGES = DIFF_EDGES
ROW_FIELDS = ("rows", "makespan", "busy_gpus_sum", "running_sum", "queued_sum", "busy_gpus_max", "running_max", "queued_max",
              "pend_max_max", "pend_sum_sum", "mem_busy_sum", "pending_rows", "avg_pending_sum")
JOB_KINDS = ("tied", "two", "shared", "extremes")
JCT_KS = (1, 2, 255, 256, 257, 999, 1000, 1001)


# ---------------------------------------------------------------- regime predicates
def select_passes(span):
    """radix passes of gs_sum_select for a value range `span` (gs_sum_passes): ceil(max(1, bit length) / 9)"""
    return (max(1, int(span).bit_length()) + 8) // 9


def summary_span(jobs):
    """the largest range of wait / turnaround / jct over finished jobs (arrive, gpus, start, end, jct, preempt)"""
    arrive, _, start, end, jct, _ = (np.asarray(a, dtype=np.int64) for a in jobs)
    if len(start) == 0:
        return 0
    return max(int(v.max() - v.min()) for v in (start - arrive, end - arrive, jct))


def pair_span(arrive, run_a, fin_a, run_b, fin_b):
    """the largest range of the three differences d = x_b - x_a over the jobs finished in both runs (one class)"""
    both = np.intersect1d(np.asarray(fin_a), np.asarray(fin_b))
    if len(both) == 0:
        return 0, 0, 0
    va = [np.asarray(x, dtype=np.int64)[both] for x in run_a]
    vb = [np.asarray(x, dtype=np.int64)[both] for x in run_b]
    d = [vb[0] - va[0], vb[1] - va[1], vb[2] - va[2]]
    return max(int(x.max() - x.min()) for x in d), int((d[0] < 0).sum()), int((d[0] > 0).sum())


def grid_bound(sms):
    """an upper bound on the grid of the three job kernels: 256 threads and >= 30 KB of shared memory per block leave
    at most 8 blocks on an SM (228 KB of shared memory, 2048 threads)"""
    return 8 * sms


# ---------------------------------------------------------------- trace builders (shared with test_gpu_stats_edges.py)
def make_table(arrive, gpus, duration, mem_bytes=None, seed=0):
    """a JobTable from columns (one GPU per task, synthetic utilisation columns for the horus engine)"""
    from gpuschedule_b200 import ingest
    n = len(arrive)
    rng = np.random.default_rng(seed)
    ua = np.round(rng.uniform(5.0, 90.0, n), 3)
    if mem_bytes is None:
        mem_bytes = rng.integers(512, 16384, n, endpoint=True).astype(np.int64) << 20
    a = np.asarray(arrive, dtype=np.int32)
    return ingest.JobTable(n=n, label=[str(i) for i in range(n)], num_gpu_text=None, arrive_tick=a, submit=a.copy(),
                           gpus=np.asarray(gpus, dtype=np.int32), gpu_per_task=np.ones(n, dtype=np.int32),
                           duration=np.ascontiguousarray(duration, dtype=np.float64), mem_bytes=np.asarray(mem_bytes, dtype=np.int64),
                           util_avg=ua, util_max=np.minimum(100.0, ua + np.round(rng.uniform(1.0, 30.0, n), 3)))


def long_cluster(nodes=2):
    """8-GPU nodes whose devices hold BIG_MEM-byte tasks in full"""
    from gpuschedule_b200 import capi
    return capi.make_cluster(1, nodes, 8, gpu_memory_capacity=CAP_GIB)


def long_trace(seed=0, n_long=60, n_short=24):
    """node-wide jobs of 2^25 .. 2^26 - 4 ticks and short jobs, all queued within the first 64 ticks, every job with
    memory_max near 2^45.  On two nodes the queue drains for about 2^30.5 ticks (below 2^31 whatever the draw: at most
    30 long jobs per node), so waits and turnarounds span more than 2^27 (four radix passes), their squares sum past
    2^64, and a row holds 16 * 2^45 bytes, so mem_busy_sum leaves 64 bits within 2^15 rows.  Jobs are node-wide, not
    cluster-wide: the engines stop when nothing runs and nothing is left to arrive, so a queue behind cluster-wide
    jobs would end the run at the first completion."""
    rng = np.random.default_rng(1000 + seed)
    n = n_long + n_short
    big = rng.permutation(np.r_[np.ones(n_long, dtype=bool), np.zeros(n_short, dtype=bool)])
    gpus = np.where(big, 8, rng.choice([1, 2, 4], n))
    dur = np.where(big, rng.integers(2 ** 25, 2 ** 26 - 4, n), rng.integers(1, 4096, n)).astype(np.float64)
    dur[np.flatnonzero(big)[0]] = 2 ** 26 - 4
    dur[np.flatnonzero(~big)[0]] = 0.25                          # a run length of max(1, ceil(0.25)) = 1
    arrive = np.sort(rng.integers(0, 64, n))
    mem = rng.integers(BIG_MEM - 2 ** 40, BIG_MEM, n)
    return make_table(arrive, gpus, dur, mem, seed=seed)


def long_policies():
    """(name, policy) of the event-driven schedules that reorder the long trace"""
    from gpuschedule_b200 import capi
    return [("sjf", capi.make_policy("sjf")), ("dlas-gpu", capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,)))]


def jct_values(kind, k, seed=0):
    """k designed job lengths (ticks, 1 .. 2^26) for the radix select:
    tied     -- one value k times;
    two      -- two values, the larger from rank 90 % on;
    shared   -- the 50 / 90 / 95 % ranks share the top two 9-bit digits (of three) and split in the last;
    extremes -- values at 1 and at 2^26 (the top 1 % and at least one at 2^26)"""
    rng = np.random.default_rng(7 * k + JOB_KINDS.index(kind))
    if kind == "tied":
        return np.full(k, 12345)
    if kind == "two":
        v = np.full(k, 3)
        v[(9 * k) // 10:] = 2 ** 22 + 1
        return rng.permutation(v)
    if kind == "shared":
        top = (77 << 18) | (300 << 9)                            # u = v - 1: digits 77, 300, then the low digit splits
        v = np.empty(k, dtype=np.int64)
        lo, hi = k // 3, k - k // 40
        v[:lo] = rng.integers(1, 2 ** 17, lo)
        v[lo:hi] = 1 + top + rng.integers(0, 512, hi - lo)
        v[hi:] = 1 + (200 << 18) + rng.integers(0, 2 ** 18, k - hi)
        v[0] = 1
        return rng.permutation(v)
    v = np.ones(k, dtype=np.int64)
    v[k - max(1, k // 100):] = 2 ** 26
    return rng.permutation(v)


def jct_trace(kind, k):
    """one 1-GPU job per designed value, arriving one per tick in ascending order of length on an 8-GPU node (fifo's
    jct is max(1, ceil(duration)) whatever the waits; the longest jobs come last, so a job is still running or still
    to arrive at every completion and the run does not stop early)"""
    v = np.sort(jct_values(kind, k))
    dur = v.astype(np.float64) - 0.5                                # ceil(v - 0.5) = v
    return make_table(np.arange(k), np.ones(k), dur, seed=k)


def replica_sizes(count, seed, big=100000):
    """job counts of a many-replica handle: pseudo-random 2 .. 160, with 0 and 1 early and late, and a `big`-job
    replica followed by small ones"""
    rng = np.random.default_rng(seed)
    s = rng.integers(2, 161, count)
    s[3], s[5], s[7], s[count - 2], s[count - 5] = 0, 1, big, 0, 1
    return s


def small_table(n, seed):
    """a synthetic n-job trace (bench.fast_table), or an empty one"""
    from bench import fast_table
    if n == 0:
        return make_table([], [], [], seed=seed)
    return fast_table(int(n), int(seed))


def fifo_configs(count, seed=11, big=100000):
    """(cluster, table, None) per replica: fifo on clusters of 8 to 256 GPUs"""
    from gpuschedule_b200 import capi
    clusters = [capi.make_cluster(1, 2, 8), capi.make_cluster(1, 4, 8), capi.make_cluster(2, 8, 8), capi.make_cluster(4, 8, 8)]
    return [(clusters[i % 4] if n < 1000 else capi.make_cluster(4, 32, 8), small_table(n, seed * 100000 + i), None)
            for i, n in enumerate(replica_sizes(count, seed, big).tolist())]


def policy_configs(count, seed=12, big=100000):
    """(cluster, table, policy) per replica: sjf / dlas-gpu / gittins in turn (sjf for empty traces)"""
    from gpuschedule_b200 import capi, policies
    out = []
    for i, n in enumerate(replica_sizes(count, seed, big).tolist()):
        table = small_table(n, seed * 100000 + i)
        sched = "sjf" if n == 0 else ("sjf", "dlas-gpu", "gittins")[i % 3]
        kw = dict(num_queue=2, queue_limit=(3600,)) if sched == "dlas-gpu" else {}
        if sched == "gittins":
            kw["gittins_table"] = policies.build_gittins_table(policies.gittins_samples(table), 3250.0)
        cl = capi.make_cluster(1, 4 + 4 * (i % 2), 8) if n < 1000 else capi.make_cluster(4, 32, 8)
        out.append((cl, table, capi.make_policy(sched, **kw)))
    return out


HORUS_KINDS = (("horus", "horus", 5, 1), ("horus+", "horus+", 5, 3), ("gandiva", "gandiva", 5, 1))


def horus_configs(count, seed=13, big=300):
    """(cluster, table, params) per replica: horus / horus+ / gandiva in turn on 3- to 6-node clusters (the horus
    engine steps every tick and scores the whole queue, so its largest replica stays at a few hundred jobs)"""
    from gpuschedule_b200 import capi
    out = []
    for i, n in enumerate(replica_sizes(count, seed, big).tolist()):
        scheme, sched, nbuf, nq = HORUS_KINDS[i % 3]
        cl = capi.make_cluster(1, 3 + i % 4, 8)
        out.append((cl, small_table(n, seed * 100000 + i), capi.make_horus_params(scheme, sched, nbuf, nq)))
    return out


# ---------------------------------------------------------------- the rows of compact fifo records, in closed form
def record_segments(ev, qr, ticks, wm):
    """(v_lo, v_hi, record, arrive_sum, oldest) of the rows v_lo .. v_hi (`delta`) each record of one window describes,
    rows with delta <= wm (folded by an earlier window) left out: record k stands for the ticks now_k .. now_(k+1) - 1,
    the last one up to `ticks`; its queue statistics are the gs_qrow with the same `now`"""
    q = {int(r["now"]): (int(r["arrive_sum"]), int(r["oldest_arrive"])) for r in qr}
    out = []
    for k in range(len(ev)):
        e = ev[k]
        lo = max(int(e["now"]), wm + 1)
        hi = int(ev[k + 1]["now"]) - 1 if k + 1 < len(ev) else int(ticks)
        if hi >= lo:
            a, o = q[int(e["now"])] if int(e["queued"]) > 0 else (0, 0)
            out.append((lo, hi, e, a, o))
    return out


def _fold(d, lo, hi, e, a, o):
    """add the rows lo .. hi of one record to a dict of row fields (Python ints; avg_pending_sum as a float)"""
    L = hi - lo + 1
    d["rows"] += L
    for f, col in (("busy_gpus", "busy_gpus"), ("running", "running"), ("queued", "queued")):
        d[f + "_sum"] += int(e[col]) * L
        d[f + "_max"] = max(d[f + "_max"], int(e[col]))
    d["mem_busy_sum"] += int(e["mem_busy_bytes"]) * L
    q = int(e["queued"])
    if q > 0:
        x = q * ((lo + hi) * L // 2) - L * a                    # the sum over v of the pending sum q * v - arrive_sum
        d["pend_sum_sum"] += x
        d["pend_max_max"] = max(d["pend_max_max"], hi - o)
        zero = a % q == 0 and lo <= a // q <= hi
        nz = L - (1 if zero else 0)
        d["pending_rows"] += nz
        if nz:
            d["avg_pending_sum"] += x / (q + 1e-9)


def records_summary(windows):
    """the row part of gs_summary (reference_summary's row keys) from [(ev, qr, ticks, wm)] windows"""
    d = dict.fromkeys(ROW_FIELDS, 0)
    d["avg_pending_sum"] = 0.0
    for ev, qr, ticks, wm in windows:
        for seg in record_segments(ev, qr, ticks, wm):
            _fold(d, *seg)
            d["makespan"] = seg[1]
    return d


def records_bins(windows, W, B):
    """reference_bins of the rows the windows' records describe (every record split at the bin boundaries)"""
    out = []
    for _ in range(B):
        d = dict.fromkeys(INT_FIELDS, 0)
        d["avg_pending_sum"] = 0.0
        out.append(d)
    for ev, qr, ticks, wm in windows:
        for lo, hi, e, a, o in record_segments(ev, qr, ticks, wm):
            v = lo
            while v <= hi:
                b = min(v // W, B - 1)
                end = hi if b == B - 1 else min(hi, (b + 1) * W - 1)
                d = out[b]
                if d["rows"] == 0:
                    d["delta_min"] = v
                d["delta_max"] = end
                d["finished_last"] = int(e["finished"])
                saved = d["rows"]
                _fold(d, v, end, e, a, o)
                assert d["rows"] > saved
                v = end + 1
    return out


def tight2_windows(t2, **run_kw):
    """run the Tight2 yardstick to the end in windows: ([(ev, qr, ticks, wm)], job records, finish order, last window)"""
    import oracle
    from gpuschedule_b200 import log_manager as lm
    t2.restart()
    wins, wm = [], 0
    while True:
        rc, w, _, _, done = t2.run_window(**run_kw)
        assert rc == 0
        wins.append((t2.ev[:w.ev_rows].copy(), t2.qr[:w.q_rows].copy(), int(w.ticks), wm))
        wm = int(w.ticks)
        if done or t2.n == 0:
            break
    n = t2.n
    both = np.ctypeslib.as_array(C.cast(oracle.lib().tight2_jobs(t2.h), C.POINTER(C.c_int32)), shape=(max(n, 1) * 2,)).reshape(-1, 2)[:n]
    jobs = np.zeros(n, dtype=lm.JOBRUN_DTYPE)
    jobs["start"] = both[:, 0]
    recs = lm.expand_jobs(jobs, int(w.admitted), t2.cols[3])
    nf = int(w.finished)
    order = np.ctypeslib.as_array(C.cast(oracle.lib().tight2_finish_order(t2.h), C.POINTER(C.c_int32)), shape=(max(nf, 1),))[:nf].copy()
    return wins, recs, order, w


# ---------------------------------------------------------------- host builds
def _build(tmp_path_factory, name):
    import os
    import subprocess
    from conftest import REPO
    out = str(tmp_path_factory.mktemp(name) / f"lib{name}.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", f"{name}.cpp")], check=True)
    return C.CDLL(out)


@pytest.fixture(scope="module")
def emus(tmp_path_factory):
    libs = {name: _build(tmp_path_factory, name) for name in ("summary_emu", "timeline_emu", "jobdist_emu", "compare_emu")}
    libs["jobdist_emu"].emu_jd_jobs.restype = C.c_int
    libs["compare_emu"].emu_cmp_pair.restype = C.c_int
    return libs


def _p(a):
    return np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def emu_windows(libs, windows, W, B):
    """the summary accumulator and timeline bins the host build folds from the windows' records"""
    from gpuschedule_b200.capi import SUMMARY_DTYPE, TBIN_DTYPE
    acc = np.zeros(1, dtype=SUMMARY_DTYPE)
    bins = np.zeros(B, dtype=TBIN_DTYPE)
    for ev, qr, ticks, wm in windows:
        libs["summary_emu"].emu_sum_compact(_p(ev), C.c_longlong(len(ev)), _p(qr), C.c_longlong(len(qr)), C.c_longlong(wm),
                                            C.c_longlong(ticks), _p(acc))
        libs["timeline_emu"].emu_tl_compact(_p(ev), C.c_int(len(ev)), _p(qr), C.c_int(len(qr)), C.c_longlong(ticks), C.c_longlong(wm),
                                            C.c_longlong(W), C.c_int(B), _p(bins))
    return acc, bins


def _row_dtype():
    from gpuschedule_b200.log_manager import ROW_DTYPE
    return ROW_DTYPE


# ---------------------------------------------------------------- the closed-form record fold against expanded rows
@pytest.mark.parametrize("case", golden_cases())
def test_records_fold_equals_expanded_rows(case):
    import oracle
    table, cluster, _, _, _ = load_golden(case)
    if cluster.enable_network_costs:
        pytest.skip("the record yardstick runs the plain fifo + yarn tick only (no network-cost branch)")
    rows = oracle.run_fifo(cluster, table).rows
    ref = reference_summary(rows, *([np.zeros(0)] * 6))
    t2 = oracle.Tight2(cluster, table)
    for kw in (dict(), dict(max_ticks=7), dict(cap_a=1, cap_b=1)):
        wins, _, _, _ = tight2_windows(t2, **kw)
        got = records_summary(wins)
        for key in ROW_FIELDS:
            if key in FLOAT_FIELDS:
                assert math.isclose(got[key], ref[key], rel_tol=1e-9, abs_tol=1e-12), (case, kw, key)
            else:
                assert got[key] == ref[key], (case, kw, key, got[key], ref[key])
        for W, B in ((1, 1024), (3, 1024), (64, 2), (int(rows["now"][-1]) + 5, 1)):
            want = reference_bins(rows, W, B)
            got_bins = records_bins(wins, W, B)
            for b, (g, w) in enumerate(zip(got_bins, want)):
                for key, v in w.items():
                    if key in FLOAT_FIELDS:
                        assert math.isclose(g[key], v, rel_tol=1e-9, abs_tol=1e-12), (case, kw, W, B, b, key)
                    else:
                        assert g[key] == v, (case, kw, W, B, b, key, g[key], v)


# ---------------------------------------------------------------- long fifo runs: four passes, 128-bit sums
LONG_W, LONG_B = 2 ** 21, 1024


@pytest.fixture(scope="module")
def long_fifo():
    """(table, windows of one window, windows of 64-record windows, job records, finish order) of the long trace on
    two nodes, through Tight2"""
    import oracle
    table = long_trace()
    t2 = oracle.Tight2(long_cluster(), table)
    whole, recs, order, w = tight2_windows(t2)
    many, recs2, order2, _ = tight2_windows(t2, cap_a=8, cap_b=8)
    assert int(w.finished) == table.n and recs.tobytes() == recs2.tobytes() and np.array_equal(order, order2)
    return table, whole, many, recs, order


def test_long_fifo_trace_reaches_four_passes_and_high_words(long_fifo):
    table, whole, many, recs, order = long_fifo
    jobs = job_columns(table, recs, order)
    assert len(many) > 8 and len(whole) == 1
    makespan = records_summary(whole)["makespan"]
    assert 2 ** 30 < makespan < 2 ** 31 - 2 ** 26
    span = summary_span(jobs)
    assert span.bit_length() >= 28 and select_passes(span) == 4
    ref = reference_summary(np.zeros(0, dtype=_row_dtype()), *jobs)
    assert ref["finished"] == table.n and ref["jct_q"][4] == 2 ** 26 - 4 and min(jobs[4]) == 1
    rows = records_summary(whole)
    assert rows["mem_busy_sum"] >= TWO64 and rows["pend_sum_sum"] >= TWO64
    assert sum(1 for b in records_bins(whole, LONG_W, LONG_B) if b["mem_busy_sum"] >= TWO64) > 100
    cls, _ = reference_jobdist(*jobs, JD_BOUNDS, JD_EDGES)
    assert max(c[q + "_sq"] for c in cls for q in ("wait", "turnaround")) >= TWO64
    node_wide = np.asarray(jobs[1]) == 8                         # jobdist's class of 8-GPU jobs selects in four passes too
    assert select_passes(summary_span(tuple(np.asarray(x)[node_wide] for x in jobs))) == 4


def test_long_fifo_records_on_the_host_builds(emus, long_fifo):
    table, whole, many, recs, order = long_fifo
    jobs = job_columns(table, recs, order)
    for wins in (whole, many):
        acc, bins = emu_windows(emus, wins, LONG_W, LONG_B)
        add_jobs(emus["summary_emu"], acc, jobs)
        want = records_summary(wins)
        want.update({k: v for k, v in reference_summary(np.zeros(0, dtype=_row_dtype()), *jobs).items() if k not in ROW_FIELDS})
        assert_summary(acc[0], want, f"{len(wins)} windows")
        assert_bins(bins, records_bins(wins, LONG_W, LONG_B), f"{len(wins)} windows", rel=1e-9)
        assert int(acc[0]["mem_busy_hi"]) > 0 and int(bins["mem_busy_hi"].max()) > 0
    rc, classes, hist = emu_jobdist(emus["jobdist_emu"], jobs, JD_BOUNDS, JD_EDGES)
    assert rc == 0
    assert_jobdist(classes, hist, reference_jobdist(*jobs, JD_BOUNDS, JD_EDGES), "long fifo")
    assert int(classes["wait_sq_hi"].max()) > 0 and int(classes["turnaround_sq_hi"].max()) > 0


@pytest.fixture(scope="module")
def long_runs(long_fifo):
    """{name: (run columns by trace index, finish order)} of the long trace: fifo on two and on 32 nodes (Tight2), sjf
    and dlas-gpu on two nodes (the policy oracle)"""
    import oracle
    table, _, _, recs, order = long_fifo
    out = {"fifo": (run_cols(recs), order)}
    wide, recs32, order32, w = tight2_windows(oracle.Tight2(long_cluster(32), table))
    assert int(w.finished) == table.n
    out["fifo32"] = (run_cols(recs32), order32)
    for name, pol in long_policies():
        res = oracle.run_policy(long_cluster(), pol, table)
        assert len(res.finish_order) == table.n, name
        out[name] = (run_cols(res.recs), res.finish_order)
    return out


LONG_PAIRS = (("fifo", "sjf"), ("sjf", "fifo"), ("fifo", "dlas-gpu"), ("dlas-gpu", "fifo"), ("sjf", "dlas-gpu"), ("fifo", "fifo32"),
              ("fifo32", "fifo"), ("fifo", "fifo"))


def test_long_compares_reach_four_passes_both_ways_and_high_words(emus, long_fifo, long_runs):
    table = long_fifo[0]
    seen_sq = 0
    for a, b in LONG_PAIRS:
        (ra, fa), (rb, fb) = long_runs[a], long_runs[b]
        span, lt, gt = pair_span(table.arrive_tick, ra, fa, rb, fb)
        if a == b:
            assert span == 0
        else:
            assert select_passes(span) == 4, (a, b, span)         # q_hi's select, and q_lo's on the negated values
        if {a, b} <= {"fifo", "sjf", "dlas-gpu"} and a != b:
            assert lt > 0 and gt > 0, (a, b)
        for bounds, edges in (((), ()), (JD_BOUNDS, CMP_EDGES)):
            rc, recs, hist = emu_pair(emus["compare_emu"], table.arrive_tick, table.gpus, ra, fa, rb, fb, bounds, edges)
            assert rc == 0
            ref = reference_pair(table.arrive_tick, table.gpus, ra, fa, rb, fb, bounds, edges)
            assert_pair(recs, hist, ref, f"{a},{b} {bounds}")
            seen_sq = max(seen_sq, max(max(c["d_sq"]) for c in ref[0]))
            if {a, b} == {"fifo", "fifo32"} and not bounds:
                assert int(recs[0]["d_sq_hi"][0]) > 0 and int(recs[0]["d_sq_hi"][1]) > 0
    assert seen_sq >= TWO64
    # what test_gpu_stats_edges reads off the device summaries: max - median of the waits or turnarounds needs
    # four passes
    for name in ("fifo", "sjf", "dlas-gpu"):
        rc, fin = long_runs[name]
        s = reference_summary(np.zeros(0, dtype=_row_dtype()), table.arrive_tick[fin], table.gpus[fin], rc[0][fin], rc[1][fin], rc[2][fin],
                              np.zeros(len(fin)))
        assert select_passes(max(s[f][4] - s[f][0] for f in ("wait_q", "turnaround_q"))) == 4, name


# ---------------------------------------------------------------- designed jct multisets
def test_jct_designs():
    for k in JCT_KS:
        for kind in JOB_KINDS:
            v = np.sort(jct_values(kind, k))
            assert len(v) == k and v.min() >= 1 and v.max() <= 2 ** 26
            ranks = [(q * k + 999) // 1000 - 1 for q in (500, 900, 950, 990, 1000)]
            if kind == "tied":
                assert len(set(v.tolist())) == 1
            elif kind == "two":
                assert len(set(v.tolist())) == min(k, 2)
            elif kind == "shared" and k >= 255:
                u = v[ranks[:3]] - v.min()
                assert select_passes(int(v.max() - v.min())) == 3
                assert len(set((u >> 9).tolist())) == 1 and len(set(u.tolist())) == 3, u
            elif kind == "extremes":
                assert v.max() == 2 ** 26 and (v.min() == 1 or k == 1)


@pytest.mark.parametrize("kind", JOB_KINDS)
def test_jct_traces_through_tight2_and_the_host_select(emus, kind):
    """the fifo yardstick runs every designed trace to the end, jct = the designed values, and the host build's job
    part and jobdist match the references"""
    import oracle
    from gpuschedule_b200.capi import SUMMARY_DTYPE
    for k in JCT_KS:
        table = jct_trace(kind, k)
        _, recs, order, w = tight2_windows(oracle.Tight2(long_cluster(1), table))
        assert int(w.finished) == k, (kind, k)
        jobs = job_columns(table, recs, order)
        assert sorted(jobs[4].tolist()) == sorted(jct_values(kind, k).tolist())
        acc = np.zeros(1, dtype=SUMMARY_DTYPE)
        add_jobs(emus["summary_emu"], acc, jobs)
        ref = reference_summary(np.zeros(0, dtype=_row_dtype()), *jobs)
        assert_summary(acc[0], {key: v for key, v in ref.items() if key not in ROW_FIELDS}, f"{kind} k={k}")
        rc, classes, hist = emu_jobdist(emus["jobdist_emu"], jobs, JD_BOUNDS, JD_EDGES)
        assert rc == 0
        assert_jobdist(classes, hist, reference_jobdist(*jobs, JD_BOUNDS, JD_EDGES), f"{kind} k={k}")


# ---------------------------------------------------------------- many-replica handles
def test_replica_sizes_differ_at_every_grid_stride():
    """the sizes of replicas r and r + g differ for some r, for every grid g a device could launch"""
    for seed in (11, 12, 13):
        s = replica_sizes(1200, seed)
        assert s[3] == 0 and s[5] == 1 and s[7] == 100000 and s[8] < 200
        for g in range(1, len(s)):
            assert (s[:-g] != s[g:]).any(), (seed, g)
    assert grid_bound(132) == 1056 < 1100


def test_small_tables_are_well_formed():
    for n in (0, 1, 2, 150):
        t = small_table(n, 5)
        assert t.n == n and len(t.arrive_tick) == n and (np.diff(t.arrive_tick) >= 0).all()
    cfg = policy_configs(12, big=300)
    assert [p.schedule for _, _, p in cfg][:3] == [1, 3, 4] and cfg[3][2].schedule == 1          # the empty trace runs sjf

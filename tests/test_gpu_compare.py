"""Paired per-job comparisons on the device (gs_compare, gs_horus_compare) on the H100.

Device records and CDF counts must equal test_compare_cpu.reference_pair, the numpy restatement of gs_jpair, over
the job records and finish orders the engine itself hands out: fifo against sjf / dlas / dlas-gpu / gittins on the
fixtures and on bootstrap handles (iid and blocked, with clusters that differ inside a pair), runs compared between
windows, and horus against horus+ / gandiva on the horus fixtures' traces.  Also the invariants (self-pairs, swapped
pairs, classes adding up, agreement with gs_summarize), the error codes, an unchanged gs_summarize, and the sweep."""
import numpy as np
import pytest

from conftest import GOLDEN, REPO, horus_cases
from test_compare_cpu import DIFF_EDGES, assert_pair, horus_pairs_setup, reference_pair, run_cols
from test_summary_cpu import _policy_cases, load_policy

pytestmark = pytest.mark.gpu

SETTINGS = (((), ()), ((5, 17, 65), DIFF_EDGES), ((1, 2, 3, 4, 8, 16, 32), tuple(range(-127 * 40, 128 * 40, 40))), ((2,), (-100, -1, 0, 1, 100)))


def check_handle(eng, tables, pa, pb, bounds, edges, tag=""):
    """gs_compare of the pairs against numpy over eng.fetch_jobs; tables[r]: the trace of replica r"""
    recs, hist = eng.compare(pa, pb, bounds, edges)
    jobs = {}
    for r in set(pa) | set(pb):
        jobs[r] = eng.fetch_jobs(r)
    for p, (a, b) in enumerate(zip(pa, pb)):
        t = tables[a]
        (ra, fa), (rb, fb) = jobs[a], jobs[b]
        assert_pair(recs[p], hist[p], reference_pair(t.arrive_tick, t.gpus, run_cols(ra), fa, run_cols(rb), fb, bounds, edges), f"{tag} {a},{b} {bounds}")
    return recs, hist


def check_invariants(eng, a, b, summaries=None):
    """self-pairs, the swapped pair, classes adding up to C = 1, and (finished runs) agreement with gs_summarize"""
    bounds = (5, 17, 65)
    recs, _ = eng.compare([a, b, a, a], [b, a, a, b], bounds, DIFF_EDGES)
    one, _ = eng.compare([a], [b])
    ab, ba, aa = recs[0], recs[1], recs[2]
    assert (aa["only_a"] == 0).all() and (aa["only_b"] == 0).all() and (aa["eq"] == aa["jobs"][:, None]).all()
    assert not aa["d_sum"].any() and not aa["d_sq_lo"].any() and not aa["q_hi"].any() and not aa["q_lo"].any()
    assert (ba["lt"] == ab["gt"]).all() and (ba["only_a"] == ab["only_b"]).all() and (ba["d_sum"] == -ab["d_sum"]).all()
    assert (ba["d_sq_lo"] == ab["d_sq_lo"]).all() and (ba["d_sq_hi"] == ab["d_sq_hi"]).all() and (ba["q_hi"] == -ab["q_lo"]).all()
    assert recs[3].tobytes() == ab.tobytes()
    for f in ("jobs", "only_a", "only_b", "lt", "eq", "gt", "d_sum"):
        assert (ab[f].sum(axis=0) == one[0][0][f]).all(), f
    if summaries is None:
        return False
    r, sa, sb = one[0][0], summaries[a], summaries[b]
    assert int(r["jobs"]) + int(r["only_a"]) == int(sa["finished"]) and int(r["jobs"]) + int(r["only_b"]) == int(sb["finished"])
    if int(r["only_a"]) or int(r["only_b"]):
        return False
    assert r["d_sum"].tolist() == [int(sb[f]) - int(sa[f]) for f in ("wait_sum", "turnaround_sum", "jct_sum")]
    return True


@pytest.mark.parametrize("case", _policy_cases())
def test_fifo_against_policy_on_fixture(case):
    from gpuschedule_b200 import capi
    table, cluster, pol = load_policy(case)
    with capi.Engine(device=0, nsims=2) as eng:
        eng.config(0, cluster)
        eng.config(1, cluster, pol)
        eng.load_trace(0, table)
        eng.load_trace(1, table)
        eng.run_all(collect_rows=False)
        for bounds, edges in SETTINGS:
            check_handle(eng, [table, table], [0, 1, 0], [1, 0, 0], bounds, edges, case)
        check_invariants(eng, 0, 1, eng.summarize())


def test_complete_runs_agree_with_summaries():
    """bench.py's generated trace, which fifo and sjf finish: with both runs complete and C = 1, `jobs` is both
    summaries' `finished` and d_sum the difference of their sums"""
    import sys
    from gpuschedule_b200 import capi
    sys.path.insert(0, REPO)
    from bench import BASE_SEED, fast_table
    t = fast_table(20000, BASE_SEED)
    with capi.Engine(device=0, nsims=3) as eng:
        for r, p in enumerate((None, capi.make_policy("sjf"), None)):
            eng.config(r, capi.make_cluster(4, 32, 8) if r < 2 else capi.make_cluster(2, 32, 8), p)
            eng.load_trace(r, t)
        summ = eng.run_summarized()
        assert (summ["finished"] == t.n).all()
        assert check_invariants(eng, 0, 1, summ) and check_invariants(eng, 2, 1, summ)
        check_handle(eng, [t] * 3, [0, 2, 1], [1, 1, 0], (5,), DIFF_EDGES, "bench trace")


def test_partial_runs_between_windows():
    """fifo and a policy run window by window; every comparison between windows matches the finish orders so far, and
    the last one the whole run's"""
    from gpuschedule_b200 import capi
    table, cluster, pol = load_policy("policy_dlas_gpu")
    with capi.Engine(device=0, nsims=3) as eng:
        eng.config(0, cluster)
        eng.config(1, cluster, pol)
        eng.config(2, cluster, capi.make_policy("sjf"))
        for r in range(3):
            eng.load_trace(r, table)
        calls = 0
        while True:
            eng.run(0, 16)
            check_handle(eng, [table] * 3, [0, 0, 1], [1, 2, 2], (5, 17, 65), DIFF_EDGES, f"window {calls}")
            calls += 1
            if all(eng.stats(r).done for r in range(3)):
                break
        last = eng.compare([0, 0, 1], [1, 2, 2], (5, 17, 65), DIFF_EDGES)
    assert calls > 3
    with capi.Engine(device=0, nsims=3) as eng:
        eng.config(0, cluster)
        eng.config(1, cluster, pol)
        eng.config(2, cluster, capi.make_policy("sjf"))
        for r in range(3):
            eng.load_trace(r, table)
        eng.run_all(collect_rows=False)
        whole = eng.compare([0, 0, 1], [1, 2, 2], (5, 17, 65), DIFF_EDGES)
    assert last[0].tobytes() == whole[0].tobytes() and last[1].tobytes() == whole[1].tobytes()


def _boot_flags(tmp_schedules, trace, clusters):
    from gpuschedule_b200 import sweep
    return [sweep.make_flags(trace_file=trace, schedule=sc, num_switch=ns, num_node_p_switch=npn)
            for sc, (ns, npn) in zip(tmp_schedules, clusters)]


def _boot_handle(sets, R, loads, seed, block_len=None):
    """the handle summarize_bootstrap builds for one trace file, run to the end (open: the caller closes it)"""
    from gpuschedule_b200 import capi, sweep
    sims = sweep._plain_setup(sets)
    base = sims[0][2].table
    params = np.zeros(len(sets) * len(loads) * R, dtype=capi.BOOT_PARAMS_DTYPE)
    eng = capi.Engine(device=0, nsims=len(params))
    i = 0
    for fl, infra, jm, pol in sims:
        for L in loads:
            num, den = sweep.load_gap_scale(L)
            for r in range(R):
                eng.config(i, infra.gs_cluster(), pol)
                params[i] = (seed, r, base.n, num, den)
                i += 1
    eng.boot_population(base)
    eng.boot_traces(params, block_len=block_len)
    eng.run_summarized()
    return eng


@pytest.mark.parametrize("block_len", [None, 16])
def test_bootstrap_handle_against_numpy_and_sweep(block_len):
    """fifo against sjf / dlas / dlas-gpu / gittins on the same bootstrap replicas (the policies on a smaller
    cluster than fifo's), device against numpy; summarize_bootstrap's compare path gives the same records"""
    import os
    from gpuschedule_b200 import capi, sweep
    trace = os.path.join(GOLDEN, "policy_dlas_gpu", "trace.csv")
    schedules = ["fifo", "sjf", "dlas", "dlas-gpu", "gittins"]
    sets = _boot_flags(schedules, trace, [(4, 32)] + [(1, 32)] * 4)
    R, loads, seed = 6, [1.0, 2.0], 7
    pairs = tuple((0, b) for b in range(1, 5))
    bounds, edges = (5, 17), DIFF_EDGES
    eng = _boot_handle(sets, R, loads, seed, block_len)
    try:
        tables = []
        for r in range(eng.nsims):
            tr = eng.fetch_trace(r)
            tables.append(type("T", (), dict(arrive_tick=tr["arrive_tick"], gpus=tr["gpus"]))())
        span = np.arange(len(loads) * R)
        pa = np.concatenate([a * len(loads) * R + span for a, _ in pairs])
        pb = np.concatenate([b * len(loads) * R + span for _, b in pairs])
        recs, hist = check_handle(eng, tables, pa.tolist(), pb.tolist(), bounds, edges, f"boot L={block_len}")
        check_invariants(eng, int(pa[0]), int(pb[0]), eng.summarize())
        with pytest.raises(capi.GsError) as e:                            # two loads: the same stream, different traces
            eng.compare([0], [R])
        assert e.value.code == capi.GS_ERR_ARG
    finally:
        eng.close()
    res = sweep.summarize_bootstrap(sets, R, loads, seed=seed, block_len=1 if block_len is None else block_len, compare=(pairs, bounds, edges))
    got_recs, got_hist = res[-1]
    assert got_recs.shape == (len(pairs), len(loads), R, len(bounds) + 1)
    assert got_recs.reshape(-1).tobytes() == recs.reshape(-1).tobytes()
    assert got_hist.reshape(-1).tobytes() == hist.reshape(-1).tobytes()


def test_heterogeneous_handle_of_150_replicas():
    """150 replicas: five fixture traces under fifo and four policies, each trace on a cluster of its own size,
    paired in every order within a trace"""
    from gpuschedule_b200 import capi
    cases = _policy_cases()[:5]
    cfgs, tables = [], []
    for case in cases:
        table, cluster, pol = load_policy(case)
        for k in range(30):
            kind = k % 5
            p = pol if kind in (0, 3) else capi.make_policy("sjf") if kind == 2 else None
            cfgs.append((cluster if k % 2 else capi.make_cluster(2, 16, 8), p))
            tables.append(table)
    with capi.Engine(device=0, nsims=len(cfgs)) as eng:
        for r, ((cl, p), t) in enumerate(zip(cfgs, tables)):
            eng.config(r, cl, p)
            eng.load_trace(r, t)
        eng.run_all(collect_rows=False)
        rng = np.random.default_rng(1)
        pa = rng.integers(0, 150, 300)
        pb = pa // 30 * 30 + rng.integers(0, 30, 300)
        check_handle(eng, tables, pa.tolist(), pb.tolist(), (5, 17, 65), DIFF_EDGES, "150")
        check_handle(eng, tables, pa[:50].tolist(), pb[:50].tolist(), (1, 2, 3, 4, 8, 16, 32), tuple(range(-127 * 40, 128 * 40, 40)), "150 C=8")


def test_errors_leave_outputs_untouched_and_summaries_unchanged():
    import ctypes as C
    from gpuschedule_b200 import capi
    table, cluster, pol = load_policy("policy_sjf_sat")
    short = load_policy("policy_dlas_gpu")[0]
    with capi.Engine(device=0, nsims=4) as eng:
        for r, t in enumerate((table, table, short, table)):
            eng.config(r, cluster, pol if r == 1 else None)
            eng.load_trace(r, t)
        assert _code(eng, [0], [1]) == capi.GS_ERR_STATE                   # nothing has run
        eng.run_all(collect_rows=False)
        base = eng.summarize()
        n0 = eng.launch_count()
        for a, b, bounds, edges, code in (([0], [2], (), (), capi.GS_ERR_ARG),     # different n
                                          ([0], [4], (), (), capi.GS_ERR_ARG), ([-1], [0], (), (), capi.GS_ERR_ARG),
                                          ([0], [1], (0,), (), capi.GS_ERR_ARG), ([0], [1], (3, 3), (), capi.GS_ERR_ARG),
                                          ([0], [1], (), (2, 1), capi.GS_ERR_ARG), ([0], [1], (), tuple(range(256)), capi.GS_ERR_ARG)):
            assert _code(eng, a, b, bounds, edges) == code, (a, b, bounds, len(edges))
        assert eng.launch_count() == n0
        rc = eng.lib.gs_compare(eng.h, 1, None, None, 1, None, 0, None, None, None, None)
        assert rc == capi.GS_ERR_ARG
        eng.reset()
        eng.run_all(collect_rows=False)
        again = eng.summarize()
        recs, hist = eng.compare([0, 1], [1, 0], (5, 17), DIFF_EDGES)
        after = eng.summarize()
        assert eng.launch_count() - n0 > 0
        n1 = eng.launch_count()
        eng.summarize()
        n2 = eng.launch_count()
        eng.compare([0], [1])
        n3 = eng.launch_count()
        eng.summarize()
        assert n3 - n2 == 1 and eng.launch_count() - n3 == n2 - n1
        assert after.tobytes() == again.tobytes()
        for f in ("finished", "wait_sum", "jct_q"):
            assert np.array_equal(again[f], base[f])
        # a pair whose traces differ, found on the device: out untouched, the message names the pair
        eng2 = capi.Engine(device=0, nsims=2)
        try:
            eng2.config(0, cluster)
            eng2.config(1, cluster)
            eng2.load_trace(0, table)
            eng2.load_trace(1, _perturbed(table))
            eng2.run_all(collect_rows=False)
            a, b = np.array([0, 0], dtype=np.int32), np.array([0, 1], dtype=np.int32)
            buf2 = np.full(2 * capi.JPAIR_DTYPE.itemsize, 0x5a, dtype=np.uint8)
            hb2 = np.full(8, 0x5a5a5a5a, dtype=np.uint32)
            rc = eng2.lib.gs_compare(eng2.h, 2, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), 1, None, 0, None,
                                     buf2.ctypes.data_as(C.c_void_p), hb2.ctypes.data_as(C.c_void_p), None)
            assert rc == capi.GS_ERR_ARG and b"pair 1" in eng2.lib.gs_last_error(eng2.h)
            assert (buf2 == 0x5a).all() and (hb2 == 0x5a5a5a5a).all()
        finally:
            eng2.close()


def _perturbed(table):
    """the same trace with job 3's duration one tick longer"""
    import copy
    t = copy.deepcopy(table)
    t.duration = np.array(t.duration, dtype=np.float64).copy()
    t.duration[3] += 1.0
    return t


def _code(eng, a, b, bounds=(), edges=()):
    from gpuschedule_b200 import capi
    with pytest.raises(capi.GsError) as e:
        eng.compare(a, b, bounds, edges)
    return e.value.code


def test_horus_pairs_on_fixture_traces():
    from gpuschedule_b200 import capi
    cases = horus_cases()
    with capi.HorusEngine(device=0, nsims=2 * len(cases)) as eng:
        tables = horus_pairs_setup(eng, cases)
        with pytest.raises(capi.GsError) as e:
            eng.compare([0], [1])
        assert e.value.code == capi.GS_ERR_STATE
        eng.run(rows_cap=1 << 15)
        pa = [2 * i for i in range(len(cases))] + [2 * i + 1 for i in range(len(cases))]
        pb = [2 * i + 1 for i in range(len(cases))] + [2 * i for i in range(len(cases))]
        for bounds, edges in SETTINGS:
            recs, hist = eng.compare(pa, pb, bounds, edges)
            for p, (a, b) in enumerate(zip(pa, pb)):
                t = tables[a // 2]
                _, _, _, ra, fa = eng.fetch(a)
                _, _, _, rb, fb = eng.fetch(b)
                assert_pair(recs[p], hist[p], reference_pair(t.arrive_tick, t.gpus, run_cols(ra), fa, run_cols(rb), fb, bounds, edges),
                            f"{cases[a // 2]} {bounds}")
        if len(cases) > 1:
            with pytest.raises(capi.GsError) as e:                            # two fixtures' traces
                eng.compare([0], [2])
            assert e.value.code == capi.GS_ERR_ARG


def test_sweep_batched_compare_matches_handle():
    import os
    from gpuschedule_b200 import capi, sweep
    trace = os.path.join(GOLDEN, "policy_sjf_sat", "trace.csv")
    sets = [sweep.make_flags(trace_file=trace, schedule=sc) for sc in ("fifo", "sjf", "dlas-gpu")]
    pairs, bounds, edges = ((0, 1), (0, 2), (2, 1)), (5, 17), DIFF_EDGES
    summ, (recs, hist) = sweep.summarize_batched(sets, compare=(pairs, bounds, edges))
    sims = sweep._plain_setup(sets)
    with capi.Engine(device=0, nsims=3) as eng:
        sweep._plain_load(eng, sims)
        eng.run_summarized()
        want = check_handle(eng, [s[2].table for s in sims], [a for a, _ in pairs], [b for _, b in pairs], bounds, edges, "sweep")
    assert recs.tobytes() == want[0].tobytes() and hist.tobytes() == want[1].tobytes()


def test_sweep_cli_writes_paired_files(tmp_path):
    import csv
    import os
    from gpuschedule_b200 import sweep
    trace = os.path.join(GOLDEN, "policy_sjf_sat", "trace.csv")
    out = {k: str(tmp_path / f"{k}.csv") for k in ("s", "p", "c", "ps", "bs", "bp", "bc", "bps")}
    sweep.main(["--trace", trace, "--schedule", "fifo", "sjf", "dlas-gpu", "--compare", "fifo", "--summary", out["s"], "--num_switch", "1",
                "--gpu-classes", "5", "17", "--paired", out["p"], "--paired-cdf", out["c"], "--paired-summary", out["ps"]])
    rows = list(csv.DictReader(open(out["p"])))
    assert len(rows) == 2 * 3 * 3 and {r["base_schedule"] for r in rows} == {"fifo"} and {r["schedule"] for r in rows} == {"sjf", "dlas-gpu"}
    assert len(list(csv.DictReader(open(out["c"])))) == 2 * 3 * 3 * 63
    assert len(list(csv.DictReader(open(out["ps"])))) == 2
    sweep.main(["--trace", trace, "--schedule", "fifo", "sjf", "--compare", "fifo", "--summary", out["bs"], "--num_switch", "1",
                "--bootstrap", "4", "--load", "1.0", "2.0", "--block-len", "8", "--paired", out["bp"], "--paired-cdf", out["bc"],
                "--paired-summary", out["bps"]])
    rows = list(csv.DictReader(open(out["bp"])))
    assert len(rows) == 2 * 3 and rows[0]["block_len"] == "8" and rows[0]["base_schedule"] == "fifo"
    assert len(list(csv.DictReader(open(out["bps"])))) == 2

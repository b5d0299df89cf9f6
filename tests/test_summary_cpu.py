"""Run summaries (gs_summary, gpuschedule_b200/csrc/gs_summary.cuh) on a box without a GPU.

The __host__ __device__ part of gs_summary.cuh -- the row fold, the closed-form fold of the fifo engine's compact
records, the rank and radix-digit arithmetic of the job part -- is compiled with g++ (tests/emu/summary_emu.cpp) and
compared with a numpy summary computed here from rows and job records: of the pinned oracles on every fixture, of
the fifo records folded window by window, and of the host-emulation build of gs_horus.cu through
gs_horus_summarize itself."""
import ctypes as C
import functools
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, REPO, golden_cases, horus_cases, load_golden, load_horus

PERMILLE = (500, 900, 950, 990, 1000)
FLOAT_FIELDS = ("avg_pending_sum", "util_sum")


# ---------------------------------------------------------------- the numpy summary (shared with test_gpu_summary.py)
def reference_summary(rows, arrive, gpus, start, end, jct, preempt, util=None):
    """the fields of gs_summary from cluster.csv-style rows (ROW_DTYPE) and the finished jobs' columns in finish order
    (arrive = arrival tick); 128-bit fields as exact ints, util_sum only when `util` is given"""
    t = len(rows)
    r = dict(rows=t, makespan=int(rows["now"][-1]) if t else 0)
    for f in ("busy_gpus", "running", "queued"):
        col = rows[f].astype(np.int64)
        r[f + "_sum"] = int(col.sum())
        r[f + "_max"] = int(col.max()) if t else 0
    r["pend_max_max"] = int(rows["pend_max"].max()) if t else 0
    r["pend_sum_sum"] = sum(rows["pend_sum"].tolist())
    r["mem_busy_sum"] = sum(rows["mem_busy_bytes"].tolist())
    nz = (rows["queued"] > 0) & (rows["pend_sum"] != 0)
    r["pending_rows"] = int(nz.sum())
    r["avg_pending_sum"] = math.fsum((rows["pend_sum"][nz].astype(np.float64) / (rows["queued"][nz].astype(np.float64) + 1e-9)).tolist())
    if util is not None:
        r["util_sum"] = math.fsum(np.nan_to_num(np.asarray(util, dtype=np.float64), nan=0.0).tolist())
    arrive, gpus, start, end, jct, preempt = (np.asarray(a, dtype=np.int64) for a in (arrive, gpus, start, end, jct, preempt))
    k = len(start)
    wait, turn = start - arrive, end - arrive
    r.update(finished=k, wait_sum=int(wait.sum()), turnaround_sum=int(turn.sum()), jct_sum=int(jct.sum()),
             preempt_sum=int(preempt.sum()), gpu_ticks_sum=int((gpus * jct).sum()))
    for name, v in (("wait_q", wait), ("turnaround_q", turn), ("jct_q", jct)):
        s = np.sort(v)
        r[name] = [int(s[(q * k + 999) // 1000 - 1]) for q in PERMILLE] if k else [0] * 5
    return r


def job_columns(table, recs, order):
    """(arrive, gpus, start, end, jct, preempt) of the finished jobs in finish order from job records"""
    o = np.asarray(order, dtype=np.int64)
    return (table.arrive_tick[o], table.gpus[o], recs["start"][o], recs["end"][o], recs["jct"][o], recs["preempt"][o])


def record_fields(rec):
    """one SUMMARY_DTYPE record as the dict reference_summary makes"""
    d = {name: (rec[name].tolist() if rec[name].shape else rec[name].item()) for name in rec.dtype.names}
    d["pend_sum_sum"] = (int(rec["pend_sum_hi"]) << 64) | int(rec["pend_sum_lo"])
    d["mem_busy_sum"] = (int(rec["mem_busy_hi"]) << 64) | int(rec["mem_busy_lo"])
    return d


def assert_summary(rec, ref, tag="", rel=1e-9, skip=()):
    got = record_fields(rec)
    for key, want in ref.items():
        if key in skip:
            continue
        if key in FLOAT_FIELDS:
            assert math.isclose(got[key], want, rel_tol=rel, abs_tol=1e-12), (tag, key, got[key], want)
        else:
            assert got[key] == want, (tag, key, got[key], want)


# ---------------------------------------------------------------- host build of gs_summary.cuh
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("summary_emu") / "libsummary_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "summary_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.emu_sum_rank.restype = C.c_longlong
    lib.emu_sum_run_length.restype = C.c_int
    lib.emu_sum_run_length.argtypes = [C.c_double]
    return lib


def _p(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def emu_summary(lib, rows, jobs, util=None):
    from gpuschedule_b200.capi import SUMMARY_DTYPE
    acc = np.zeros(1, dtype=SUMMARY_DTYPE)
    rows = np.ascontiguousarray(rows)
    u = None if util is None else np.ascontiguousarray(util, dtype=np.float64)
    lib.emu_sum_rows(_p(rows), _p(u), C.c_longlong(len(rows)), _p(acc))
    add_jobs(lib, acc, jobs)
    return acc


def add_jobs(lib, acc, jobs):
    arrive, gpus, start, end, jct, preempt = jobs
    cols = [_i32(c) for c in (arrive, start, end, jct, preempt, gpus)]
    lib.emu_sum_jobs(*[_p(c) for c in cols], C.c_longlong(len(cols[0])), _p(acc))


# ---------------------------------------------------------------- row fold + job part against the oracles
@pytest.mark.parametrize("case", golden_cases())
def test_fifo_fixture_summary(emu, case):
    import oracle
    table, cluster, _, _, _ = load_golden(case)
    res = oracle.run_fifo(cluster, table)
    jobs = job_columns(table, res.recs, res.finish_order)
    acc = emu_summary(emu, res.rows, jobs)
    assert_summary(acc[0], reference_summary(res.rows, *jobs), case)


def _policy_cases():
    return sorted(d for d in os.listdir(GOLDEN) if d.startswith("policy_") and os.path.isfile(os.path.join(GOLDEN, d, "expected.json")))


@functools.lru_cache(maxsize=None)
def load_policy(case):
    """(table, cluster, policy) of a policy_* fixture"""
    import json
    from gpuschedule_b200 import capi, ingest, policies
    d = os.path.join(GOLDEN, case)
    with open(os.path.join(d, "params.json")) as f:
        meta = json.load(f)
    table = ingest.JobTraceReader(os.path.join(d, "trace.csv")).prepare_jobs().table(0.5)
    kw = dict(meta["params"])
    if meta["policy"] == "gittins":
        kw["gittins_table"] = policies.build_gittins_table(policies.gittins_samples(table), kw.get("gittins_delta", 3250.0))
    return table, capi.make_cluster(**meta["cluster"]), capi.make_policy(meta["policy"], **kw)


@pytest.mark.parametrize("case", _policy_cases())
def test_policy_fixture_summary(emu, case):
    import oracle
    table, cluster, pol = load_policy(case)
    res = oracle.run_policy(cluster, pol, table)
    jobs = job_columns(table, res.recs, res.finish_order)
    acc = emu_summary(emu, res.rows, jobs)
    assert_summary(acc[0], reference_summary(res.rows, *jobs), case)


@pytest.mark.parametrize("case", horus_cases())
def test_horus_fixture_summary(emu, case):
    import oracle
    table, cluster, params, _, _ = load_horus(case)
    res = oracle.run_horus(cluster, table, **params)
    jobs = job_columns(table, res.recs, res.finish_order)
    acc = emu_summary(emu, res.rows, jobs, res.util)
    ref = reference_summary(res.rows, *jobs, util=res.util)
    assert_summary(acc[0], ref, case)
    assert ref["finished"] > 0 and ref["util_sum"] > 0


# ---------------------------------------------------------------- the fifo engine's compact records, window by window
def fold_windows(lib, t2, **run_kw):
    """restart the Tight2 yardstick and fold the records of every window as gs_summarize does after every gs_run"""
    from gpuschedule_b200.capi import SUMMARY_DTYPE
    acc = np.zeros(1, dtype=SUMMARY_DTYPE)
    t2.restart()
    windows = 0
    while True:
        rc, w, _, _, done = t2.run_window(**run_kw)
        assert rc == 0
        ev, qr = t2.ev[:w.ev_rows], t2.qr[:w.q_rows]
        lib.emu_sum_compact(_p(ev), C.c_longlong(len(ev)), _p(qr), C.c_longlong(len(qr)), C.c_longlong(w.row_first),
                            C.c_longlong(w.ticks), _p(acc))
        lib.emu_sum_compact(_p(ev), C.c_longlong(len(ev)), _p(qr), C.c_longlong(len(qr)), C.c_longlong(w.row_first),
                            C.c_longlong(w.ticks), _p(acc))      # a second fold of the same window adds nothing
        windows += 1
        if done or t2.n == 0:
            return acc, windows


@pytest.mark.parametrize("case", golden_cases())
def test_fifo_records_fold_window_by_window(emu, case):
    import oracle
    table, cluster, _, _, _ = load_golden(case)
    if cluster.enable_network_costs:
        pytest.skip("the record yardstick runs the plain fifo + yarn tick only (no network-cost branch)")
    ref_run = oracle.run_fifo(cluster, table)
    ref = reference_summary(ref_run.rows, *job_columns(table, ref_run.recs, ref_run.finish_order))
    row_fields = {k: v for k, v in ref.items() if k in ("rows", "makespan", "pend_sum_sum", "mem_busy_sum", "pending_rows",
                                                        "avg_pending_sum", "pend_max_max") or k.endswith(("_sum", "_max"))
                  and k not in ("wait_sum", "turnaround_sum", "jct_sum", "preempt_sum", "gpu_ticks_sum")}
    t2 = oracle.Tight2(cluster, table)
    whole, n1 = fold_windows(emu, t2)
    assert n1 == 1
    assert_summary(whole[0], row_fields, case)
    for kw, tag in ((dict(max_ticks=7), "7-tick windows"), (dict(cap_a=1, cap_b=1), "one record per window")):
        acc, nw = fold_windows(emu, t2, **kw)
        assert nw > 1, tag
        assert_summary(acc[0], row_fields, f"{case} {tag}", rel=1e-12)
        got, want = record_fields(acc[0]), record_fields(whole[0])
        for k in row_fields:
            if k not in FLOAT_FIELDS:
                assert got[k] == want[k], (case, tag, k)


# ---------------------------------------------------------------- order statistics
def _select(lib, v):
    v = _i32(v)
    out = np.zeros(5, dtype=np.int32)
    lib.emu_sum_select(_p(v), C.c_longlong(len(v)), _p(out))
    return out.tolist()


def _nearest_rank(v):
    s = np.sort(np.asarray(v, dtype=np.int64))
    k = len(s)
    return [int(s[(q * k + 999) // 1000 - 1]) for q in PERMILLE] if k else [0] * 5


def test_order_statistic_edge_cases(emu):
    assert [emu.emu_sum_rank(q, 1) for q in PERMILLE] == [0] * 5
    assert [emu.emu_sum_rank(q, 2) for q in PERMILLE] == [0, 1, 1, 1, 1]
    assert [emu.emu_sum_rank(q, 1000) for q in PERMILLE] == [499, 899, 949, 989, 999]
    assert [emu.emu_sum_rank(q, 1001) for q in PERMILLE] == [500, 900, 950, 990, 1000]
    rng = np.random.default_rng(11)
    cases = [[], [0], [7], [5, 3], [0, 0], [4] * 1000, [2 ** 31 - 1, 0, 2 ** 31 - 1], [-5, 3, -5, 9]]
    for b in (1, 8, 9, 10, 17, 18, 19, 26, 27, 28, 30):
        cases.append([2 ** b - 1, 2 ** b, 2 ** b + 1, 0, 2 ** b] * 3)
        cases.append(rng.integers(0, 2 ** b + 1, 1001).tolist())
    cases += [rng.integers(0, 300000, 100000).tolist(), rng.integers(0, 3, 777).tolist(), np.repeat([1, 2 ** 20], [999, 1]).tolist()]
    for v in cases:
        assert _select(emu, v) == _nearest_rank(v), v[:8]


def test_fifo_run_length_matches_expand_jobs(emu):
    from gpuschedule_b200 import log_manager as lm
    d = np.array([0.0, 0.2, 1.0, 1.5, 2.0, 2.0000001, 1e6 + 0.5, -3.0])
    recs = lm.expand_jobs(np.zeros(len(d), dtype=lm.JOBRUN_DTYPE), len(d), d)
    assert [emu.emu_sum_run_length(float(x)) for x in d] == recs["jct"].tolist()


# ---------------------------------------------------------------- gs_horus_summarize through the host build of gs_horus.cu
@pytest.fixture(scope="module")
def horus_emu_engine():
    import importlib.util
    import sys
    spec = importlib.util.spec_from_file_location("tests_emu_summary", os.path.join(REPO, "tests", "emu", "__init__.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["tests_emu_summary"] = mod
    spec.loader.exec_module(mod)
    out = mod._ABI_OUT
    hdr = os.path.join(REPO, "gpuschedule_b200", "csrc", "gs_summary.cuh")
    if os.path.exists(out) and os.path.getmtime(out) < os.path.getmtime(hdr) and mod._abi_lib is None:
        mod.build_abi(force=True)                 # gs_summary.cuh is not among the emu build's own dependencies
    return mod.emu_engine_class()


def test_horus_summarize_host_build_matches_reference(horus_emu_engine):
    from gpuschedule_b200 import capi
    cases = horus_cases()
    assert len(cases) == 12
    loaded = [load_horus(c) for c in cases]
    with horus_emu_engine(device=0, nsims=len(cases)) as eng:
        for i, (table, cluster, params, _, _) in enumerate(loaded):
            eng.config(i, cluster, capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"]))
            eng.load_trace(i, table)
            np.random.seed(params["seed"])
            eng.load_words(i, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))
        with pytest.raises(capi.GsError) as e:
            eng.summarize()
        assert e.value.code == capi.GS_ERR_STATE
        eng.run(rows_cap=1 << 15)
        recs = eng.summarize()
        with pytest.raises(capi.GsError) as e:
            eng.summarize(first=3, count=len(cases))
        assert e.value.code == capi.GS_ERR_ARG
        part = eng.summarize(first=2, count=3)
        assert part.tobytes() == recs[2:5].tobytes()
        for i, (case, (table, cluster, params, _, _)) in enumerate(zip(cases, loaded)):
            rows, util, _, hrecs, order = eng.fetch(i)
            assert recs[i]["done"] == 1 and recs[i]["n"] == table.n, case
            assert_summary(recs[i], reference_summary(rows, *job_columns(table, hrecs, order), util=util), case)

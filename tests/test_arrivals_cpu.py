"""Job statistics by arrival time (gs_abin, gpuschedule_b200/csrc/gs_summary.cuh) on a box without a GPU.

The setting's validation and gs_arr_serial, the host form of gs_arr_jobs_kernel, are compiled with g++
(tests/emu/arrivals_emu.cpp) and compared with `reference_arrivals`: bin the finished jobs by
min(arrival // W, B - 1), then restate every bin with test_slowdown_cpu.reference_slowdown as one class.  The cases are
the fixtures' job records and seeded random job sets that meet the kernel's cut-over between its warp and block paths.
gs_horus_set_arrivals / gs_horus_fetch_arrivals run through the host-emulation build of gs_horus.cu;
summary.arrivals_derived is checked against pandas, and the sweep's argument errors and file columns too."""
import csv
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, REPO, horus_cases, load_golden, load_horus
from test_jobdist_cpu import FIXTURES, QUANTS, _code, csv_jobs, horus_emu_engine  # noqa: F401
from test_slowdown_cpu import SD_MAX, reference_slowdown, sdclass_fields
from test_summary_cpu import PERMILLE, job_columns, load_policy

CUT = 256                        # GS_ARR_CUT: bins of at most this many finished jobs are finished by one warp
SUM_THREADS = 256                # GS_SUM_THREADS


# ---------------------------------------------------------------- the restatement (shared with test_gpu_arrivals.py)
def arrival_bin(a, W, B):
    return 0 if a < 0 else min(a // W, B - 1)


def reference_arrivals(arrive, gpus, start, end, jct, preempt, trace_arrive, W, B, tau):
    """per bin a dict of gs_abin fields (reference_slowdown's fields of the bin's finished jobs as one class, key_sum the
    exact sum of their arrival ticks, and `arrived`) of the finished jobs' columns and the trace's arrival ticks"""
    cols = [np.asarray(a, dtype=np.int64) for a in (arrive, gpus, start, end, jct, preempt)]
    bins = np.array([arrival_bin(int(a), W, B) for a in cols[0].tolist()], dtype=np.int64)
    arrived = [0] * B
    for a in np.asarray(trace_arrive, dtype=np.int64).tolist():
        arrived[arrival_bin(a, W, B)] += 1
    out = []
    for b in range(B):
        sel = bins == b
        (d,), _ = reference_slowdown(*(c[sel] for c in cols), "gpus", (), tau, (), ())
        d["key_sum"] = int(cols[0][sel].sum())
        d["arrived"] = arrived[b]
        out.append(d)
    return out


def abin_fields(rec):
    """one ABIN_DTYPE record as the dict reference_arrivals makes (key_sum as a signed 128-bit value)"""
    d = sdclass_fields(rec["s"])
    if d["key_sum"] >> 127:
        d["key_sum"] -= 1 << 128
    d["arrived"] = int(rec["arrived"])
    return d


def assert_arrivals(recs, ref, tag=""):
    assert len(recs) == len(ref), tag
    for b, (rec, w) in enumerate(zip(recs, ref)):
        got = abin_fields(rec)
        for key, v in w.items():
            assert got[key] == v, (tag, b, key, got[key], v)


# ---------------------------------------------------------------- host build
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("arrivals_emu") / "libarrivals_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "arrivals_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.emu_arr_bin.argtypes = [C.c_longlong, C.c_longlong, C.c_int]
    lib.emu_arr_check.argtypes = [C.c_longlong, C.c_int, C.c_longlong]
    for name in ("emu_arr_bin", "emu_arr_check", "emu_arr_jobs"):
        getattr(lib, name).restype = C.c_int
    return lib


def _p(a):
    return np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def emu_arrivals(lib, jobs, trace_arrive, W, B, tau):
    """(rc, records) of gs_arr_serial over the job columns (arrive, gpus, start, end, jct, preempt); the output starts
    filled with 0xAB bytes so that an untouched output can be told apart"""
    from gpuschedule_b200 import capi
    cols = [np.ascontiguousarray(c, dtype=np.int32) for c in jobs]
    ta = np.ascontiguousarray(trace_arrive, dtype=np.int32)
    nb = max(B, 1) if 0 <= B <= 1024 else 1
    recs = np.frombuffer(b"\xab" * (nb * capi.ABIN_DTYPE.itemsize), dtype=capi.ABIN_DTYPE).copy()
    rc = lib.emu_arr_jobs(*[_p(c) for c in (cols[0], cols[2], cols[3], cols[4], cols[5], cols[1])], C.c_longlong(len(cols[0])),
                          _p(ta), C.c_longlong(len(ta)), C.c_longlong(W), C.c_int(B), C.c_longlong(tau), _p(recs))
    return rc, recs


def check(lib, jobs, trace_arrive, W, B, tau, tag):
    rc, recs = emu_arrivals(lib, jobs, trace_arrive, W, B, tau)
    assert rc == 0, tag
    assert_arrivals(recs, reference_arrivals(*jobs, trace_arrive, W, B, tau), tag)
    assert int(recs["arrived"].sum()) == len(trace_arrive), tag
    assert int(recs["s"]["jc"]["jobs"].sum()) == len(jobs[0]), tag
    return recs


def test_bin_rule(emu):
    for a, W, B, want in ((0, 1, 1, 0), (5, 1, 10, 5), (10, 1, 10, 9), (-1, 7, 4, 0), (-2 ** 31, 1, 1024, 0), (6, 7, 4, 0), (7, 7, 4, 1),
                          (27, 7, 4, 3), (2 ** 31 - 1, 500, 128, 127), (2 ** 31 - 1, 2 ** 40, 1024, 0), (2 ** 31 - 1, 1, 1024, 1023)):
        assert emu.emu_arr_bin(a, W, B) == want == arrival_bin(a, W, B), (a, W, B)


# ---------------------------------------------------------------- fixtures
def _fixture(kind, case):
    """(job columns in finish order, arrival ticks of the whole trace) of a fixture run"""
    import oracle
    if kind in ("fifo", "horus"):
        table = (load_golden if kind == "fifo" else load_horus)(case)[0]
        return csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table), table.arrive_tick
    table, cluster, pol = load_policy(case)
    res = oracle.run_policy(cluster, pol, table)
    return job_columns(table, res.recs, res.finish_order), table.arrive_tick


@pytest.mark.parametrize("kind,case", FIXTURES)
def test_fixture_arrivals(emu, kind, case):
    jobs, ta = _fixture(kind, case)
    last = int(np.max(ta))
    assert len(jobs[0]) > 0
    for W, B, tau in ((1, 1, 1), (1, 1024, 1), (max(1, last // 100), 128, 1), (max(1, last // 7), 8, 60), (last + 1, 4, 1),
                      (2 ** 40, 1024, 10 ** 9), (500, 128, 1)):
        check(emu, jobs, ta, W, B, tau, f"{case} W={W} B={B} tau={tau}")


# ---------------------------------------------------------------- seeded random job sets
def _jobs_at(rng, arrive, scale):
    """finished-job columns for the given arrival ticks, in a shuffled finish order"""
    k = len(arrive)
    arrive = np.asarray(arrive, dtype=np.int64)
    start = arrive + rng.integers(0, scale, k)
    jct = rng.integers(1, max(2, scale // 64), k)
    jct[: k // 3] = rng.integers(1, 4, k // 3)
    end = start + jct + rng.integers(0, 3, k)
    gpus = rng.choice([1, 2, 4, 8, 64], k)
    preempt = rng.integers(0, 4, k)
    perm = rng.permutation(k)
    return tuple(c[perm] for c in (arrive, gpus, start, end, jct, preempt))


def cutover_arrivals(W=10):
    """arrival ticks whose bins of width W hold 0, CUT - 1, CUT, CUT + 1, 1, 0, SUM_THREADS + 7 and 3 * CUT jobs, the
    last bin open-ended past the others; every tick is on or inside a bin edge"""
    sizes = (0, CUT - 1, CUT, CUT + 1, 1, 0, SUM_THREADS + 7, 3 * CUT)
    return np.sort(np.concatenate([b * W + np.arange(s) % W for b, s in enumerate(sizes)])).astype(np.int64), len(sizes)


def test_random_job_sets(emu):
    rng = np.random.default_rng(41)
    arr, B = cutover_arrivals()
    for scale in (10, 2 ** 16, 2 ** 29):                      # 2^29: wait and turnaround need 4 radix passes
        jobs = _jobs_at(rng, arr, scale)
        recs = check(emu, jobs, arr, 10, B, 1, f"cut-over scale={scale}")
        assert recs["s"]["jc"]["jobs"].tolist() == [0, CUT - 1, CUT, CUT + 1, 1, 0, SUM_THREADS + 7, 3 * CUT]
        if scale == 2 ** 29:
            assert int(recs["s"]["sd_clamped"].sum()) > 0      # saturated slowdown
    for k in (0, 1, 5, 3000):
        for scale in (10, 2 ** 20):
            arrive = np.sort(rng.integers(0, 10 ** 6, k))
            jobs = _jobs_at(rng, arrive, scale)
            for W, B, tau in ((1, 1024, 1), (10 ** 6 + 1, 16, 1), (1000, 128, 30), (10 ** 4, 4, 1), (997, 1024, 10 ** 9)):
                check(emu, jobs, arrive, W, B, tau, f"k={k} scale={scale} W={W} B={B}")
    # most jobs in the open-ended last bin; every arrival on a bin edge
    arrive = np.sort(np.concatenate([rng.integers(0, 100, 20), rng.integers(10 ** 5, 10 ** 6, 2000)]))
    check(emu, _jobs_at(rng, arrive, 100), arrive, 10, 8, 1, "open-ended last bin")
    edges = np.repeat(np.arange(0, 64) * 50, 3)
    check(emu, _jobs_at(rng, edges, 1000), edges, 50, 64, 1, "arrivals on bin edges")


def test_unfinished_jobs_are_arrived_only(emu):
    rng = np.random.default_rng(3)
    ta = np.sort(rng.integers(0, 5000, 1200))
    fin = rng.permutation(1200)[:700]                        # 500 jobs have not finished
    jobs = _jobs_at(rng, ta[fin], 100)
    recs = check(emu, jobs, ta, 100, 64, 1, "unfinished")
    assert int((recs["arrived"] - recs["s"]["jc"]["jobs"]).sum()) == 500 and (recs["arrived"] >= recs["s"]["jc"]["jobs"]).all()


def test_one_bin_is_the_slowdown_class_but_for_the_key(emu):
    """at B = 1 the record is gs_sd_serial's C = 1 record with the same tau, except key_sum"""
    from test_slowdown_cpu import emu_slowdown
    out = os.path.join(os.path.dirname(emu._name), "libslowdown_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "slowdown_emu.cpp")], check=True)
    sd = C.CDLL(out)
    sd.emu_sd_jobs.restype = C.c_int
    rng = np.random.default_rng(8)
    arrive = np.sort(rng.integers(0, 10 ** 5, 900))
    jobs = _jobs_at(rng, arrive, 2 ** 18)
    for tau in (1, 60):
        _, recs = emu_arrivals(emu, jobs, arrive, 7, 1, tau)
        _, s, _ = emu_slowdown(sd, jobs, "gpus", (), tau, (), ())
        a, b = recs[0]["s"].copy(), s[0].copy()
        a["key_sum_lo"] = a["key_sum_hi"] = b["key_sum_lo"] = b["key_sum_hi"] = 0
        assert a.tobytes() == b.tobytes()


def test_setting_errors_leave_outputs_untouched(emu):
    jobs = tuple(np.ones(4, dtype=np.int64) for _ in range(6))
    ta = np.ones(4, dtype=np.int64)
    for W, B, tau in ((1, 1, 1), (1, 1024, 1), (2 ** 62, 5, 2 ** 62)):
        assert emu.emu_arr_check(W, B, tau) == 0
    assert emu.emu_arr_check(0, 0, 0) == 0 and emu.emu_arr_check(-5, 0, -5) == 0         # off: W and tau are ignored
    for W, B, tau in ((0, 1, 1), (-1, 1, 1), (1, 1, 0), (1, 1, -3), (1, 1025, 1), (1, -1, 1), (1, 2 ** 30, 1)):
        assert emu.emu_arr_check(W, B, tau) == -1, (W, B, tau)
        rc, recs = emu_arrivals(emu, jobs, ta, W, B, tau)
        assert rc == -1 and recs.tobytes() == b"\xab" * len(recs.tobytes())
    assert emu_arrivals(emu, jobs, ta, 1, 0, 1)[0] == -1                                   # off: nothing to compute


# ---------------------------------------------------------------- gs_horus_set_arrivals / gs_horus_fetch_arrivals, host build of gs_horus.cu
def test_horus_arrivals_host_build_matches_reference(horus_emu_engine):
    from gpuschedule_b200 import capi
    cases = horus_cases()
    loaded = [load_horus(c) for c in cases]
    with horus_emu_engine(device=0, nsims=len(cases)) as eng:
        for i, (table, cluster, params, _, _) in enumerate(loaded):
            eng.config(i, cluster, capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"]))
            eng.load_trace(i, table)
            np.random.seed(params["seed"])
            eng.load_words(i, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))
        for W, B, tau in ((0, 1, 1), (1, 1, 0), (1, 1025, 1), (1, -1, 1)):
            assert _code(eng.set_arrivals, W, B, tau) == capi.GS_ERR_ARG, (W, B, tau)
        assert _code(eng.arrivals) == capi.GS_ERR_STATE                        # off
        eng.set_arrivals(100, 16)
        assert _code(eng.arrivals) == capi.GS_ERR_STATE                        # nothing has run
        eng.run(rows_cap=1 << 15)
        assert _code(eng.arrivals) == capi.GS_ERR_STATE                        # not summarised
        eng.set_arrivals(0, 0)
        plain = eng.summarize()
        eng.set_slowdown("length", (60,), 1, (), ())                           # both on: each keeps its own state
        sd_before = None
        for W, B, tau in ((100, 16, 1), (1, 1024, 1), (7, 1, 60), (10 ** 9, 3, 1)):
            eng.set_arrivals(W, B, tau)
            assert _code(eng.arrivals) == capi.GS_ERR_STATE                    # setting it asks for a new summary
            assert eng.summarize().tobytes() == plain.tobytes()                # the summaries do not change
            sd = eng.slowdown()[0]
            assert sd_before is None or sd.tobytes() == sd_before.tobytes()
            sd_before = sd
            recs = eng.arrivals()
            assert recs.shape == (len(cases), B)
            assert eng.arrivals(first=2, count=3).tobytes() == recs[2:5].tobytes()
            assert _code(eng.arrivals, 3, len(cases)) == capi.GS_ERR_ARG
            assert _code(eng.arrivals, -1, 1) == capi.GS_ERR_ARG
            for i, (case, (table, _, _, _, _)) in enumerate(zip(cases, loaded)):
                _, _, _, hrecs, order = eng.fetch(i)
                assert_arrivals(recs[i], reference_arrivals(*job_columns(table, hrecs, order), table.arrive_tick, W, B, tau), f"{case} W={W}")
                assert_arrivals(recs[i], reference_arrivals(*csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table), table.arrive_tick,
                                                            W, B, tau), f"{case} job.csv W={W}")
        eng.set_arrivals(0, 0)
        assert _code(eng.arrivals) == capi.GS_ERR_STATE
        assert eng.slowdown()[0].shape[1] == 2                                 # slowdown is still on


# ---------------------------------------------------------------- summary.arrivals_derived / arrivals_spread
def test_arrivals_derived_matches_pandas_on_a_fixture_job_csv(emu):
    import pandas as pd
    from gpuschedule_b200 import summary
    case = next(c for k, c in FIXTURES if k == "fifo")
    table = load_golden(case)[0]
    jobs = csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table)
    jb = pd.read_csv(os.path.join(GOLDEN, case, "job.csv"))
    jb["arrive"] = jobs[0]
    W, B, tau = max(1, int(table.arrive_tick.max()) // 9), 8, 5
    _, recs = emu_arrivals(emu, jobs, table.arrive_tick, W, B, tau)
    d = summary.arrivals_derived(recs)
    jb["bin"] = np.minimum(jb["submit_time"] // W, B - 1)
    assert (jb["submit_time"].to_numpy() == jobs[0]).all()
    jb["wait"] = jb["start_time"] - jb["submit_time"]
    jb["turnaround"] = jb["end_time"] - jb["submit_time"]
    jb["sd"] = [min(SD_MAX, max(1024, (1024 * t) // max(j, tau))) / 1024 for t, j in zip(jb["turnaround"], jb["jct"])]
    g = jb.groupby("bin")
    for b in range(B):
        if b not in g.groups:
            assert d["jobs"][b] == 0 and math.isnan(d["wait_mean"][b]) and math.isnan(d["key_mean"][b])
            continue
        x = g.get_group(b)
        assert d["jobs"][b] == len(x)
        assert math.isclose(d["key_mean"][b], x["submit_time"].mean(), rel_tol=1e-12)
        for q in ("wait", "turnaround", "jct", "sd"):
            m = q + "_mean" if q != "sd" else "sd_mean"
            assert math.isclose(d[m][b], x[q].mean(), rel_tol=1e-12), (b, q)
            if len(x) > 1:
                assert math.isclose(d[q + "_std"][b], x[q].std(), rel_tol=1e-9), (b, q)
            s = np.sort(x[q].to_numpy())
            for p, pm in zip(summary.QUANTILES, PERMILLE):
                assert d[f"{q}_p{p}"][b] == s[(pm * len(s) + 999) // 1000 - 1]
    assert d["arrived"].sum() == table.n and (d["unfinished"] == d["arrived"] - d["jobs"]).all()
    assert len(summary.arrivals_flat(d, 0)) == len(summary.arrivals_columns())
    with pytest.raises(ValueError):
        summary.arrivals_derived(np.stack([recs, recs]))


def test_arrivals_spread_over_the_replicas_with_finished_jobs_in_a_bin(emu):
    from gpuschedule_b200 import summary
    rng = np.random.default_rng(12)
    recs = []
    for r in range(5):
        arrive = np.sort(rng.integers(0, 300 if r % 2 else 200, 60))         # bin 2 of width 100 only in odd replicas
        recs.append(emu_arrivals(emu, _jobs_at(rng, arrive, 50), arrive, 100, 3, 1)[1])
    recs = np.stack(recs)
    sp = summary.arrivals_spread(recs, level=0.9)
    assert sp["replicas"].tolist() == [5, 5, 2]
    per = [summary.arrivals_derived(recs[r]) for r in range(5)]
    v = np.array([per[r]["sd_mean"][2] for r in (1, 3)])
    ref = summary._spread_of(v, summary.Fraction("0.9"))
    assert [sp["sd_mean"][s][2] for s in summary.SPREAD_STATS] == pytest.approx([ref[s] for s in summary.SPREAD_STATS])
    assert sp["arrived"]["mean"][0] == pytest.approx(np.mean([per[r]["arrived"][0] for r in range(5)]))
    assert len(summary.arrivals_spread_flat(sp, 0)) == len(summary.arrivals_spread_columns())
    with pytest.raises(ValueError):
        summary.arrivals_spread(recs[0])
    with pytest.raises(ValueError):
        summary.arrivals_spread(recs, level=0)


# ---------------------------------------------------------------- the sweep: argument errors (before any engine exists) and columns
def test_sweep_arrivals_argument_errors(tmp_path, monkeypatch):
    from gpuschedule_b200 import capi, sweep

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(capi, "Engine", no_engine)
    monkeypatch.setattr(capi, "HorusEngine", no_engine)
    fl = [sweep.make_flags(trace_file=str(tmp_path / "missing.csv"))]
    for bad in ((0, 8, 1), (-1, 8, 1), (2 ** 63, 8, 1), (10, 0, 1), (10, 1025, 1), (10, 8, 0), (10, 8, 2 ** 63), (10, 8), 5, "abc",
                ("x", 8, 1)):
        with pytest.raises(ValueError):
            sweep.summarize_batched(fl, arrivals=bad)
        with pytest.raises(ValueError):
            sweep.summarize_bootstrap(fl, 2, arrivals=bad)
    assert sweep.check_arrivals(("500", 128, 1)) == (500, 128, 1)
    base = ["--trace", str(tmp_path / "missing.csv")]
    for argv in (["--arrivals", "a.csv", "--arrival-width", "10"],                                  # no --summary
                 ["--summary", "s.csv", "--arrivals", "a.csv"],                                     # no --arrival-width
                 ["--summary", "s.csv", "--arrival-width", "10"], ["--summary", "s.csv", "--arrival-bins", "5"],   # no --arrivals
                 ["--summary", "s.csv", "--arrival-bound", "5"],
                 ["--summary", "s.csv", "--arrivals", "a.csv", "--arrival-width", "0"],
                 ["--summary", "s.csv", "--arrivals", "a.csv", "--arrival-width", "10", "--arrival-bins", "0"],
                 ["--summary", "s.csv", "--arrivals", "a.csv", "--arrival-width", "10", "--arrival-bins", "1025"],
                 ["--summary", "s.csv", "--arrivals", "a.csv", "--arrival-width", "10", "--arrival-bound", "0"],
                 ["--summary", "s.csv", "--arrivals", "a.csv", "--arrival-width", "10", "--slowdown-bound", "5"],
                 ["--summary", "s.csv", "--arrivals", "a.csv", "--arrival-width", "10", "--bins", "5"],
                 ["--summary", "s.csv", "--arrivals", "a.csv", "--arrival-width", "10", "--bootstrap", "0"],
                 ["--summary", "s.csv", "--arrivals", "a.csv", "--arrival-width", "10", "--bootstrap", "2", "--schedule", "horus"]):
        with pytest.raises(SystemExit) as e:
            sweep.main(base + argv)
        assert e.value.code == 2, argv
    for name in ("a.csv", "s.csv"):
        assert not (tmp_path / name).exists()


def _flag_set(tmp_path):
    from gpuschedule_b200 import sweep
    return [sweep.make_flags(trace_file=str(tmp_path / "t.csv"), schedule=sc, seed=3) for sc in ("fifo", "dlas-gpu")]


def test_sweep_arrivals_writers_columns(emu, tmp_path):
    from gpuschedule_b200 import summary, sweep
    rng = np.random.default_rng(2)
    arrive = np.sort(rng.integers(0, 1000, 200))
    rec = emu_arrivals(emu, _jobs_at(rng, arrive, 50), arrive, 100, 4, 3)[1]
    sets = _flag_set(tmp_path)
    path = tmp_path / "a.csv"
    sweep.write_arrivals_csv(str(path), sets, np.stack([rec, rec]), (100, 4, 3))
    with open(path, newline="") as f:
        lines = list(csv.reader(f))
    assert lines[0] == sweep.SUMMARY_KEYS + ["bin", "bin_start", "bin_end", "tau"] + summary.arrivals_columns()
    assert len(lines) == 1 + 2 * 4
    assert [ln[6:10] for ln in lines[1:5]] == [["0", "0", "100", "3"], ["1", "100", "200", "3"], ["2", "200", "300", "3"], ["3", "300", "inf", "3"]]
    assert sum(int(ln[10]) for ln in lines[1:5]) == 200
    recs = np.broadcast_to(rec, (2, 2, 2, 3, 4)).copy()                       # (configurations, loads, profiles, replicas, B)
    ci = tmp_path / "ci.csv"
    sweep.write_arrivals_ci_csv(str(ci), sets, [1.0, 2.0], recs, (100, 4, 3), block_len=4, profile=["0:1", "0:1,50:3"])
    with open(ci, newline="") as f:
        lines = list(csv.reader(f))
    assert lines[0] == (sweep.SUMMARY_KEYS + ["load", "block_len", "profile", "bin", "bin_start", "bin_end", "tau", "replicas", "level"]
                        + summary.arrivals_spread_columns())
    assert len(lines) == 1 + 2 * 2 * 2 * 4 and lines[1][6:9] == ["1.0", "4", "0:1"] and lines[4][11:15] == ["inf", "3", "3", "0.95"]

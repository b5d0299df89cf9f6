"""Job statistics by arrival time on the device (gs_set_arrivals / gs_fetch_arrivals, gs_horus_set_arrivals /
gs_horus_fetch_arrivals) on the H100.

Device records must equal test_arrivals_cpu.reference_arrivals over the job records, finish orders and traces the
engine itself hands out (and, for the fixtures, the reference-made job.csv or the policy oracles' records), byte for
byte in every field.  The bins add up to the summary's job part and to the trace; at B = 1 a bin is slowdown's C = 1
record but for the key sum; with the feature off nothing changes."""
import csv
import os
import subprocess
import sys
import types

import numpy as np
import pytest

from conftest import GOLDEN, REPO, golden_cases, horus_cases, load_golden, load_horus
from test_arrivals_cpu import CUT, SUM_THREADS, assert_arrivals, cutover_arrivals, reference_arrivals
from test_gpu_summary import _engine_run, _fifo_handle, _sweep_flags, _synth
from test_jobdist_cpu import csv_jobs
from test_summary_cpu import _policy_cases, job_columns, load_policy

pytestmark = pytest.mark.gpu

JOB_FIELDS = ("wait_sum", "turnaround_sum", "jct_sum", "preempt_sum", "gpu_ticks_sum")


def settings(last):
    """(W, B, tau) settings: one bin, W = 1 at 1024 bins, about 100 bins over the trace, W past the last arrival"""
    return ((1, 1, 1), (1, 1024, 1), (max(1, last // 100), 128, 1), (max(1, last // 7), 8, 60), (last + 1, 4, 1), (500, 128, 1))


def check_invariants(recs, rec, n, tag=""):
    """sum of arrived = n; the bins' jobs and sums add up to the summary's; the largest bin maximum is the summary's"""
    jc = recs["s"]["jc"]
    assert int(recs["arrived"].sum()) == n, tag
    assert int(jc["jobs"].sum()) == int(rec["finished"]), tag
    assert (recs["arrived"] >= jc["jobs"]).all(), tag
    for f in JOB_FIELDS:
        assert int(jc[f].sum()) == int(rec[f]), (tag, f)
    has = jc["jobs"] > 0
    if has.any():
        for f in ("wait_q", "turnaround_q", "jct_q"):
            assert int(jc[f][has, 4].max()) == int(rec[f][4]), (tag, f)


def _trace_cols(packed):
    return types.SimpleNamespace(arrive_tick=packed["arrive_tick"].astype(np.int64), gpus=packed["gpus"].astype(np.int64))


def _table_at(arrive, seed=1):
    """a synthetic trace whose jobs arrive at the given ticks (the first at tick 0: a trace's ticks start at its first
    arrival)"""
    from gpuschedule_b200 import ingest, tracegen
    cols = tracegen.synth_columns(len(arrive), seed=seed)
    cols["normalized_time"] = np.asarray(arrive, dtype=np.int64) * 10000
    table = ingest.table_from_columns(cols)
    assert np.array_equal(table.arrive_tick, arrive)
    return table


@pytest.mark.parametrize("case", golden_cases())
def test_fifo_fixture_arrivals_on_device(case):
    from gpuschedule_b200 import capi
    table, cluster, _, _, _ = load_golden(case)
    want_jobs = csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table)
    with capi.Engine(device=0, nsims=1) as eng:
        eng.config(0, cluster)
        eng.load_trace(0, table)
        out, _, _ = _engine_run(eng)
        recs_j, order = eng.fetch_jobs(0)
        for W, B, tau in settings(int(table.arrive_tick.max())):
            eng.set_arrivals(W, B, tau)
            assert eng.summarize().tobytes() == out.tobytes()
            recs = eng.arrivals()[0]
            tag = f"{case} W={W} B={B} tau={tau}"
            assert_arrivals(recs, reference_arrivals(*want_jobs, table.arrive_tick, W, B, tau), tag)
            assert_arrivals(recs, reference_arrivals(*job_columns(table, recs_j, order), table.arrive_tick, W, B, tau), tag)
            check_invariants(recs, out[0], table.n, tag)


@pytest.mark.parametrize("case", _policy_cases())
def test_policy_fixture_arrivals_on_device(case):
    import oracle
    from gpuschedule_b200 import capi
    table, cluster, pol = load_policy(case)
    res = oracle.run_policy(cluster, pol, table)
    want_jobs = job_columns(table, res.recs, res.finish_order)
    with capi.Engine(device=0, nsims=1) as eng:
        eng.config(0, cluster, pol)
        eng.load_trace(0, table)
        eng.set_arrivals(10, 16)
        out, _, _ = _engine_run(eng)
        recs_j, order = eng.fetch_jobs(0)
        for W, B, tau in settings(int(table.arrive_tick.max())):
            eng.set_arrivals(W, B, tau)
            eng.summarize()
            recs = eng.arrivals()[0]
            tag = f"{case} W={W} B={B} tau={tau}"
            assert_arrivals(recs, reference_arrivals(*want_jobs, table.arrive_tick, W, B, tau), tag)
            assert_arrivals(recs, reference_arrivals(*job_columns(table, recs_j, order), table.arrive_tick, W, B, tau), tag)
            check_invariants(recs, out[0], table.n, tag)


def test_horus_fixtures_arrivals_on_device():
    from gpuschedule_b200 import capi
    cases = horus_cases()
    loaded = [load_horus(c) for c in cases]
    with capi.HorusEngine(device=0, nsims=len(cases)) as eng:
        for i, (table, cluster, params, _, _) in enumerate(loaded):
            eng.config(i, cluster, capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"]))
            eng.load_trace(i, table)
            np.random.seed(params["seed"])
            eng.load_words(i, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))
        eng.run(rows_cap=1 << 15)
        n0 = eng.lib.gs_horus_launch_count(eng.h)
        plain = eng.summarize()
        assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 2
        last = max(int(t[0].arrive_tick.max()) for t in loaded)
        for W, B, tau in settings(last):
            eng.set_arrivals(W, B, tau)
            n0 = eng.lib.gs_horus_launch_count(eng.h)
            out = eng.summarize()
            assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 3
            assert out.tobytes() == plain.tobytes()
            recs = eng.arrivals()
            for i, (case, (table, _, _, _, _)) in enumerate(zip(cases, loaded)):
                _, _, _, hrecs, order = eng.fetch(i)
                tag = f"{case} W={W} B={B}"
                assert_arrivals(recs[i], reference_arrivals(*job_columns(table, hrecs, order), table.arrive_tick, W, B, tau), tag)
                assert_arrivals(recs[i], reference_arrivals(*csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table), table.arrive_tick,
                                                            W, B, tau), tag)
                check_invariants(recs[i], out[i], table.n, tag)
        eng.set_arrivals(0, 0)
        n0 = eng.lib.gs_horus_launch_count(eng.h)
        assert eng.summarize().tobytes() == plain.tobytes()
        assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 2


def test_cutover_bins_and_more_replicas_than_the_grid():
    """bins of exactly GS_ARR_CUT finished jobs and one on each side of it, a bin past GS_SUM_THREADS, empty bins and a
    crowded open-ended last bin, under fifo and the policies, on a handle of 700 replicas (more than the launched
    grid); a second trace spreads the same jobs over 2^17 times the ticks.  One more job arrives at tick 0, where a
    trace's ticks start."""
    from gpuschedule_b200 import capi, policies
    arr, B = cutover_arrivals(10)
    arr = np.concatenate([[0], arr])
    base = _table_at(arr)
    wide = _table_at(arr * 2 ** 17 // 10, seed=2)
    R = 700
    pols = [None, capi.make_policy("sjf"), capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,)),
            capi.make_policy("gittins", gittins_table=policies.build_gittins_table(policies.gittins_samples(base), 3250.0)), None]
    configs = [(capi.make_cluster(2, 8, 8), wide if i % 5 == 4 else base, pols[i % 5]) for i in range(R)]
    with capi.Engine(device=0, nsims=R) as eng:
        for i, (cl, table, pol) in enumerate(configs):
            eng.config(i, cl, pol)
            eng.load_trace(i, table)
        out, _, _ = _engine_run(eng, 3000)
        res = {}
        for W, Bn in ((10, B), (2 ** 17, B), (1, 1024)):
            eng.set_arrivals(W, Bn)
            eng.summarize()
            res[(W, Bn)] = eng.arrivals()
        assert eng.arrivals(first=640, count=60).tobytes() == res[(1, 1024)][640:].tobytes()
        jobs = [job_columns(configs[i][1], *eng.fetch_jobs(i)) for i in range(R)]
    for i in range(0, R, 7):
        for (W, Bn), recs in res.items():
            tag = f"replica {i} W={W} B={Bn}"
            assert_arrivals(recs[i], reference_arrivals(*jobs[i], configs[i][1].arrive_tick, W, Bn, 1), tag)
            check_invariants(recs[i], out[i], configs[i][1].n, tag)
    sizes = res[(10, B)][0]["s"]["jc"]["jobs"].tolist()
    assert sizes == [1, CUT - 1, CUT, CUT + 1, 1, 0, SUM_THREADS + 7, 3 * CUT]


def test_multi_window_arrivals_follow_the_finished_jobs():
    from gpuschedule_b200 import capi
    for table, pol in ((_synth(100000, 3), None), (_synth(20000, 4), capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,)))):
        W, B = int(table.arrive_tick.max()) // 64 + 1, 64
        with capi.Engine(device=0, nsims=1) as eng:
            eng.config(0, capi.make_cluster(4, 32, 8), pol)
            eng.load_trace(0, table)
            eng.set_arrivals(W, B)
            _engine_run(eng)
            whole = eng.arrivals()
            eng.reset()
            seen = []
            while True:
                eng.run(0, 7000)
                s = eng.summarize()
                seen.append((s[0].copy(), eng.arrivals()[0].copy()))
                if s[0]["done"]:
                    break
            recs, order = eng.fetch_jobs(0)
        assert len(seen) >= 3
        for s, r in seen:
            k = int(s["finished"])
            assert_arrivals(r, reference_arrivals(*job_columns(table, recs, order[:k]), table.arrive_tick, W, B, 1), f"finished={k}")
            check_invariants(r, s, table.n, f"finished={k}")
        assert int((seen[0][1]["arrived"] - seen[0][1]["s"]["jc"]["jobs"]).sum()) > 0     # arrived > jobs after a window
        assert seen[-1][1].tobytes() == whole[0].tobytes()


@pytest.mark.parametrize("kind", ["iid", "blocked", "mixed", "profiled"])
def test_bootstrap_replicas(kind):
    from gpuschedule_b200 import capi, tracegen
    base = _synth(4000, 21)
    R = 12
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, capi.make_cluster(2, 16, 8), None if i % 2 else capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,)))
        eng.boot_population(base)
        params = np.zeros(R, dtype=capi.BOOT_PARAMS_DTYPE)
        params["seed"], params["stream"], params["n"], params["gap_num"], params["gap_den"] = 7, np.arange(R), 4000, 5, 6
        if kind == "mixed":
            eng.boot_mixes(np.stack([tracegen.class_weights(base.gpus, (4,), (1, 5)), tracegen.class_weights(base.gpus, (4,), (3, 1))]))
            eng.boot_traces(params, block_len=8, mix=np.arange(R) % 3 - 1)
        elif kind == "profiled":                                    # a 3x surge from tick 2000 to 2600
            params["gap_num"], params["gap_den"] = 1, 1
            eng.boot_profiles([([(0, 1, 1), (2000, 1, 3), (2600, 1, 1)], 0)])
            eng.boot_traces(params, profile=np.zeros(R, dtype=np.int32))
        else:
            eng.boot_traces(params, block_len=None if kind == "iid" else 16)
        W, B = 100, 128
        eng.set_arrivals(W, B, 30)
        out = eng.run_summarized()
        recs = eng.arrivals()
        for r in range(R):
            table = _trace_cols(eng.fetch_trace(r))
            jobs = job_columns(table, *eng.fetch_jobs(r))
            assert_arrivals(recs[r], reference_arrivals(*jobs, table.arrive_tick, W, B, 30), f"{kind} replica {r}")
            check_invariants(recs[r], out[r], 4000, f"{kind} replica {r}")
        if kind == "profiled":                                       # the surge's bins receive three times the jobs
            a = recs["arrived"].astype(np.int64)
            assert a[:, 20:26].mean() > 2 * a[:, 10:16].mean()
        params["stream"] = params["stream"][::-1]                   # regenerated replicas must be summarised again
        eng.boot_traces(params)
        with pytest.raises(capi.GsError) as e:
            eng.arrivals()
        assert e.value.code == capi.GS_ERR_STATE


def test_100k_job_replica_at_1024_bins_and_one_bin_is_the_slowdown_class():
    from gpuschedule_b200 import capi
    table = _synth(100000, 5)
    W = int(table.arrive_tick.max()) // 1024 + 1
    with capi.Engine(device=0, nsims=1) as eng:
        eng.config(0, capi.make_cluster(4, 32, 8))
        eng.load_trace(0, table)
        eng.set_arrivals(W, 1024)
        out, _, _ = _engine_run(eng)
        recs = eng.arrivals()[0]
        jobs = job_columns(table, *eng.fetch_jobs(0))
        assert_arrivals(recs, reference_arrivals(*jobs, table.arrive_tick, W, 1024, 1), "100k jobs")
        check_invariants(recs, out[0], table.n, "100k jobs")
        assert eng.arrivals().tobytes() == recs.tobytes()                     # a repeated fetch gives the same bytes
        for tau in (1, 60, 10 ** 6):
            eng.set_arrivals(7, 1, tau)
            eng.set_slowdown("gpus", (), tau, (), ())
            eng.summarize()
            a = eng.arrivals()[0][0]["s"].copy()
            b = eng.slowdown()[0][0][0].copy()
            assert int(eng.arrivals()[0][0]["arrived"]) == table.n
            a["key_sum_lo"] = a["key_sum_hi"] = b["key_sum_lo"] = b["key_sum_hi"] = 0
            assert a.tobytes() == b.tobytes(), tau


def test_feature_off_changes_nothing_and_repeats_are_byte_equal():
    """summaries, results and launch counts with the feature off are those of a handle that never had it; on, one
    more launch per summarize, and a repeated call or a reset run gives the same bytes"""
    from gpuschedule_b200 import capi
    tables = [_synth(5000, 40 + i) for i in range(4)]
    cluster = capi.make_cluster(4, 32, 8)
    got, per_call = [], []
    for mode in ("never", "off", "on"):
        eng = _fifo_handle(capi, tables, cluster)
        if mode != "never":
            eng.set_arrivals(50, 256, 10)
            if mode == "off":
                eng.set_arrivals(0, 0)
        blobs, calls = [], []
        while True:
            eng.run(0, 3000)
            n0 = eng.launch_count()
            blobs.append(eng.summarize().tobytes())
            calls.append(eng.launch_count() - n0)
            pitch = max(eng.result_layout(i).block_bytes for i in range(len(tables)))
            buf = np.zeros(pitch * len(tables), dtype=np.uint8)
            eng.fetch_results(buf, pitch)
            eng.sync()
            blobs.append(buf.tobytes())
            if all(eng.stats(i).done for i in range(len(tables))):
                break
        if mode == "on":
            a = eng.arrivals()
            s = eng.summarize()
            assert eng.arrivals().tobytes() == a.tobytes()
            eng.reset()
            assert eng.run_summarized(rows_cap=3000).tobytes() == s.tobytes()
            assert eng.arrivals().tobytes() == a.tobytes()
        eng.close()
        got.append(blobs)
        per_call.append(set(calls))
    assert got[0] == got[1] == got[2]
    assert per_call == [{2}, {2}, {3}]


def test_error_codes_on_device():
    from gpuschedule_b200 import capi
    eng = _fifo_handle(capi, [_synth(20000, 9)] * 2, capi.make_cluster(4, 32, 8))

    def code(fn, *a):
        with pytest.raises(capi.GsError) as e:
            fn(*a)
        return e.value.code
    try:
        for W, B, tau in ((0, 1, 1), (1, 1, 0), (1, 1025, 1), (1, -1, 1)):
            assert code(eng.set_arrivals, W, B, tau) == capi.GS_ERR_ARG
        assert code(eng.arrivals) == capi.GS_ERR_STATE                      # off
        eng.set_arrivals(100, 8)
        assert code(eng.arrivals) == capi.GS_ERR_STATE                      # nothing has run
        eng.run(0, 5000)
        assert code(eng.arrivals) == capi.GS_ERR_STATE                      # not summarised
        eng.summarize()
        r1 = eng.arrivals()
        for first, count in ((-1, 1), (0, 3), (2, 1)):
            assert code(eng.arrivals, first, count) == capi.GS_ERR_ARG
        eng.set_arrivals(7, 3)
        assert code(eng.arrivals) == capi.GS_ERR_STATE
        eng.summarize()
        assert eng.arrivals().shape == (2, 3)
        eng.set_arrivals(100, 8)
        eng.summarize()
        assert eng.arrivals().tobytes() == r1.tobytes()
        big = capi.Engine(device=0, nsims=350000)                           # 350000 x 1024 x 240 B: more than the card holds
        try:
            assert code(big.set_arrivals, 1, 1024) == capi.GS_ERR_CAPACITY
            big.set_arrivals(1, 4)                                          # the handle is still usable
        finally:
            big.close()
        eng.reset()
        assert code(eng.arrivals) == capi.GS_ERR_STATE
    finally:
        eng.close()


# ---------------------------------------------------------------- sweep
def test_sweep_arrivals_equal_the_files_run_batched_writes(tmp_path):
    from gpuschedule_b200 import ingest, sweep
    trace, sets = _sweep_flags(tmp_path)
    arr = (50, 32, 10)
    recs, arec = sweep.summarize_batched(sets, arrivals=arr)
    recs2, (srec, _), arec2 = sweep.summarize_batched(sets, slowdown=("length", (60,), 1, (), ()), arrivals=arr)
    assert recs2.tobytes() == recs.tobytes() and arec2.tobytes() == arec.tobytes()
    written = sweep.run_batched(sets, out_root=str(tmp_path / "log"))
    table = ingest.JobTraceReader(trace).prepare_jobs().table(0.5)
    for fl, rec, rc, (out_dir, _) in zip(sets, recs, arec, written):
        assert_arrivals(rc, reference_arrivals(*csv_jobs(os.path.join(out_dir, "job.csv"), table), table.arrive_tick, *arr), fl.schedule)
        check_invariants(rc, rec, table.n, fl.schedule)


def test_sweep_command_line_writes_the_arrivals_csv(tmp_path):
    from gpuschedule_b200 import summary, sweep
    trace, _ = _sweep_flags(tmp_path)
    env = {**os.environ, "PYTHONPATH": REPO}
    run = lambda argv: subprocess.run([sys.executable, "-m", "gpuschedule_b200.sweep", "--trace", trace, "--num_switch", "1",
                                       "--num_node_p_switch", "8"] + argv, check=True, cwd=str(tmp_path), env=env)
    read = lambda p: list(csv.reader(open(p, newline="")))
    # without --bootstrap, with horus under --repeats: the summary and timeline files do not change
    common = ["--schedule", "fifo", "dlas-gpu", "horus", "--repeats", "2", "--seed", "3"]
    run(common + ["--summary", "s0.csv", "--timeline", "t0.csv", "--bin-width", "50"])
    run(common + ["--summary", "s1.csv", "--timeline", "t1.csv", "--bin-width", "50", "--arrivals", "a.csv", "--arrival-width", "50",
                  "--arrival-bins", "16", "--arrival-bound", "5"])
    for a, b in (("s0.csv", "s1.csv"), ("t0.csv", "t1.csv")):
        assert open(tmp_path / a, "rb").read() == open(tmp_path / b, "rb").read()
    lines, srows = read(tmp_path / "a.csv"), read(tmp_path / "s1.csv")
    assert lines[0] == sweep.SUMMARY_KEYS + ["bin", "bin_start", "bin_end", "tau"] + summary.arrivals_columns()
    assert len(lines) == 1 + 6 * 16 and lines[16][6:10] == ["15", "750", "inf", "5"]
    fin = srows[0].index("finished")
    for c in range(6):
        part = lines[1 + 16 * c:17 + 16 * c]
        assert sum(int(ln[10]) for ln in part) == 400                       # arrived
        assert sum(int(ln[11]) for ln in part) == int(srows[1 + c][fin])   # finished jobs
    # with --bootstrap and a 3x surge of the offered load
    run(["--schedule", "fifo", "dlas-gpu", "--bootstrap", "3", "--load", "1", "--load-profile", "0:1,200:3,300:1", "0:1",
         "--summary", "b.csv", "--arrivals", "ci.csv", "--arrival-width", "25", "--arrival-bins", "32"])
    lines = read(tmp_path / "ci.csv")
    assert lines[0] == (sweep.SUMMARY_KEYS + ["load", "profile", "bin", "bin_start", "bin_end", "tau", "replicas", "level"]
                        + summary.arrivals_spread_columns())
    assert len(lines) == 1 + 2 * 2 * 32 and lines[1][7] == "0:1,200:3,300:1"
    assert all(0 <= int(ln[12]) <= 3 for ln in lines[1:])

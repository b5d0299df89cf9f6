"""Job statistics by job size on the device (gs_set_jobdist / gs_fetch_jobdist, gs_horus_set_jobdist /
gs_horus_fetch_jobdist) on the H100.

Device class records and CDF counts must equal the numpy breakdown of test_jobdist_cpu.py over two judges: the
fixtures' reference-made job.csv (fifo, horus) or the pinned policy oracles' records, and the job records the engine
itself hands out.  With one class they must equal gs_summarize's job part."""
import csv
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, REPO, golden_cases, horus_cases, load_golden, load_horus
from test_gpu_summary import _engine_run, _fifo_handle, _sweep_flags, _synth
from test_jobdist_cpu import DEFAULT_EDGES, assert_jobdist, csv_jobs, reference_jobdist
from test_summary_cpu import _policy_cases, job_columns, load_policy

pytestmark = pytest.mark.gpu

SETTINGS = (((), ()), ((5, 17, 65), DEFAULT_EDGES), ((1, 2, 3, 4, 8, 16, 32), tuple(range(0, 255 * 40, 40))), ((2,), (3, 100, 10 ** 6)))
JOB_FIELDS = ("wait_sum", "turnaround_sum", "jct_sum", "preempt_sum", "gpu_ticks_sum")


def check_against_summary(classes, hist, rec, tag=""):
    """class counts and sums add up to the summary's, histogram rows to their class's jobs; one class is the summary"""
    assert int(classes["jobs"].sum()) == int(rec["finished"]), tag
    for f in JOB_FIELDS:
        assert int(classes[f].sum()) == int(rec[f]), (tag, f)
    assert (hist.astype(np.int64).sum(axis=-1) == classes["jobs"][:, None]).all(), tag
    if len(classes) == 1:
        for f in ("wait_q", "turnaround_q", "jct_q"):
            assert classes[0][f].tolist() == rec[f].tolist(), (tag, f)


def _run(eng, bounds, edges, rows_cap=0):
    eng.set_jobdist(bounds, edges)
    out, _, _ = _engine_run(eng, rows_cap)
    return out, eng.jobdist()


@pytest.mark.parametrize("case", golden_cases())
def test_fifo_fixture_jobdist_on_device(case):
    from gpuschedule_b200 import capi
    table, cluster, _, _, _ = load_golden(case)
    want_jobs = csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table)
    for bounds, edges in SETTINGS:
        with capi.Engine(device=0, nsims=1) as eng:
            eng.config(0, cluster)
            eng.load_trace(0, table)
            out, (classes, hist) = _run(eng, bounds, edges)
            recs, order = eng.fetch_jobs(0)
        tag = f"{case} bounds={bounds}"
        assert_jobdist(classes[0], hist[0], reference_jobdist(*want_jobs, bounds, edges), tag)
        assert_jobdist(classes[0], hist[0], reference_jobdist(*job_columns(table, recs, order), bounds, edges), tag)
        check_against_summary(classes[0], hist[0], out[0], tag)


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("case", _policy_cases())
def test_policy_fixture_jobdist_on_device(case, mode):
    import oracle
    from gpuschedule_b200 import capi
    table, cluster, pol = load_policy(case)
    res = oracle.run_policy(cluster, pol, table)
    want_jobs = job_columns(table, res.recs, res.finish_order)
    for bounds, edges in SETTINGS:
        with capi.Engine(device=0, nsims=1) as eng:
            eng.set_engine(mode)
            eng.config(0, cluster, pol)
            eng.load_trace(0, table)
            out, (classes, hist) = _run(eng, bounds, edges)
            recs, order = eng.fetch_jobs(0)
        tag = f"{case} mode={mode} bounds={bounds}"
        assert_jobdist(classes[0], hist[0], reference_jobdist(*want_jobs, bounds, edges), tag)
        assert_jobdist(classes[0], hist[0], reference_jobdist(*job_columns(table, recs, order), bounds, edges), tag)
        check_against_summary(classes[0], hist[0], out[0], tag)


@pytest.mark.parametrize("case", horus_cases())
def test_horus_fixture_jobdist_on_device(case):
    from gpuschedule_b200 import capi
    table, cluster, params, _, _ = load_horus(case)
    want_jobs = csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table)
    with capi.HorusEngine(device=0, nsims=1) as eng:
        eng.config(0, cluster, capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"]))
        eng.load_trace(0, table)
        np.random.seed(params["seed"])
        eng.load_words(0, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))
        eng.run(rows_cap=1 << 15)
        _, _, _, hrecs, order = eng.fetch(0)
        plain = eng.summarize()
        for bounds, edges in SETTINGS:
            eng.set_jobdist(bounds, edges)
            n0 = eng.lib.gs_horus_launch_count(eng.h)
            out = eng.summarize()
            assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 3
            assert out.tobytes() == plain.tobytes()
            classes, hist = eng.jobdist()
            tag = f"{case} bounds={bounds}"
            assert_jobdist(classes[0], hist[0], reference_jobdist(*want_jobs, bounds, edges), tag)
            assert_jobdist(classes[0], hist[0], reference_jobdist(*job_columns(table, hrecs, order), bounds, edges), tag)
            check_against_summary(classes[0], hist[0], out[0], tag)
        eng.set_jobdist(None, None)
        n0 = eng.lib.gs_horus_launch_count(eng.h)
        eng.summarize()
        assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 2


def test_heterogeneous_replicas_in_one_handle():
    from gpuschedule_b200 import capi, policies
    configs = []
    for i in range(150):
        kind = i % 6
        table = _synth(300 + 7 * i, 100 + i, network=kind == 1)
        if kind in (0, 1):
            configs.append((capi.make_cluster(2, 8, 8, enable_network_costs=kind == 1), table, None))
        elif kind == 2:
            configs.append((capi.make_cluster(1, 8, 16, num_cpu_p_node=256, mem_p_node=1024), table, None))
        elif kind == 3:
            configs.append((capi.make_cluster(1, 4, 64, num_cpu_p_node=1024, mem_p_node=4096), table, None))
        else:
            sched = ("sjf", "dlas-gpu", "gittins")[i % 3]
            kw = dict(num_queue=2, queue_limit=(3600,)) if sched == "dlas-gpu" else {}
            if sched == "gittins":
                kw["gittins_table"] = policies.build_gittins_table(policies.gittins_samples(table), 3250.0)
            configs.append((capi.make_cluster(1, 16, 8), table, capi.make_policy(sched, **kw)))
    bounds, edges = (2, 5, 9, 17, 33, 65, 129), tuple(range(-3, 255 * 97 - 3, 97))
    with capi.Engine(device=0, nsims=len(configs)) as eng:
        for i, (cl, table, pol) in enumerate(configs):
            eng.config(i, cl, pol)
            eng.load_trace(i, table)
        out, (classes, hist) = _run(eng, bounds, edges, rows_cap=3000)
        part = eng.jobdist(first=40, count=7)
        assert part[0].tobytes() == classes[40:47].tobytes() and part[1].tobytes() == hist[40:47].tobytes()
        jobs = [job_columns(configs[i][1], *eng.fetch_jobs(i)) for i in range(len(configs))]
    for i in range(len(configs)):
        assert_jobdist(classes[i], hist[i], reference_jobdist(*jobs[i], bounds, edges), f"replica {i}")
        check_against_summary(classes[i], hist[i], out[i], f"replica {i}")


def test_multi_window_jobdist_follows_the_finished_jobs():
    """summarised after every window, the records are those of the jobs finished so far (finish order only grows),
    and the last window's equal a single-window run's"""
    from gpuschedule_b200 import capi
    bounds, edges = (2, 4, 8), DEFAULT_EDGES
    for table, pol in ((_synth(100000, 3), None), (_synth(20000, 4), capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,)))):
        with capi.Engine(device=0, nsims=1) as eng:
            eng.config(0, capi.make_cluster(4, 32, 8), pol)
            eng.load_trace(0, table)
            _, (whole_c, whole_h) = _run(eng, bounds, edges)
            eng.reset()
            seen = []
            while True:
                eng.run(0, 7000)
                s = eng.summarize()
                c, h = eng.jobdist()
                seen.append((int(s[0]["finished"]), c[0].copy(), h[0].copy()))
                if s[0]["done"]:
                    break
            recs, order = eng.fetch_jobs(0)
        assert len(seen) >= 3
        for k, c, h in seen:
            assert_jobdist(c, h, reference_jobdist(*job_columns(table, recs, order[:k]), bounds, edges), f"finished={k}")
        assert seen[-1][1].tobytes() == whole_c[0].tobytes() and seen[-1][2].tobytes() == whole_h[0].tobytes()


def test_repeat_reset_and_unchanged_outputs():
    """a second summarise and a reset run give the same bytes; summaries, results and launch counts with the feature
    off are those of a handle that never had it"""
    from gpuschedule_b200 import capi
    tables = [_synth(5000, 40 + i) for i in range(4)]
    cluster = capi.make_cluster(4, 32, 8)
    got, per_call = [], []
    for on in (False, True):
        eng = _fifo_handle(capi, tables, cluster)
        if on:
            eng.set_jobdist((5, 17, 65), DEFAULT_EDGES)
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
        if on:
            a = eng.jobdist()
            s = eng.summarize()
            b = eng.jobdist()
            assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
            eng.reset()                                                 # the same windows again
            assert eng.run_summarized(rows_cap=3000).tobytes() == s.tobytes()
            c = eng.jobdist()
            assert a[0].tobytes() == c[0].tobytes() and a[1].tobytes() == c[1].tobytes()
        eng.close()
        got.append(blobs)
        per_call.append(set(calls))
    assert len(got[0]) == len(got[1]) and all(x == y for x, y in zip(*got))
    assert per_call == [{2}, {3}]


def test_error_codes_setting_changes_and_restarts():
    from gpuschedule_b200 import capi
    table = _synth(20000, 9)
    eng = _fifo_handle(capi, [table, table], capi.make_cluster(4, 32, 8))

    def code(fn, *a):
        with pytest.raises(capi.GsError) as e:
            fn(*a)
        return e.value.code
    try:
        for bounds, edges in (((0,), ()), ((3, 3), ()), ((5, 2), ()), ((), (2, 2)), ((), (3, 1)), ((1, 2, 3, 4, 5, 6, 7, 8), ()),
                              ((), tuple(range(256)))):
            assert code(eng.set_jobdist, bounds, edges) == capi.GS_ERR_ARG, (bounds, len(edges))
        assert eng.lib.gs_set_jobdist(eng.h, 9, None, 0, None) == capi.GS_ERR_ARG
        assert eng.lib.gs_set_jobdist(eng.h, 2, None, 0, None) == capi.GS_ERR_ARG             # NULL bounds
        assert eng.lib.gs_set_jobdist(eng.h, 1, None, 3, None) == capi.GS_ERR_ARG             # NULL edges
        assert code(eng.jobdist) == capi.GS_ERR_STATE                       # off
        eng.set_jobdist((8,), (10, 100))
        assert code(eng.jobdist) == capi.GS_ERR_STATE                       # nothing has run
        eng.run(0, 5000)
        assert code(eng.jobdist) == capi.GS_ERR_STATE                       # not summarised
        s1 = eng.summarize()
        c1, h1 = eng.jobdist()
        for first, count in ((-1, 1), (0, 3), (2, 1), (1, -1)):
            assert code(eng.jobdist, first, count) == capi.GS_ERR_ARG, (first, count)
        eng.set_jobdist((2, 4), (5,))                                       # between two summarise calls: takes effect
        assert code(eng.jobdist) == capi.GS_ERR_STATE
        s2 = eng.summarize()
        c2, h2 = eng.jobdist()
        assert s2.tobytes() == s1.tobytes() and c2.shape == (2, 3) and h2.shape == (2, 3, 3, 2)
        check_against_summary(c2[0], h2[0], s2[0])
        eng.set_jobdist((8,), (10, 100))
        eng.summarize()
        c3, h3 = eng.jobdist()
        assert c3.tobytes() == c1.tobytes() and h3.tobytes() == h1.tobytes()
        eng.reset()                                                         # a reset replica is prepared afresh
        assert code(eng.jobdist) == capi.GS_ERR_STATE
        eng.run(0, 5000)
        eng.summarize()
        assert eng.jobdist()[0].tobytes() == c1.tobytes()
        eng.set_jobdist(None, None)
        assert code(eng.jobdist) == capi.GS_ERR_STATE
    finally:
        eng.close()
    # generated replicas: gs_boot_traces prepares them afresh
    base = _synth(3000, 12)
    with capi.Engine(device=0, nsims=2) as eng:
        for i in range(2):
            eng.config(i, capi.make_cluster(2, 8, 8))
        eng.boot_population(base)
        params = np.zeros(2, dtype=capi.BOOT_PARAMS_DTYPE)
        params["seed"], params["stream"], params["n"], params["gap_num"], params["gap_den"] = 3, [0, 1], 3000, 1, 1
        eng.set_jobdist((2, 4), DEFAULT_EDGES)
        eng.boot_traces(params)
        eng.run_summarized()
        ca, ha = eng.jobdist()
        params["stream"] = [1, 0]
        eng.boot_traces(params)
        with pytest.raises(capi.GsError) as e:
            eng.jobdist()
        assert e.value.code == capi.GS_ERR_STATE
        eng.run_summarized()
        cb, hb = eng.jobdist()
    assert cb[0].tobytes() == ca[1].tobytes() and cb[1].tobytes() == ca[0].tobytes()
    assert hb[0].tobytes() == ha[1].tobytes() and hb[1].tobytes() == ha[0].tobytes()


# ---------------------------------------------------------------- sweep
def test_sweep_jobdist_equals_the_files_run_batched_writes(tmp_path):
    from gpuschedule_b200 import ingest, sweep
    trace, sets = _sweep_flags(tmp_path)
    bounds, edges = (2, 4), (1, 10, 100, 1000)
    recs, (classes, hist) = sweep.summarize_batched(sets, jobdist=(bounds, edges))
    recs2, bins, (classes2, hist2) = sweep.summarize_batched(sets, timeline=(9, 40), jobdist=(bounds, edges))
    assert recs2.tobytes() == recs.tobytes() and classes2.tobytes() == classes.tobytes() and hist2.tobytes() == hist.tobytes()
    written = sweep.run_batched(sets, out_root=str(tmp_path / "log"))
    table = ingest.JobTraceReader(trace).prepare_jobs().table(0.5)
    for fl, rec, cl, hs, (out_dir, _) in zip(sets, recs, classes, hist, written):
        assert_jobdist(cl, hs, reference_jobdist(*csv_jobs(os.path.join(out_dir, "job.csv"), table), bounds, edges), fl.schedule)
        check_against_summary(cl, hs, rec, fl.schedule)


def test_sweep_bootstrap_jobdist_equals_the_ordinary_path(tmp_path):
    from gpuschedule_b200 import capi, summary, sweep, tracegen
    trace = tracegen.write_trace(str(tmp_path / "t.csv"), 500, seed=8)
    sets = [sweep.make_flags(trace_file=trace, schedule=sc, num_switch=1, num_node_p_switch=8, num_queue=2) for sc in ("fifo", "dlas-gpu")]
    R, loads, bounds, edges = 6, (1.0, 1.5), (2, 4), (10, 100, 1000, 10000)
    recs, (classes, hist) = sweep.summarize_bootstrap(sets, R, loads, seed=2, jobdist=(bounds, edges))
    assert classes.shape == (2, 2, R, 3) and hist.shape == (2, 2, R, 3, 3, 5)
    for c, (fl, infra, jm, pol) in enumerate(sweep._plain_setup(sets)):
        for li, L in enumerate(loads):
            num, den = sweep.load_gap_scale(L)
            tables = [tracegen.bootstrap_table(jm.table, 2, r, jm.table.n, num, den) for r in range(R)]
            with capi.Engine(device=0, nsims=R) as eng:
                for r in range(R):
                    eng.config(r, infra.gs_cluster(), pol)
                    eng.load_trace(r, tables[r])
                eng.set_jobdist(bounds, edges)
                want = eng.run_summarized()
                wc, wh = eng.jobdist()
                jobs = [job_columns(tables[r], *eng.fetch_jobs(r)) for r in range(R)]
            assert want.tobytes() == recs[c, li].tobytes()
            assert wc.tobytes() == classes[c, li].tobytes() and wh.tobytes() == hist[c, li].tobytes(), (fl.schedule, L)
            for r in range(R):
                assert_jobdist(wc[r], wh[r], reference_jobdist(*jobs[r], bounds, edges), (fl.schedule, L, r))
            sp = summary.jobdist_spread(classes[c, li], hist[c, li], edges)
            ref = summary.jobdist_spread(wc, wh, edges)
            for m in ("wait_cdf", "jct_cdf", "jct_mean"):
                for s in summary.SPREAD_STATS:
                    np.testing.assert_array_equal(sp[m][s], ref[m][s])


def test_sweep_command_line_writes_the_jobdist_csv(tmp_path):
    from gpuschedule_b200 import summary, sweep
    trace, _ = _sweep_flags(tmp_path)
    out, jd, cdf = tmp_path / "out.csv", tmp_path / "jd.csv", tmp_path / "cdf.csv"
    env = {**os.environ, "PYTHONPATH": REPO}
    subprocess.run([sys.executable, "-m", "gpuschedule_b200.sweep", "--trace", trace, "--schedule", "fifo", "horus",
                    "--num_switch", "1", "--num_node_p_switch", "8", "--seed", "3", "--summary", str(out),
                    "--jobdist", str(jd), "--gpu-classes", "2", "4", "--jobdist-cdf", str(cdf)], check=True, cwd=str(tmp_path), env=env)
    with open(jd, newline="") as f:
        lines = list(csv.reader(f))
    assert lines[0] == sweep.SUMMARY_KEYS + ["class", "gpus_min", "gpus_max"] + summary.jobdist_columns()
    assert len(lines) == 1 + 2 * 3
    assert [ln[6:9] for ln in lines[1:4]] == [["0", "0", "1"], ["1", "2", "3"], ["2", "4", "inf"]]
    with open(out, newline="") as f:
        srows = list(csv.reader(f))
    fin = srows[0].index("finished")
    assert sum(int(ln[9]) for ln in lines[1:4]) == int(srows[1][fin])
    with open(cdf, newline="") as f:
        clines = list(csv.reader(f))
    assert clines[0] == sweep.SUMMARY_KEYS + ["class", "gpus_min", "gpus_max", "quantity", "edge", "jobs", "cdf"]
    assert len(clines) == 1 + 2 * 3 * 3 * 31 and clines[-1][10] == str(2 ** 30)
    ci, cci, bout = tmp_path / "ci.csv", tmp_path / "cci.csv", tmp_path / "b.csv"
    subprocess.run([sys.executable, "-m", "gpuschedule_b200.sweep", "--trace", trace, "--schedule", "fifo", "sjf",
                    "--num_switch", "1", "--num_node_p_switch", "8", "--bootstrap", "3", "--load", "1", "2", "--summary", str(bout),
                    "--jobdist", str(ci), "--cdf-edges", "10", "100", "--jobdist-cdf", str(cci)], check=True, cwd=str(tmp_path), env=env)
    with open(ci, newline="") as f:
        lines = list(csv.reader(f))
    assert lines[0] == sweep.SUMMARY_KEYS + ["load", "class", "gpus_min", "gpus_max", "replicas", "level"] + summary.jobdist_spread_columns()
    assert len(lines) == 1 + 2 * 2 and int(lines[1][10]) == 3
    with open(cci, newline="") as f:
        clines = list(csv.reader(f))
    assert len(clines) == 1 + 2 * 2 * 3 * 2
    assert all(0.0 <= float(ln[-4]) <= 1.0 for ln in clines[1:])

"""Job statistics by a chosen key with bounded slowdown on the device (gs_set_slowdown / gs_fetch_slowdown,
gs_horus_set_slowdown / gs_horus_fetch_slowdown) on the H100.

Device records and CDF counts must equal test_slowdown_cpu.reference_slowdown over the job records and finish orders
the engine itself hands out (and, for the fixtures, the reference-made job.csv or the policy oracles' records).  With
key = gpus and jobdist's bounds and edges, every record's gs_jclass part and its three histogram rows equal
gs_fetch_jobdist's; the classes add up to the summary's job part; with the feature off nothing changes."""
import csv
import os
import subprocess
import sys
import types

import numpy as np
import pytest

from conftest import GOLDEN, REPO, golden_cases, horus_cases, load_golden, load_horus
from test_gpu_summary import _engine_run, _fifo_handle, _sweep_flags, _synth
from test_jobdist_cpu import DEFAULT_EDGES, csv_jobs
from test_slowdown_cpu import DEFAULT_SD_EDGES, assert_slowdown, reference_slowdown
from test_summary_cpu import _policy_cases, job_columns, load_policy

pytestmark = pytest.mark.gpu

SETTINGS = (("length", (), 1, (), ()), ("length", (60, 720, 2880), 1, DEFAULT_EDGES, DEFAULT_SD_EDGES),
            ("gpus", (5, 17, 65), 30, DEFAULT_EDGES, tuple(range(1024, 1024 * 256, 1024))),
            ("gpu-time", (10, 100, 1000, 10 ** 4, 10 ** 5, 10 ** 6, 2 ** 31), 1, tuple(range(0, 255 * 40, 40)), (1024, 4096)),
            ("length", (2, 50), 10 ** 9, (3, 100), (1023, 1024, 1025)))
JOB_FIELDS = ("wait_sum", "turnaround_sum", "jct_sum", "preempt_sum", "gpu_ticks_sum")


def check_against_summary(recs, hist, rec, tag=""):
    """class counts and sums add up to the summary's; every histogram row sums to its class's jobs"""
    jc = recs["jc"]
    assert int(jc["jobs"].sum()) == int(rec["finished"]), tag
    for f in JOB_FIELDS:
        assert int(jc[f].sum()) == int(rec[f]), (tag, f)
    n = jc["jobs"].astype(np.int64)
    assert (hist.astype(np.int64).sum(axis=-1) == 4 * n).all(), tag
    if len(recs) == 1:
        for f in ("wait_q", "turnaround_q", "jct_q"):
            assert jc[0][f].tolist() == rec[f].tolist(), (tag, f)


def _trace_cols(packed):
    """arrive_tick / gpus of a replica's own trace (JOBIN_DTYPE records), as job_columns reads them from a table"""
    return types.SimpleNamespace(arrive_tick=packed["arrive_tick"].astype(np.int64), gpus=packed["gpus"].astype(np.int64))


def _run(eng, sd, rows_cap=0):
    eng.set_slowdown(*sd)
    out, _, _ = _engine_run(eng, rows_cap)
    return out, eng.slowdown()


@pytest.mark.parametrize("case", golden_cases())
def test_fifo_fixture_slowdown_on_device(case):
    from gpuschedule_b200 import capi
    table, cluster, _, _, _ = load_golden(case)
    want_jobs = csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table)
    with capi.Engine(device=0, nsims=1) as eng:
        eng.config(0, cluster)
        eng.load_trace(0, table)
        eng.set_jobdist((5, 17, 65), DEFAULT_EDGES)
        out, _ = _run(eng, SETTINGS[0])
        recs_j, order = eng.fetch_jobs(0)
        cls, jh = eng.jobdist()
        for sd in SETTINGS + (("gpus", (5, 17, 65), 1, DEFAULT_EDGES, DEFAULT_SD_EDGES),):
            eng.set_slowdown(*sd)
            assert eng.summarize().tobytes() == out.tobytes()
            recs, hist = eng.slowdown()
            tag = f"{case} {sd[0]} bounds={sd[1]} tau={sd[2]}"
            assert_slowdown(recs[0], hist[0], reference_slowdown(*want_jobs, *sd), tag)
            assert_slowdown(recs[0], hist[0], reference_slowdown(*job_columns(table, recs_j, order), *sd), tag)
            check_against_summary(recs[0], hist[0], out[0], tag)
            if sd[0] == "gpus" and sd[1] == (5, 17, 65) and sd[3] == DEFAULT_EDGES:    # jobdist's classes and edges
                ne = len(DEFAULT_EDGES) + 1
                assert recs[0]["jc"].tobytes() == cls[0].tobytes()
                assert hist[0][:, :3 * ne].tobytes() == jh[0].reshape(len(cls[0]), 3 * ne).tobytes()


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("case", _policy_cases())
def test_policy_fixture_slowdown_on_device(case, mode):
    import oracle
    from gpuschedule_b200 import capi
    table, cluster, pol = load_policy(case)
    res = oracle.run_policy(cluster, pol, table)
    want_jobs = job_columns(table, res.recs, res.finish_order)
    with capi.Engine(device=0, nsims=1) as eng:
        eng.set_engine(mode)
        eng.config(0, cluster, pol)
        eng.load_trace(0, table)
        out, _ = _run(eng, SETTINGS[1])
        recs_j, order = eng.fetch_jobs(0)
        for sd in SETTINGS:
            eng.set_slowdown(*sd)
            eng.summarize()
            recs, hist = eng.slowdown()
            tag = f"{case} mode={mode} {sd[0]} tau={sd[2]}"
            assert_slowdown(recs[0], hist[0], reference_slowdown(*want_jobs, *sd), tag)
            assert_slowdown(recs[0], hist[0], reference_slowdown(*job_columns(table, recs_j, order), *sd), tag)
            check_against_summary(recs[0], hist[0], out[0], tag)


def test_horus_fixtures_slowdown_on_device():
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
        for sd in SETTINGS:
            eng.set_slowdown(*sd)
            n0 = eng.lib.gs_horus_launch_count(eng.h)
            out = eng.summarize()
            assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 3
            assert out.tobytes() == plain.tobytes()
            recs, hist = eng.slowdown()
            for i, (case, (table, _, _, _, _)) in enumerate(zip(cases, loaded)):
                _, _, _, hrecs, order = eng.fetch(i)
                tag = f"{case} {sd[0]} tau={sd[2]}"
                assert_slowdown(recs[i], hist[i], reference_slowdown(*job_columns(table, hrecs, order), *sd), tag)
                assert_slowdown(recs[i], hist[i], reference_slowdown(*csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table), *sd), tag)
                check_against_summary(recs[i], hist[i], out[i], tag)
        eng.set_slowdown(None)
        n0 = eng.lib.gs_horus_launch_count(eng.h)
        assert eng.summarize().tobytes() == plain.tobytes()
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
    sd = ("length", (2, 10, 60, 300, 720, 2880, 10 ** 5), 5, tuple(range(-3, 255 * 97 - 3, 97)), DEFAULT_SD_EDGES)
    with capi.Engine(device=0, nsims=len(configs)) as eng:
        for i, (cl, table, pol) in enumerate(configs):
            eng.config(i, cl, pol)
            eng.load_trace(i, table)
        out, (recs, hist) = _run(eng, sd, rows_cap=3000)
        part = eng.slowdown(first=40, count=7)
        assert part[0].tobytes() == recs[40:47].tobytes() and part[1].tobytes() == hist[40:47].tobytes()
        jobs = [job_columns(configs[i][1], *eng.fetch_jobs(i)) for i in range(len(configs))]
    for i in range(len(configs)):
        assert_slowdown(recs[i], hist[i], reference_slowdown(*jobs[i], *sd), f"replica {i}")
        check_against_summary(recs[i], hist[i], out[i], f"replica {i}")


def test_multi_window_slowdown_follows_the_finished_jobs():
    from gpuschedule_b200 import capi
    sd = ("length", (60, 720, 2880), 1, DEFAULT_EDGES, DEFAULT_SD_EDGES)
    for table, pol in ((_synth(100000, 3), None), (_synth(20000, 4), capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,)))):
        with capi.Engine(device=0, nsims=1) as eng:
            eng.config(0, capi.make_cluster(4, 32, 8), pol)
            eng.load_trace(0, table)
            _, (whole_r, whole_h) = _run(eng, sd)
            eng.reset()
            seen = []
            while True:
                eng.run(0, 7000)
                s = eng.summarize()
                r, h = eng.slowdown()
                seen.append((int(s[0]["finished"]), r[0].copy(), h[0].copy()))
                if s[0]["done"]:
                    break
            recs, order = eng.fetch_jobs(0)
        assert len(seen) >= 3
        for k, r, h in seen:
            assert_slowdown(r, h, reference_slowdown(*job_columns(table, recs, order[:k]), *sd), f"finished={k}")
        assert seen[-1][1].tobytes() == whole_r[0].tobytes() and seen[-1][2].tobytes() == whole_h[0].tobytes()


@pytest.mark.parametrize("kind", ["iid", "blocked", "mixed"])
def test_bootstrap_replicas(kind):
    from gpuschedule_b200 import capi, tracegen
    base = _synth(4000, 21)
    R = 12
    sd = ("gpu-time", (100, 10 ** 4, 10 ** 6), 60, DEFAULT_EDGES, DEFAULT_SD_EDGES)
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, capi.make_cluster(2, 16, 8), None if i % 2 else capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,)))
        eng.boot_population(base)
        params = np.zeros(R, dtype=capi.BOOT_PARAMS_DTYPE)
        params["seed"], params["stream"], params["n"], params["gap_num"], params["gap_den"] = 7, np.arange(R), 4000, 5, 6
        if kind == "mixed":
            eng.boot_mixes(np.stack([tracegen.class_weights(base.gpus, (4,), (1, 5)), tracegen.class_weights(base.gpus, (4,), (3, 1))]))
            eng.boot_traces(params, block_len=8, mix=np.arange(R) % 3 - 1)
        else:
            eng.boot_traces(params, block_len=None if kind == "iid" else 16)
        eng.set_slowdown(*sd)
        out = eng.run_summarized()
        recs, hist = eng.slowdown()
        for r in range(R):
            jobs = job_columns(_trace_cols(eng.fetch_trace(r)), *eng.fetch_jobs(r))
            assert_slowdown(recs[r], hist[r], reference_slowdown(*jobs, *sd), f"{kind} replica {r}")
            check_against_summary(recs[r], hist[r], out[r], f"{kind} replica {r}")
        params["stream"] = params["stream"][::-1]                   # regenerated replicas must be summarised again
        eng.boot_traces(params)
        with pytest.raises(capi.GsError) as e:
            eng.slowdown()
        assert e.value.code == capi.GS_ERR_STATE


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
            eng.set_slowdown(*SETTINGS[1])
            if mode == "off":
                eng.set_slowdown(None)
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
            a = eng.slowdown()
            s = eng.summarize()
            b = eng.slowdown()
            assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
            eng.reset()
            assert eng.run_summarized(rows_cap=3000).tobytes() == s.tobytes()
            c = eng.slowdown()
            assert a[0].tobytes() == c[0].tobytes() and a[1].tobytes() == c[1].tobytes()
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
        for bounds, tau, edges, sd_edges in (((0,), 1, (), ()), ((3, 3), 1, (), ()), ((), 0, (), ()), ((), 1, (2, 2), ()), ((), 1, (), (5, 1)),
                                             ((), 1, tuple(range(256)), ()), ((), 1, (), tuple(range(256)))):
            assert code(eng.set_slowdown, "length", bounds, tau, edges, sd_edges) == capi.GS_ERR_ARG
        assert code(eng.slowdown) == capi.GS_ERR_STATE                      # off
        eng.set_slowdown("length", (60,), 1, (10,), (2048,))
        assert code(eng.slowdown) == capi.GS_ERR_STATE                      # nothing has run
        eng.run(0, 5000)
        assert code(eng.slowdown) == capi.GS_ERR_STATE                      # not summarised
        eng.summarize()
        r1, h1 = eng.slowdown()
        for first, count in ((-1, 1), (0, 3), (2, 1)):
            assert code(eng.slowdown, first, count) == capi.GS_ERR_ARG
        eng.set_slowdown("gpus", (2, 4), 1, (5,), ())
        assert code(eng.slowdown) == capi.GS_ERR_STATE
        eng.summarize()
        assert eng.slowdown()[1].shape == (2, 3, 3 * 2 + 1)
        eng.set_slowdown("length", (60,), 1, (10,), (2048,))
        eng.summarize()
        r3, h3 = eng.slowdown()
        assert r3.tobytes() == r1.tobytes() and h3.tobytes() == h1.tobytes()
        eng.reset()
        assert code(eng.slowdown) == capi.GS_ERR_STATE
    finally:
        eng.close()


# ---------------------------------------------------------------- sweep
def test_sweep_slowdown_equals_the_files_run_batched_writes(tmp_path):
    from gpuschedule_b200 import ingest, sweep
    trace, sets = _sweep_flags(tmp_path)
    sd = sweep.check_slowdown(("length", (60, 720), 10, (1, 10, 100, 1000), DEFAULT_SD_EDGES))
    recs, (srec, shist) = sweep.summarize_batched(sets, slowdown=sd)
    recs2, (cls, jh), (srec2, shist2) = sweep.summarize_batched(sets, jobdist=((2, 4), (1, 10)), slowdown=sd)
    assert recs2.tobytes() == recs.tobytes() and srec2.tobytes() == srec.tobytes() and shist2.tobytes() == shist.tobytes()
    written = sweep.run_batched(sets, out_root=str(tmp_path / "log"))
    table = ingest.JobTraceReader(trace).prepare_jobs().table(0.5)
    for fl, rec, rc, hs, (out_dir, _) in zip(sets, recs, srec, shist, written):
        assert_slowdown(rc, hs, reference_slowdown(*csv_jobs(os.path.join(out_dir, "job.csv"), table), *sd), fl.schedule)
        check_against_summary(rc, hs, rec, fl.schedule)


def test_sweep_command_line_writes_the_slowdown_csv(tmp_path):
    from gpuschedule_b200 import summary, sweep
    trace, _ = _sweep_flags(tmp_path)
    out, sdf, cdf = tmp_path / "out.csv", tmp_path / "sd.csv", tmp_path / "cdf.csv"
    out0 = tmp_path / "out0.csv"
    env = {**os.environ, "PYTHONPATH": REPO}
    common = [sys.executable, "-m", "gpuschedule_b200.sweep", "--trace", trace, "--schedule", "fifo", "dlas-gpu", "horus",
              "--num_switch", "1", "--num_node_p_switch", "8", "--seed", "3"]
    subprocess.run(common + ["--summary", str(out0)], check=True, cwd=str(tmp_path), env=env)
    subprocess.run(common + ["--summary", str(out), "--slowdown", str(sdf), "--key-classes", "60", "720", "2880",
                             "--slowdown-cdf", str(cdf)], check=True, cwd=str(tmp_path), env=env)
    with open(out0, "rb") as f0, open(out, "rb") as f1:                   # the summary file does not change
        assert f0.read() == f1.read()
    with open(sdf, newline="") as f:
        lines = list(csv.reader(f))
    assert lines[0] == sweep.SUMMARY_KEYS + ["key", "class", "key_min", "key_max", "tau"] + summary.slowdown_columns()
    assert len(lines) == 1 + 3 * 4
    assert [ln[6:10] for ln in lines[1:5]] == [["length", "0", "0", "59"], ["length", "1", "60", "719"], ["length", "2", "720", "2879"],
                                               ["length", "3", "2880", "inf"]]
    with open(out, newline="") as f:
        srows = list(csv.reader(f))
    fin = srows[0].index("finished")
    for c in range(3):
        assert sum(int(ln[11]) for ln in lines[1 + 4 * c:5 + 4 * c]) == int(srows[1 + c][fin])
    with open(cdf, newline="") as f:
        clines = list(csv.reader(f))
    assert len(clines) == 1 + 3 * 4 * (3 * 31 + 21) and clines[-1][11] == "sd" and float(clines[-1][12]) == 2.0 ** 20
    ci, cci, bout = tmp_path / "ci.csv", tmp_path / "cci.csv", tmp_path / "b.csv"
    subprocess.run([sys.executable, "-m", "gpuschedule_b200.sweep", "--trace", trace, "--schedule", "fifo", "dlas-gpu",
                    "--num_switch", "1", "--num_node_p_switch", "8", "--bootstrap", "3", "--load", "1", "1.2", "--block-len", "4",
                    "--summary", str(bout), "--slowdown", str(ci), "--job-key", "gpu-time", "--key-classes", "100",
                    "--slowdown-bound", "60", "--cdf-edges", "10", "100", "--sd-edges", "1024", "4096", "--slowdown-cdf", str(cci)],
                   check=True, cwd=str(tmp_path), env=env)
    with open(ci, newline="") as f:
        lines = list(csv.reader(f))
    assert lines[0] == (sweep.SUMMARY_KEYS + ["load", "block_len", "key", "class", "key_min", "key_max", "tau", "replicas", "level"]
                        + summary.slowdown_spread_columns())
    assert len(lines) == 1 + 2 * 2 * 2 and lines[1][8] == "gpu-time" and lines[1][12] == "60"
    with open(cci, newline="") as f:
        clines = list(csv.reader(f))
    assert len(clines) == 1 + 2 * 2 * 2 * (3 * 2 + 2)
    assert all(0.0 <= float(ln[-4]) <= 1.0 for ln in clines[1:] if ln[-4] != "nan")

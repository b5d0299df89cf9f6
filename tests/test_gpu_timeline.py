"""Timelines (gs_set_timeline / gs_fetch_timeline, gs_horus_set_timeline / gs_horus_fetch_timeline) on the H100.

Device bins are checked against a pandas binning of the fixtures' reference-made cluster.csv (the columns it carries),
against the numpy binning of test_timeline_cpu.py over the rows the engine itself hands out (every field, the 128-bit
sums and finished_last included), and against the replica's own gs_summary (sums over bins, maxima, first / last delta)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import REPO, golden_cases, horus_cases, load_golden, load_horus
from test_gpu_summary import _engine_run, _fifo_handle, _sweep_flags, _synth
from test_summary_cpu import _policy_cases, load_policy, record_fields
from test_timeline_cpu import FLOAT_FIELDS, assert_bins, bin_fields, bin_of, reference_bins

pytestmark = pytest.mark.gpu

GRID = ((1, 1024), (3, 2), (64, 1024), (10 ** 7, 1))


def csv_bins(case_dir, W, B, horus=False):
    """per bin, the gs_tbin fields a run's cluster.csv carries, binned by its delta column (pandas, as a notebook)"""
    import pandas as pd
    cl = pd.read_csv(os.path.join(case_dir, "cluster.csv"))
    cl["bin"] = bin_of(cl["delta"].to_numpy(), W, B)
    avg = cl["avg_pending_time"].astype(float)
    if horus:
        cl["util"] = cl["avg_gpu_utilization"].astype(str).str.strip("[]").astype(float).fillna(0.0)
    out = []
    for b in range(B):
        g = cl[cl["bin"] == b]
        a = avg[cl["bin"] == b]
        d = dict(rows=len(g), pending_rows=int((a != 0).sum()), avg_pending_sum=math.fsum(a[a != 0].tolist()))
        for f, col in (("busy_gpus", "num_busy_gpus"), ("running", "num_running_jobs"), ("queued", "num_queuing_jobs")):
            d[f + "_sum"] = int(g[col].astype(np.int64).sum())
            d[f + "_max"] = int(g[col].max()) if len(g) else 0
        d["pend_max_max"] = int(g["max_pending_time"].astype(float).max()) if len(g) else 0
        d["delta_min"] = int(g["delta"].min()) if len(g) else 0
        d["delta_max"] = int(g["delta"].max()) if len(g) else 0
        if horus:
            d["util_sum"] = math.fsum(g["util"].tolist())
        out.append(d)
    return out


def assert_csv_bins(tl, want, tag=""):
    """bins against csv_bins: every field at 1e-12, except util_sum -- the bracketed values of avg_gpu_utilization are
    printed with 8 decimals (numpy's array format), so the CSV's sum is off by up to 5e-9 per row"""
    assert_bins(tl, want, tag, skip=("util_sum",))
    for b, (t, w) in enumerate(zip(tl, want)):
        if "util_sum" in w:
            assert abs(float(t["util_sum"]) - w["util_sum"]) <= 5e-9 * int(t["rows"]) + 1e-12 * abs(w["util_sum"]), (tag, b)


def check_against_summary(tl, rec, tag=""):
    """exact invariants of one replica's bins against its gs_summary"""
    f = record_fields(rec)
    bins = [bin_fields(t) for t in tl]
    for key in ("rows", "busy_gpus_sum", "running_sum", "queued_sum", "pend_sum_sum", "mem_busy_sum", "pending_rows"):
        assert sum(b[key] for b in bins) == f[key], (tag, key)
    for key in ("busy_gpus_max", "running_max", "queued_max", "pend_max_max"):
        assert max(b[key] for b in bins) == f[key], (tag, key)
    full = [b for b in bins if b["rows"] > 0]
    if f["rows"]:
        assert full[-1]["delta_max"] == f["makespan"], tag
    return full


def _run_with_timeline(eng, W, B, rows_cap=0):
    eng.set_timeline(W, B)
    out, rows, launches = _engine_run(eng, rows_cap)
    return out, rows, eng.timeline()


@pytest.mark.parametrize("case", golden_cases())
def test_fifo_fixture_timeline_on_device(case):
    from gpuschedule_b200 import capi
    table, cluster, _, _, _ = load_golden(case)
    d = os.path.join(REPO, "tests", "golden", case)
    for W, B in GRID:
        with capi.Engine(device=0, nsims=1) as eng:
            eng.config(0, cluster)
            eng.load_trace(0, table)
            out, rows, tl = _run_with_timeline(eng, W, B)
        tag = f"{case} W={W} B={B}"
        assert_csv_bins(tl[0], csv_bins(d, W, B), tag)
        assert_bins(tl[0], reference_bins(rows[0], W, B), tag)
        assert np.isnan(tl[0]["util_sum"]).all()
        full = check_against_summary(tl[0], out[0], tag)
        assert full[0]["delta_min"] == int(rows[0]["now"][0]), tag


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("case", _policy_cases())
def test_policy_fixture_timeline_on_device(case, mode):
    import oracle
    from gpuschedule_b200 import capi
    table, cluster, pol = load_policy(case)
    ref_rows = oracle.run_policy(cluster, pol, table).rows
    for W, B in GRID:
        with capi.Engine(device=0, nsims=1) as eng:
            eng.set_engine(mode)
            eng.config(0, cluster, pol)
            eng.load_trace(0, table)
            out, rows, tl = _run_with_timeline(eng, W, B)
        tag = f"{case} mode={mode} W={W} B={B}"
        assert_bins(tl[0], reference_bins(ref_rows, W, B), tag)
        assert_bins(tl[0], reference_bins(rows[0], W, B), tag)
        full = check_against_summary(tl[0], out[0], tag)
        assert full[0]["delta_min"] == int(rows[0]["now"][0]), tag


@pytest.mark.parametrize("case", horus_cases())
def test_horus_fixture_timeline_on_device(case):
    from gpuschedule_b200 import capi
    table, cluster, params, _, _ = load_horus(case)
    d = os.path.join(REPO, "tests", "golden", case)
    with capi.HorusEngine(device=0, nsims=1) as eng:
        eng.config(0, cluster, capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"]))
        eng.load_trace(0, table)
        np.random.seed(params["seed"])
        eng.load_words(0, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))
        eng.run(rows_cap=1 << 15)
        rows, util, _, _, _ = eng.fetch(0)
        for W, B in GRID:
            eng.set_timeline(W, B)
            n0 = eng.lib.gs_horus_launch_count(eng.h)
            out = eng.summarize()
            assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 3
            tl = eng.timeline()
            tag = f"{case} W={W} B={B}"
            assert_csv_bins(tl[0], csv_bins(d, W, B, horus=True), tag)
            assert_bins(tl[0], reference_bins(rows, W, B, util=util), tag)
            check_against_summary(tl[0], out[0], tag)
            assert math.isclose(math.fsum(tl[0]["util_sum"].tolist()), float(out[0]["util_sum"]), rel_tol=1e-12)
        eng.set_timeline(0, 0)
        n0 = eng.lib.gs_horus_launch_count(eng.h)
        eng.summarize()
        assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 2


def test_multi_window_timeline_equals_whole_run():
    from gpuschedule_b200 import capi, policies
    cases = [(_synth(100000, 3), None), (_synth(20000, 4), capi.make_policy("sjf")),
             (_synth(20000, 5), capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,)))]
    t = cases[1][0]
    cases.append((t, capi.make_policy("gittins", gittins_table=policies.build_gittins_table(policies.gittins_samples(t), 3250.0))))
    for table, pol in cases:
        with capi.Engine(device=0, nsims=1) as eng:
            eng.config(0, capi.make_cluster(4, 32, 8), pol)
            eng.load_trace(0, table)
            whole, rows1, tw = _run_with_timeline(eng, 500, 256)
            eng.reset()
            windows, rows, tm = _run_with_timeline(eng, 500, 256, rows_cap=7000)
        assert rows[0].tobytes() == rows1[0].tobytes()
        for a, b in zip(tw[0], tm[0]):
            fa, fb = bin_fields(a), bin_fields(b)
            for key in fa:
                if key in FLOAT_FIELDS:
                    assert (math.isnan(fa[key]) and math.isnan(fb[key])) or math.isclose(fa[key], fb[key], rel_tol=1e-12), key
                else:
                    assert fa[key] == fb[key], key
        assert_bins(tm[0], reference_bins(rows[0], 500, 256))
        check_against_summary(tm[0], windows[0])


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
    with capi.Engine(device=0, nsims=len(configs)) as eng:
        for i, (cl, table, pol) in enumerate(configs):
            eng.config(i, cl, pol)
            eng.load_trace(i, table)
        out, rows, tl = _run_with_timeline(eng, 37, 100, rows_cap=3000)
        assert eng.timeline(first=40, count=7).tobytes() == tl[40:47].tobytes()
    for i in range(len(configs)):
        assert_bins(tl[i], reference_bins(rows[i], 37, 100), f"replica {i}")
        check_against_summary(tl[i], out[i], f"replica {i}")


def test_reset_repeat_and_second_summarize_are_bit_identical():
    from gpuschedule_b200 import capi
    tables = [_synth(30000, 20 + i) for i in range(3)]
    eng = _fifo_handle(capi, tables, capi.make_cluster(4, 32, 8))
    try:
        eng.set_timeline(100, 512)
        a = eng.run_summarized(rows_cap=4000)
        ta = eng.timeline()
        assert eng.summarize().tobytes() == a.tobytes() and eng.timeline().tobytes() == ta.tobytes()
        eng.reset()
        b = eng.run_summarized(rows_cap=4000)
        assert b.tobytes() == a.tobytes() and eng.timeline().tobytes() == ta.tobytes()
    finally:
        eng.close()


def test_timeline_changes_no_other_output_and_no_launch_when_off():
    from gpuschedule_b200 import capi
    tables = [_synth(5000, 40 + i) for i in range(4)]
    cluster = capi.make_cluster(4, 32, 8)
    got, per_call = [], []
    for on in (False, True):
        eng = _fifo_handle(capi, tables, cluster)
        if on:
            eng.set_timeline(16, 64)
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
        eng.close()
        got.append(blobs)
        per_call.append(set(calls))
    assert len(got[0]) == len(got[1]) and all(a == b for a, b in zip(*got))
    assert per_call == [{2}, {3}]


def test_error_codes_and_restarts():
    from gpuschedule_b200 import capi
    table = _synth(20000, 9)
    eng = _fifo_handle(capi, [table, table], capi.make_cluster(4, 32, 8))
    try:
        for width, nbins in ((0, 4), (5, -1), (5, 1025), (2 ** 41, 4)):
            with pytest.raises(capi.GsError) as e:
                eng.set_timeline(width, nbins)
            assert e.value.code == capi.GS_ERR_ARG, (width, nbins)
        with pytest.raises(capi.GsError) as e:
            eng.timeline()
        assert e.value.code == capi.GS_ERR_STATE                      # off
        eng.set_timeline(50, 8)
        with pytest.raises(capi.GsError) as e:
            eng.timeline()
        assert e.value.code == capi.GS_ERR_STATE                      # nothing has run
        eng.run(0, 5000)
        with pytest.raises(capi.GsError) as e:
            eng.timeline()
        assert e.value.code == capi.GS_ERR_STATE                      # not summarised
        s1 = eng.summarize()
        t1 = eng.timeline()
        for first, count in ((-1, 1), (0, 3), (2, 1), (1, -1)):
            with pytest.raises(capi.GsError) as e:
                eng.timeline(first, count)
            assert e.value.code == capi.GS_ERR_ARG, (first, count)
        for width, nbins in ((50, 8), (10, 16), (1, 0)):
            with pytest.raises(capi.GsError) as e:
                eng.set_timeline(width, nbins)                        # rows have been folded
            assert e.value.code == capi.GS_ERR_STATE
        assert eng.timeline().tobytes() == t1.tobytes()               # and nothing changed
        eng.reset()                                                   # a reset replica starts from zero bins
        eng.set_timeline(50, 8)
        eng.run(0, 5000)
        assert eng.summarize().tobytes() == s1.tobytes() and eng.timeline().tobytes() == t1.tobytes()
        eng.reset()
        eng.set_timeline(0, 0)
        eng.run(0, 5000)
        assert eng.summarize().tobytes() == s1.tobytes()
        with pytest.raises(capi.GsError) as e:
            eng.timeline()
        assert e.value.code == capi.GS_ERR_STATE
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
        eng.set_timeline(20, 300)
        eng.boot_traces(params)
        eng.run_summarized()
        ta = eng.timeline()
        params["stream"] = [1, 0]
        eng.boot_traces(params)
        with pytest.raises(capi.GsError) as e:
            eng.timeline()
        assert e.value.code == capi.GS_ERR_STATE
        eng.run_summarized()
        tb = eng.timeline()
    assert tb[0].tobytes() == ta[1].tobytes() and tb[1].tobytes() == ta[0].tobytes()


# ---------------------------------------------------------------- sweep
def test_sweep_timeline_equals_the_files_run_batched_writes(tmp_path):
    import pandas as pd
    from gpuschedule_b200 import sweep
    trace, sets = _sweep_flags(tmp_path)
    W, B = 9, 40
    recs, bins = sweep.summarize_batched(sets, timeline=(W, B))
    written = sweep.run_batched(sets, out_root=str(tmp_path / "log"))
    for fl, tb, rec, (out_dir, _) in zip(sets, bins, recs, written):
        horus = fl.schedule in ("horus", "horus+", "gandiva")
        assert_csv_bins(tb, csv_bins(out_dir, W, B, horus=horus), fl.schedule)
        check_against_summary(tb, rec, fl.schedule)
        assert len(pd.read_csv(os.path.join(out_dir, "cluster.csv"))) == int(tb["rows"].sum())


def test_sweep_bootstrap_timeline_equals_the_ordinary_path(tmp_path):
    from gpuschedule_b200 import capi, sweep, tracegen
    trace = tracegen.write_trace(str(tmp_path / "t.csv"), 500, seed=8)
    sets = [sweep.make_flags(trace_file=trace, schedule=sc, num_switch=1, num_node_p_switch=8, num_queue=2) for sc in ("fifo", "sjf")]
    R, loads, W, B = 4, (1.0, 1.5), 25, 64
    recs, bins = sweep.summarize_bootstrap(sets, R, loads, seed=2, timeline=(W, B))
    assert bins.shape == (2, 2, R, B)
    for c, (fl, infra, jm, pol) in enumerate(sweep._plain_setup(sets)):
        for li, L in enumerate(loads):
            num, den = sweep.load_gap_scale(L)
            with capi.Engine(device=0, nsims=R) as eng:
                for r in range(R):
                    eng.config(r, infra.gs_cluster(), pol)
                    eng.load_trace(r, tracegen.bootstrap_table(jm.table, 2, r, jm.table.n, num, den))
                eng.set_timeline(W, B)
                want = eng.run_summarized()
                tw = eng.timeline()
            assert want.tobytes() == recs[c, li].tobytes()
            assert tw.tobytes() == bins[c, li].tobytes(), (fl.schedule, L)


def test_sweep_command_line_writes_the_timeline_csv(tmp_path):
    import csv
    from gpuschedule_b200 import summary, sweep
    trace, _ = _sweep_flags(tmp_path)
    out, tl = tmp_path / "out.csv", tmp_path / "tl.csv"
    env = {**os.environ, "PYTHONPATH": REPO}
    subprocess.run([sys.executable, "-m", "gpuschedule_b200.sweep", "--trace", trace, "--schedule", "fifo", "horus",
                    "--num_switch", "1", "--num_node_p_switch", "8", "--seed", "3", "--summary", str(out),
                    "--timeline", str(tl), "--bin-width", "10", "--bins", "16"], check=True, cwd=str(tmp_path), env=env)
    with open(tl, newline="") as f:
        lines = list(csv.reader(f))
    assert lines[0] == sweep.SUMMARY_KEYS + ["bin", "bin_start", "bin_end"] + summary.timeline_columns()
    assert len(lines) == 1 + 2 * 16
    assert [ln[6] for ln in lines[1:17]] == [str(b) for b in range(16)] and lines[16][8] == "inf"
    with open(out, newline="") as f:
        srows = list(csv.reader(f))
    assert sum(int(ln[11]) for ln in lines[1:17]) == int(srows[1][7])          # rows over bins = the summary's rows
    ci, bout = tmp_path / "ci.csv", tmp_path / "b.csv"
    subprocess.run([sys.executable, "-m", "gpuschedule_b200.sweep", "--trace", trace, "--schedule", "fifo", "sjf",
                    "--num_switch", "1", "--num_node_p_switch", "8", "--bootstrap", "3", "--load", "1", "2", "--summary", str(bout),
                    "--timeline", str(ci), "--bin-width", "50"], check=True, cwd=str(tmp_path), env=env)
    with open(ci, newline="") as f:
        lines = list(csv.reader(f))
    assert lines[0] == sweep.SUMMARY_KEYS + ["load", "bin", "bin_start", "bin_end", "replicas", "level"] + summary.timeline_spread_columns()
    assert len(lines) == 1 + 2 * 2 * 128
    assert int(lines[1][10]) == 3
    assert not os.path.exists(tmp_path / "log")

"""Time-weighted occupancy on the device (gs_set_occupancy / gs_fetch_occupancy and the horus twins) on the H100.

Device records and histograms must equal test_occupancy_cpu.reference over the rows the engine itself hands out, for
fifo (every row one tick), the event-driven policies (rows weighed by the step of `delta`, the last row of an
unfinished window carried to the next summarize) and horus.  The invariants: the histograms add up to the redundant
fields, fifo and horus weigh every summarised row once, and fifo's queued_sum is the Little's-law sum of the queued
jobs' waits.  With the feature off, launches and summaries are those of the parent; with it on, nothing else changes."""
import csv

import numpy as np
import pytest

from conftest import golden_cases, horus_cases, load_golden, load_horus
from test_gpu_summary import _engine_run, _synth
from test_occupancy_cpu import EDGES, _gpus, assert_occ, reference
from test_summary_cpu import _policy_cases, load_policy

pytestmark = pytest.mark.gpu


def _occ_run(eng, rows_cap=0, edges=EDGES):
    eng.set_occupancy(edges)
    out, rows, _ = _engine_run(eng, rows_cap)
    return out, rows, eng.occupancy()


def _little(table, starts, ticks):
    """fifo: a job is queued on the rows arrive + 1 .. start (never started: .. ticks), so queued_sum is this sum"""
    a = np.asarray(table.arrive_tick, dtype=np.int64)[:len(starts)]
    st = np.asarray(starts, dtype=np.int64)
    return int(np.maximum(0, np.where(st >= 0, np.minimum(st, ticks), ticks) - a).sum())


@pytest.mark.parametrize("case", golden_cases())
def test_fifo_fixture_occupancy(case):
    from gpuschedule_b200 import capi
    table, cluster, _, _, _ = load_golden(case)
    G = _gpus(cluster)
    with capi.Engine(device=0, nsims=1) as eng:
        eng.config(0, cluster)
        eng.load_trace(0, table)
        plain, _, _ = _engine_run(eng)
        n0 = eng.lib.gs_launch_count(eng.h)
        eng.summarize()
        n_off = eng.lib.gs_launch_count(eng.h) - n0
        eng.reset()
        out, rows, (rec, busy, queue) = _occ_run(eng)
        n0 = eng.lib.gs_launch_count(eng.h)
        again = eng.summarize()
        assert eng.lib.gs_launch_count(eng.h) - n0 == n_off + 1
        rec2, busy2, queue2 = eng.occupancy()
        recs, _ = eng.fetch_jobs(0)
    assert out.tobytes() == plain.tobytes() and again.tobytes() == plain.tobytes()
    assert rec.tobytes() == rec2.tobytes() and busy.tobytes() == busy2.tobytes() and queue.tobytes() == queue2.tobytes()
    assert_occ(rec[0], busy[0], queue[0], reference(rows[0], G, EDGES, True, per_tick=True), case)
    assert int(rec[0]["ticks"]) == int(out[0]["rows"]) and int(rec[0]["busy_sum"]) == int(out[0]["busy_gpus_sum"])
    assert int(rec[0]["queued_sum"]) == int(out[0]["queued_sum"]) == _little(table, recs["start"], int(out[0]["makespan"]))
    if int(out[0]["finished"]) == table.n:
        assert int(rec[0]["queued_sum"]) == int(out[0]["wait_sum"])


@pytest.mark.parametrize("case", _policy_cases())
def test_policy_fixture_occupancy(case):
    from gpuschedule_b200 import capi
    table, cluster, pol = load_policy(case)
    G = _gpus(cluster)
    with capi.Engine(device=0, nsims=1) as eng:
        eng.config(0, cluster, pol)
        eng.load_trace(0, table)
        out, rows, (rec, busy, queue) = _occ_run(eng)
        eng.reset()
        out_w, rows_w, (rec_w, busy_w, queue_w) = _occ_run(eng, rows_cap=max(16, len(rows[0]) // 5))
    assert rows_w[0].tobytes() == rows[0].tobytes()
    assert_occ(rec[0], busy[0], queue[0], reference(rows[0], G, EDGES, True), case)
    assert rec_w.tobytes() == rec.tobytes() and busy_w.tobytes() == busy.tobytes() and queue_w.tobytes() == queue.tobytes()
    assert int(rec[0]["rows"]) == int(out[0]["rows"])


def test_multi_window_runs_carry_the_last_row():
    """after every window the record equals the restatement over the rows so far, the last one not weighed yet"""
    from gpuschedule_b200 import capi
    for table, pol in ((_synth(60000, 3), None), (_synth(20000, 4), capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,))),
                       (_synth(20000, 5), capi.make_policy("dlas", num_queue=3, queue_limit=(600, 3600)))):
        cluster = capi.make_cluster(4, 32, 8)
        with capi.Engine(device=0, nsims=1) as eng:
            eng.config(0, cluster, pol)
            eng.load_trace(0, table)
            _, _, whole = _occ_run(eng)
            eng.reset()
            eng.set_occupancy(EDGES)
            parts, n = [], 0
            while True:
                eng.run(0, 7000)
                s = eng.summarize()
                w = eng.window(0)
                if w.ticks > w.row_first:
                    parts.append(eng.fetch_rows(0, w.row_first, w.ticks - w.row_first))
                rec, busy, queue = eng.occupancy()
                rows = np.concatenate(parts)
                assert_occ(rec[0], busy[0], queue[0], reference(rows, 1024, EDGES, bool(s[0]["done"]), per_tick=pol is None), f"window {n}")
                n += 1
                if s[0]["done"]:
                    break
        assert n >= 3
        assert rec.tobytes() == whole[0].tobytes() and busy.tobytes() == whole[1].tobytes()


@pytest.mark.parametrize("kind", ["iid", "blocked", "mixed"])
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
        else:
            eng.boot_traces(params, block_len=None if kind == "iid" else 16)
        out, rows, (rec, busy, queue) = _occ_run(eng, rows_cap=3000)
        for i in range(R):
            assert_occ(rec[i], busy[i], queue[i], reference(rows[i], 256, EDGES, True, per_tick=i % 2 == 1), f"{kind} replica {i}")
        eng.boot_traces(params)                        # new traces: every replica starts again
        with pytest.raises(capi.GsError) as e:
            eng.occupancy()
        assert e.value.code == capi.GS_ERR_STATE


def test_heterogeneous_handle_pitch_and_both_histogram_paths():
    """clusters of 64 to 4096 GPUs in one handle: the small ones count in shared memory, 2 * (G + 1) > 3072 in global"""
    from gpuschedule_b200 import capi
    configs = []
    for i in range(40):
        shape = ((2, 4, 8), (4, 32, 8), (4, 64, 8), (8, 64, 8), (1, 4, 16))[i % 5]
        sched = ("sjf", "dlas-gpu", "dlas")[i % 3]
        pol = None if i % 2 == 0 else capi.make_policy(sched, **({} if sched == "sjf" else dict(num_queue=2, queue_limit=(3600,))))
        configs.append((capi.make_cluster(*shape), _synth(500 + 13 * i, 300 + i), pol))
    gs = [_gpus(c) for c, _, _ in configs]
    assert min(2 * (g + 1) for g in gs) <= 3072 < max(2 * (g + 1) for g in gs)
    with capi.Engine(device=0, nsims=len(configs)) as eng:
        for i, (cl, table, pol) in enumerate(configs):
            eng.config(i, cl, pol)
            eng.load_trace(i, table)
        out, rows, (rec, busy, queue) = _occ_run(eng, rows_cap=2000, edges=tuple(range(0, 255 * 3, 3)))
        part = eng.occupancy(first=7, count=3)
        assert part[0].tobytes() == rec[7:10].tobytes() and part[2].tobytes() == queue[7:10].tobytes()
        assert np.array_equal(part[1], busy[7:10, :, :part[1].shape[2]])
    assert busy.shape[2] == max(gs) + 1
    for i in range(len(configs)):
        assert_occ(rec[i], busy[i], queue[i], reference(rows[i], gs[i], tuple(range(0, 255 * 3, 3)), True, per_tick=configs[i][2] is None),
                   f"replica {i}")


def test_horus_family():
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
        eng.set_timeline(50, 64)
        eng.set_jobdist((5, 17), (10, 100, 1000))
        eng.summarize()
        tl, jd = eng.timeline(), eng.jobdist()
        eng.set_occupancy(EDGES)
        n0 = eng.lib.gs_horus_launch_count(eng.h)
        out = eng.summarize()
        assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 5
        assert out.tobytes() == plain.tobytes()
        assert eng.timeline().tobytes() == tl.tobytes() and eng.jobdist()[0].tobytes() == jd[0].tobytes()
        rec, busy, queue = eng.occupancy()
        again = eng.summarize(), eng.occupancy()
        assert again[1][0].tobytes() == rec.tobytes() and again[1][1].tobytes() == busy.tobytes()
        schemes = set()
        for i, (case, (_, cluster, params, _, _)) in enumerate(zip(cases, loaded)):
            rows = eng.fetch(i)[0]
            assert_occ(rec[i], busy[i], queue[i], reference(rows, _gpus(cluster), EDGES, True, per_tick=True), case)
            assert int(rec[i]["ticks"]) == int(out[i]["rows"]) and int(rec[i]["busy_sum"]) == int(out[i]["busy_gpus_sum"])
            schemes.add(params["scheme"])
        assert {"horus", "horus+", "gandiva"} <= schemes
        eng.set_occupancy(None)
        n0 = eng.lib.gs_horus_launch_count(eng.h)
        assert eng.summarize().tobytes() == plain.tobytes()
        assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 4


def test_other_outputs_unchanged_and_error_codes():
    from gpuschedule_b200 import capi
    tables = [_synth(3000, 60 + i) for i in range(3)]
    pols = (None, capi.make_policy("sjf"), capi.make_policy("dlas-gpu", num_queue=2, queue_limit=(3600,)))
    got = []
    for on in (False, True):
        with capi.Engine(device=0, nsims=3) as eng:
            for i in range(3):
                eng.config(i, capi.make_cluster(2, 16, 8), pols[i])
                eng.load_trace(i, tables[i])
            eng.set_timeline(100, 32)
            eng.set_jobdist((5, 17), (10, 100, 1000))
            eng.set_slowdown("length", (60, 720), 1, (10, 100), (2048,))
            if on:
                eng.set_occupancy(EDGES)
            out, _, _ = _engine_run(eng, rows_cap=1500)
            got.append((out.tobytes(), eng.timeline().tobytes(), eng.jobdist()[1].tobytes(), eng.slowdown()[0].tobytes()))
            if on:
                with pytest.raises(capi.GsError) as e:
                    eng.set_occupancy(EDGES)                       # rows already folded
                assert e.value.code == capi.GS_ERR_STATE
                busy = np.zeros((3, 2, 256), dtype=np.uint64)
                assert eng.lib.gs_fetch_occupancy(eng.h, 0, 3, None, busy.ctypes.data_as(np.ctypeslib.ctypes.c_void_p), 256, None) == capi.GS_ERR_CAPACITY
                assert eng.lib.gs_fetch_occupancy(eng.h, 2, 2, None, None, 0, None) == capi.GS_ERR_ARG
                eng.reset()
                for bad in ([3, 3], [-2], list(range(256))):
                    with pytest.raises(capi.GsError) as e:
                        eng.set_occupancy(bad)
                    assert e.value.code == capi.GS_ERR_ARG
                with pytest.raises(capi.GsError) as e:
                    eng.occupancy()                                # reset: not summarised since
                assert e.value.code == capi.GS_ERR_STATE
                eng.set_occupancy(None)
                with pytest.raises(capi.GsError) as e:
                    eng.occupancy()
                assert e.value.code == capi.GS_ERR_STATE
    assert got[0] == got[1]
    with capi.Engine(device=0, nsims=1) as eng:                    # more GPUs than 65535
        eng.config(0, capi.make_cluster(66, 128, 8), capi.make_policy("sjf"))
        eng.load_trace(0, _synth(50, 9))
        eng.set_occupancy(EDGES)
        eng.run(0, 0)
        with pytest.raises(capi.GsError) as e:
            eng.summarize()
        assert e.value.code == capi.GS_ERR_ARG
        eng.set_occupancy(None)
        eng.summarize()


def test_sweep_files(tmp_path, monkeypatch):
    from gpuschedule_b200 import summary, sweep, tracegen
    monkeypatch.chdir(tmp_path)
    trace = tracegen.write_trace(str(tmp_path / "t.csv"), 400, seed=5)
    base = ["--trace", trace, "--schedule", "fifo", "sjf", "horus", "--num_switch", "1", "--num_node_p_switch", "8"]
    sweep.main(base + ["--summary", str(tmp_path / "s.csv"), "--occupancy", str(tmp_path / "o.csv"), "--occupancy-cdf", str(tmp_path / "c.csv"),
                       "--queue-edges", "0", "1", "5"])
    with open(tmp_path / "o.csv") as f:
        lines = list(csv.DictReader(f))
    assert len(lines) == 3
    for ln in lines:
        assert 0 <= float(ln["gpu_share"]) <= 1 and int(ln["ticks"]) > 0
    with open(tmp_path / "c.csv") as f:
        cdf = list(csv.DictReader(f))
    assert len(cdf) == 3 * (2 * 65 + 3)
    boot_args = ["--trace", trace, "--schedule", "fifo", "sjf", "--num_switch", "1", "--num_node_p_switch", "8"]
    sweep.main(boot_args + ["--summary", str(tmp_path / "b.csv"), "--bootstrap", "4", "--load", "1", "1.5", "--occupancy", str(tmp_path / "ob.csv"),
                       "--occupancy-cdf", str(tmp_path / "cb.csv")])
    with open(tmp_path / "ob.csv") as f:
        boot = list(csv.DictReader(f))
    assert len(boot) == 4 and all(int(b["replicas"]) == 4 for b in boot)
    assert all(k in boot[0] for k in summary.occupancy_spread_columns())
    sweep.main(base + ["--summary", str(tmp_path / "s2.csv")])
    with open(tmp_path / "s.csv") as f, open(tmp_path / "s2.csv") as g:
        a, b = f.read().splitlines(), g.read().splitlines()
    assert a[:3] == b[:3]              # header, fifo and sjf (the horus line's sampled utilisation is drawn anew)

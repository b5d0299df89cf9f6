"""Interference statistics of the utilisation-aware engine on the device (gs_horus_set_interference /
gs_horus_fetch_interference, gs_if_jobs_kernel) on the H100.

Device records must equal test_interference_cpu.reference_interference over the job records and finish orders the
engine itself hands out, and the host-emulation build of gs_horus.cu byte for byte, under every kernel mapping of the
engine.  Degraded + clean add up to jobdist's records; the feature adds one launch when on and changes nothing when off;
a repeated summarise gives the same bytes; the sweep's files equal pandas on the job.csv files run_batched writes."""
import csv
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import REPO, horus_cases, load_horus
from test_interference_cpu import JC_SQ, JC_SUMS, assert_interference, job_columns_if, reference_interference
from test_jobdist_cpu import horus_emu_engine  # noqa: F401
from test_stats_edges_cpu import horus_configs

pytestmark = pytest.mark.gpu

BOUNDS = ((), (2, 4, 8), (1, 2, 3, 4, 8, 16, 32))


def _load_fixtures(eng, loaded):
    from gpuschedule_b200 import capi
    for i, (table, cluster, params, _, _) in enumerate(loaded):
        eng.config(i, cluster, capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"]))
        eng.load_trace(i, table)
        np.random.seed(params["seed"])
        eng.load_words(i, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))


def _check_jobdist_identity(recs, cls, tag):
    for c in range(len(recs)):
        dg, cl, jd = recs[c]["degraded"], recs[c]["clean"], cls[c]
        for f in JC_SUMS:
            assert int(dg[f]) + int(cl[f]) == int(jd[f]), (tag, c, f)
        for q in JC_SQ:
            u = lambda r: (int(r[q + "_sq_hi"]) << 64) | int(r[q + "_sq_lo"])   # noqa: E731
            assert u(dg) + u(cl) == u(jd), (tag, c, q)


def test_horus_fixtures_on_device_equal_the_restatement_and_the_host_build(horus_emu_engine):
    from gpuschedule_b200 import capi
    cases = horus_cases()
    loaded = [load_horus(c) for c in cases]
    host = {}
    with horus_emu_engine(device=0, nsims=len(cases)) as emu:
        _load_fixtures(emu, loaded)
        emu.run(rows_cap=1 << 15)
        for bounds in BOUNDS:
            emu.set_interference(bounds)
            emu.summarize()
            host[bounds] = emu.interference()
    for lanes in (1, 32, 0):                                 # scalar (one and 32 simulations per warp), cooperative
        with capi.HorusEngine(device=0, nsims=len(cases)) as eng:
            eng.set_lanes(lanes)
            _load_fixtures(eng, loaded)
            eng.run(rows_cap=1 << 15)
            n0 = eng.lib.gs_horus_launch_count(eng.h)
            plain = eng.summarize()
            assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 2
            for bounds in BOUNDS:
                eng.set_interference(bounds)
                eng.set_jobdist(bounds, ())
                n0 = eng.lib.gs_horus_launch_count(eng.h)
                out = eng.summarize()
                assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 4          # + jobdist + interference
                assert out.tobytes() == plain.tobytes()
                recs = eng.interference()
                cls, _ = eng.jobdist()
                assert recs.tobytes() == host[bounds].tobytes(), (lanes, bounds)
                eng.summarize()
                assert eng.interference().tobytes() == recs.tobytes()           # a repeated summarise: the same bytes
                for i, (case, (table, _, _, _, _)) in enumerate(zip(cases, loaded)):
                    _, _, _, hrecs, order = eng.fetch(i)
                    tag = f"{case} lanes={lanes} bounds={bounds}"
                    assert_interference(recs[i], reference_interference(*job_columns_if(table, hrecs, order), bounds), tag)
                    _check_jobdist_identity(recs[i], cls[i], tag)
            eng.set_jobdist(None, None)
            eng.set_interference(None)
            n0 = eng.lib.gs_horus_launch_count(eng.h)
            assert eng.summarize().tobytes() == plain.tobytes()
            assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 2
            eng.set_interference((4,))
            n0 = eng.lib.gs_horus_launch_count(eng.h)
            assert eng.summarize().tobytes() == plain.tobytes()
            assert eng.lib.gs_horus_launch_count(eng.h) - n0 == 3


def test_heterogeneous_handle_with_more_jobs_than_a_block():
    from gpuschedule_b200 import capi
    configs = horus_configs(48, seed=21, big=600)
    np.random.seed(5)
    words = np.random.randint(0, 2 ** 32, size=64 << 20, dtype=np.uint32)
    bounds = (2, 4, 8, 16)
    with capi.HorusEngine(device=0, nsims=len(configs)) as eng:
        for i, (cl, table, params) in enumerate(configs):
            eng.config(i, cl, params)
            eng.load_trace(i, table)
        eng.load_words(-1, words)
        eng.set_interference(bounds)
        eng.set_jobdist(bounds, ())
        for _ in range(1000):
            eng.run(rows_cap=1 << 16)
            if all(eng.stats(i).done for i in range(len(configs))):
                break
        out = eng.summarize()
        recs = eng.interference()
        cls, _ = eng.jobdist()
        assert out["finished"].max() > 256 and (out["status"] == 0).all()
        assert int(recs["degraded"]["jobs"].sum()) > 0 and int(recs["clean"]["jobs"].sum()) > 0
        part = eng.interference(first=7, count=20)
        assert part.tobytes() == recs[7:27].tobytes()
        for i, (_, table, _) in enumerate(configs):
            _, _, _, hrecs, order = eng.fetch(i)
            assert_interference(recs[i], reference_interference(*job_columns_if(table, hrecs, order), bounds), f"replica {i}")
            _check_jobdist_identity(recs[i], cls[i], f"replica {i}")


def test_error_codes_on_device():
    from gpuschedule_b200 import capi
    from test_jobdist_cpu import _code
    table, cluster, params, _, _ = load_horus("horus_small")
    with capi.HorusEngine(device=0, nsims=2) as eng:
        _load_fixtures(eng, [(table, cluster, params, None, None)] * 2)
        assert _code(eng.interference) == capi.GS_ERR_STATE
        eng.set_interference((4,))
        assert _code(eng.interference) == capi.GS_ERR_STATE                 # nothing has run
        eng.run(rows_cap=1 << 15)
        assert _code(eng.interference) == capi.GS_ERR_STATE                 # not summarised
        eng.summarize()
        recs = eng.interference()
        for bad in ((0,), (4, 4), tuple(range(1, 9))):
            assert _code(eng.set_interference, bad) == capi.GS_ERR_ARG
        assert eng.interference().tobytes() == recs.tobytes()
        assert _code(eng.interference, 1, 2) == capi.GS_ERR_ARG
        assert eng.lib.gs_horus_fetch_interference(eng.h, 0, 1, None) == capi.GS_ERR_ARG


# ---------------------------------------------------------------- sweep
def _pandas_numbers(job_csv, bounds):
    import pandas as pd
    temp = pd.read_csv(job_csv)
    temp["cls"] = [sum(1 for b in bounds if b <= g) for g in temp["num_gpu"]]
    out = []
    for c in range(len(bounds) + 1):
        t = temp[temp["cls"] == c]
        td = t[t["actual_duration"] > t["original_duration"]]
        out.append(dict(jobs=len(t), degraded=len(td), preempted_jobs=int((t["preempt"] > 1).sum()),
                        degraded_jct_mean=td.jct.mean(), degraded_jct_median=td.jct.median(), degraded_jct_std=td.jct.std(),
                        actual_mean=t.actual_duration.mean(), actual_median=t.actual_duration.median()))
    return out


def _close(got, want, tol):
    if isinstance(want, float) and math.isnan(want):
        return math.isnan(got)
    return abs(got - want) <= tol * max(1.0, abs(want))


def test_sweep_interference_files_equal_pandas_on_the_written_job_csv(tmp_path):
    from gpuschedule_b200 import summary, sweep, tracegen
    trace = tracegen.write_trace(str(tmp_path / "t.csv"), 400, seed=5)
    env = {**os.environ, "PYTHONPATH": REPO}
    bounds = (4,)
    common = [sys.executable, "-m", "gpuschedule_b200.sweep", "--trace", trace, "--schedule", "horus", "gandiva", "fifo",
              "--num_switch", "1", "--num_node_p_switch", "8", "--repeats", "3", "--seed", "1"]
    out0, out, ifp, ifci = (tmp_path / n for n in ("s0.csv", "s.csv", "if.csv", "ifci.csv"))
    subprocess.run(common + ["--summary", str(out0)], check=True, cwd=str(tmp_path), env=env)
    subprocess.run(common + ["--summary", str(out), "--interference", str(ifp), "--interference-ci", str(ifci), "--gpu-classes", "4"],
                   check=True, cwd=str(tmp_path), env=env)
    with open(out0, "rb") as f0, open(out, "rb") as f1:                      # the summary file does not change
        assert f0.read() == f1.read()
    with open(ifp, newline="") as f:
        lines = list(csv.reader(f))
    head = lines[0]
    assert head == sweep.SUMMARY_KEYS + ["class", "gpus_min", "gpus_max"] + summary.interference_columns()
    assert len(lines) == 1 + 2 * 3 * 2                                        # horus and gandiva, 3 seeds, 2 classes
    sets = [sweep.make_flags(trace_file=trace, schedule=sc, scheme=sc, num_switch=1, num_node_p_switch=8, num_queue=4, num_buffer=5,
                             log_path=f"{sc}_{rep}", seed=1 + rep) for sc in ("horus", "gandiva") for rep in range(3)]
    written = sweep.run_batched(sets, out_root=str(tmp_path / "log"))
    col = {n: head.index(n) for n in head}
    per_run = []
    for k, (fl, (out_dir, _)) in enumerate(zip(sets, written)):
        want = _pandas_numbers(os.path.join(out_dir, "job.csv"), bounds)
        per_run.append(want)
        for c in range(2):
            ln = lines[1 + 2 * k + c]
            assert ln[2] == fl.schedule and int(ln[5]) == fl.seed and int(ln[6]) == c
            for name in ("jobs", "degraded", "preempted_jobs"):
                assert int(ln[col[name]]) == want[c][name], (fl.schedule, fl.seed, c, name)
            for name in ("degraded_jct_mean", "degraded_jct_median"):
                assert _close(float(ln[col[name]]), want[c][name], 1e-15), (fl.schedule, c, name)
            assert _close(float(ln[col["degraded_jct_std"]]), want[c]["degraded_jct_std"], 1e-12)
            for name in ("actual_mean", "actual_median"):
                assert _close(float(ln[col[name]]), want[c][name], 2 ** -11), (fl.schedule, c, name)
    with open(ifci, newline="") as f:
        ci = list(csv.reader(f))
    assert ci[0] == sweep.SUMMARY_KEYS + ["repeats", "class", "gpus_min", "gpus_max", "replicas", "level"] + summary.interference_spread_columns()
    assert len(ci) == 1 + 2 * 2
    cc = {n: ci[0].index(n) for n in ci[0]}
    for g in range(2):
        for c in range(2):
            ln = ci[1 + 2 * g + c]
            runs = [per_run[3 * g + r][c] for r in range(3) if per_run[3 * g + r][c]["jobs"] > 0]
            assert int(ln[cc["replicas"]]) == len(runs) and int(ln[cc["repeats"]]) == 3
            v = np.array([r["actual_mean"] for r in runs])
            if len(v):
                assert abs(float(ln[cc["actual_mean_mean"]]) - v.mean()) <= 2 ** -11

"""Interference statistics of the utilisation-aware engine (gs_ifclass, gpuschedule_b200/csrc/gs_summary.cuh) on a box
without a GPU.

gs_if_fp / gs_if_value and gs_if_serial, the kernel's steps run serially, are compiled with g++
(tests/emu/interference_emu.cpp) and compared with `reference_interference`, a numpy / Python-int restatement of the
definitions in include/gsched_horus.h, on seeded random job sets.  gs_horus_set_interference /
gs_horus_fetch_interference run through the host-emulation build of gs_horus.cu on every horus-family fixture, where
summary.interference_derived must give what scheduler_analysis.ipynb's interference cell computes with pandas from the
reference's own job.csv.  summary.interference_spread and the sweep's argument errors too."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, REPO, horus_cases, load_horus
from test_jobdist_cpu import _code, horus_emu_engine, reference_jobdist  # noqa: F401
from test_summary_cpu import PERMILLE

IF_MAX = 2 ** 31 - 1
JC_SUMS = ("jobs", "wait_sum", "turnaround_sum", "jct_sum", "preempt_sum", "gpu_ticks_sum")
JC_SQ = ("wait", "turnaround", "jct")


# ---------------------------------------------------------------- the restatement (shared with test_gpu_interference.py)
def fp(x):
    """(fixed-point value, saturated) of a duration: min(2^31 - 1, max(0, round-half-even(1024 x))), NaN as 0"""
    r = np.rint(1024.0 * np.float64(x))
    if math.isnan(r) or r < 0:
        return 0, True
    if r > IF_MAX:
        return IF_MAX, True
    return int(r), False


def _mid(vals):
    s = sorted(vals)
    k = len(s)
    return [s[(k - 1) // 2], s[k // 2]] if k else [0, 0]


def _q(vals):
    s = sorted(vals)
    k = len(s)
    return [s[(p * k + 999) // 1000 - 1] for p in PERMILLE] if k else [0] * 5


def reference_interference(arrive, gpus, start, end, jct, preempt, original, actual, bounds):
    """per class a dict of gs_ifclass fields: "degraded" / "clean" reference_jobdist's class dicts, 128-bit fields as
    exact ints ("actual_sq", "lost_gpu_time"), the rest as in the struct"""
    cols = [[int(x) for x in np.asarray(a, dtype=np.int64).tolist()] for a in (arrive, gpus, start, end, jct, preempt)]
    arrive, gpus, start, end, jct, preempt = cols
    original = [float(x) for x in np.asarray(original, dtype=np.float64)]
    actual = [float(x) for x in np.asarray(actual, dtype=np.float64)]
    out = []
    for c in range(len(bounds) + 1):
        idx = [i for i in range(len(gpus)) if sum(1 for b in bounds if b <= gpus[i]) == c]
        d = dict(actual_sum=0, actual_sq=0, original_sum=0, excess_sum=0, excess_max=0, lost_gpu_time=0, preempted_jobs=0,
                 preempt_max=0, clamped=0)
        a_vals, groups = [], {True: [], False: []}
        for i in idx:
            deg = actual[i] > original[i]
            a, ca = fp(actual[i])
            o, co = fp(original[i])
            e, ce = fp(np.float64(actual[i]) - np.float64(original[i])) if deg else (0, False)
            groups[deg].append(i)
            a_vals.append(a)
            d["actual_sum"] += a
            d["actual_sq"] += a * a
            d["original_sum"] += o
            if deg:
                d["excess_sum"] += e
                d["excess_max"] = max(d["excess_max"], e)
                d["lost_gpu_time"] += gpus[i] * e
            d["preempted_jobs"] += preempt[i] > 1
            d["preempt_max"] = max(d["preempt_max"], preempt[i])
            d["clamped"] += ca or co or ce
        for deg, name in ((True, "degraded"), (False, "clean")):
            g = groups[deg]
            pick = lambda col: [col[i] for i in g]            # noqa: E731
            d[name] = reference_jobdist(pick(arrive), pick(gpus), pick(start), pick(end), pick(jct), pick(preempt), (), ())[0][0]
        d["degraded_jct_mid"] = _mid([jct[i] for i in groups[True]])
        d["actual_q"] = _q(a_vals)
        d["actual_mid"] = _mid(a_vals)
        out.append(d)
    return out


def ifclass_fields(rec):
    """one IFCLASS_DTYPE record as the dict reference_interference makes"""
    from test_jobdist_cpu import jclass_fields
    d = {name: jclass_fields(rec[name]) for name in ("degraded", "clean")}
    for name in ("actual_sum", "original_sum", "excess_sum", "excess_max", "preempted_jobs", "preempt_max", "clamped"):
        d[name] = int(rec[name])
    d["actual_sq"] = (int(rec["actual_sq_hi"]) << 64) | int(rec["actual_sq_lo"])
    d["lost_gpu_time"] = (int(rec["lost_gpu_time_hi"]) << 64) | int(rec["lost_gpu_time_lo"])
    for name in ("degraded_jct_mid", "actual_q", "actual_mid"):
        d[name] = rec[name].tolist()
    return d


def assert_interference(recs, ref, tag=""):
    assert len(recs) == len(ref), tag
    for c, (rec, want) in enumerate(zip(recs, ref)):
        got = ifclass_fields(rec)
        for key, v in want.items():
            if key in ("degraded", "clean"):
                for f, x in v.items():
                    assert got[key][f] == x, (tag, c, key, f, got[key][f], x)
            else:
                assert got[key] == v, (tag, c, key, got[key], v)
        assert rec["reserved"] == 0 and rec["degraded"]["reserved"] == 0 and rec["clean"]["reserved"] == 0, (tag, c)


def job_columns_if(table, hrecs, order):
    """(arrive, gpus, start, end, jct, preempt, original, actual) of the finished jobs in finish order"""
    o = np.asarray(order, dtype=np.int64)
    return (table.arrive_tick[o], table.gpus[o], hrecs["start"][o], hrecs["end"][o], hrecs["jct"][o], hrecs["preempt"][o],
            hrecs["original"][o], hrecs["actual"][o])


# ---------------------------------------------------------------- host build
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("interference_emu") / "libinterference_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "interference_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.emu_if_fp.argtypes = [C.c_double, C.POINTER(C.c_int)]
    lib.emu_if_fp.restype = C.c_int
    lib.emu_if_jobs.restype = C.c_int
    return lib


def _p(a):
    return np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def emu_interference(lib, jobs, bounds):
    """(rc, records) of gs_if_serial over (arrive, gpus, start, end, jct, preempt, original, actual); the output starts
    filled with 0xAB bytes so that an untouched one can be told apart"""
    from gpuschedule_b200 import capi
    ints = [np.ascontiguousarray(c, dtype=np.int32) for c in jobs[:6]]
    dbl = [np.ascontiguousarray(c, dtype=np.float64) for c in jobs[6:]]
    b = np.ascontiguousarray(bounds, dtype=np.int32) if len(bounds) else np.zeros(1, dtype=np.int32)
    nc = len(bounds) + 1
    recs = np.frombuffer(b"\xab" * (nc * capi.IFCLASS_DTYPE.itemsize), dtype=capi.IFCLASS_DTYPE).copy()
    arrive, gpus, start, end, jct, preempt = ints
    rc = lib.emu_if_jobs(_p(arrive), _p(start), _p(end), _p(jct), _p(preempt), _p(gpus), _p(dbl[0]), _p(dbl[1]),
                         C.c_longlong(len(arrive)), C.c_int(nc), _p(b), _p(recs))
    return rc, recs


def test_layout_matches_the_dtype(emu):
    from gpuschedule_b200 import capi
    out = np.zeros(18, dtype=np.int64)
    emu.emu_if_layout(_p(out))
    dt = capi.IFCLASS_DTYPE
    assert out[0] == dt.itemsize == 440 and dt.itemsize % 8 == 0
    assert out[1:].tolist() == [dt.fields[n][1] for n in dt.names]


def test_fixed_point_rounding(emu):
    cases = [(5.0, 5120, 0), (4.999999999999998, 5120, 0), (5.000000000000002, 5120, 0), (0.5 / 1024, 0, 0), (1.5 / 1024, 2, 0),
             (2.5 / 1024, 2, 0), (-0.4 / 1024, 0, 0), (-1.0, 0, 1), ((2 ** 31 - 1) / 1024, IF_MAX, 0), (2 ** 21, IF_MAX, 1),
             (1e300, IF_MAX, 1), (float("inf"), IF_MAX, 1), (float("-inf"), 0, 1), (float("nan"), 0, 1), (0.0, 0, 0)]
    for x, want, cl in cases:
        c = C.c_int(-1)
        assert emu.emu_if_fp(x, C.byref(c)) == want and c.value == cl, x
        assert fp(x) == (want, bool(cl)), x
    # the reference's +5 quirk: original + 5 in double, then the difference, is 5120 whatever the rounding error
    rng = np.random.default_rng(3)
    for o in rng.uniform(0, 10 ** 5, 2000):
        a = o + 5.0
        c = C.c_int(0)
        assert emu.emu_if_fp(a - o, C.byref(c)) == 5120 and c.value == 0, o


def _random_jobs(rng, k, gpus_choice=(1, 2, 4, 8, 16, 32), p_degraded=0.4, dur_hi=5000.0):
    arrive = rng.integers(0, 10 ** 5, k)
    start = arrive + rng.integers(0, 10 ** 4, k)
    jct = rng.integers(1, 5000, k)
    end = start + jct
    gpus = rng.choice(gpus_choice, k)
    preempt = rng.integers(0, 4, k)
    original = np.round(rng.uniform(0.5, dur_hi, k), 4)
    deg = rng.random(k) < p_degraded
    actual = np.where(deg, original + np.where(rng.random(k) < 0.5, 5.0, rng.uniform(0.001, 500.0, k)), original)
    return [arrive, gpus, start, end, jct, preempt, original, actual]


def test_random_job_sets(emu):
    rng = np.random.default_rng(17)
    sets = []
    for k, p in ((0, 0.4), (1, 1.0), (2, 0.0), (7, 0.5), (300, 0.4), (2000, 0.3), (513, 1.0), (400, 0.0)):
        sets.append((f"k={k} p={p}", _random_jobs(rng, k, p_degraded=p)))
    sat = _random_jobs(rng, 200)                                       # saturating durations: clamped
    sat[7][::3] = 3.0e6
    sat[6][::7] = 2.5e6
    sat[6][1::11] = -1.0
    sets.append(("saturated", sat))
    big = _random_jobs(rng, 40, gpus_choice=(2 ** 30, 2 ** 30 + 7), p_degraded=1.0)   # lost GPU time past 2^64
    big[4][:] = 1
    big[7][:] = big[6] + 2.4e6
    sets.append(("lost past 2^64", big))
    for tag, jobs in sets:
        for bounds in ((), (4,), (5, 17, 65), (1, 2, 3, 4, 8, 16, 32), (10 ** 6,)):
            rc, recs = emu_interference(emu, jobs, bounds)
            assert rc == 0
            ref = reference_interference(*jobs, bounds)
            assert_interference(recs, ref, f"{tag} {bounds}")
            if tag == "lost past 2^64":
                assert ref[-1]["lost_gpu_time"] >= 2 ** 64 and ref[-1]["clamped"] == len(jobs[0])
            if tag == "saturated" and not bounds:
                assert ref[0]["clamped"] > 0
    assert emu_interference(emu, sets[3][1], (3, 3))[0] == -1
    assert emu_interference(emu, sets[3][1], (0,))[0] == -1


# ---------------------------------------------------------------- gs_horus_set_interference / gs_horus_fetch_interference, host build of gs_horus.cu
def _loaded_engine(eng, loaded):
    from gpuschedule_b200 import capi
    for i, (table, cluster, params, _, _) in enumerate(loaded):
        eng.config(i, cluster, capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"]))
        eng.load_trace(i, table)
        np.random.seed(params["seed"])
        eng.load_words(i, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))


def test_horus_interference_host_build(horus_emu_engine):
    import pandas as pd
    from gpuschedule_b200 import capi, summary
    cases = horus_cases()
    loaded = [load_horus(c) for c in cases]
    with horus_emu_engine(device=0, nsims=len(cases)) as eng:
        _loaded_engine(eng, loaded)
        for bounds in ((0,), (3, 3), (5, 2), tuple(range(1, 9))):
            assert _code(eng.set_interference, bounds) == capi.GS_ERR_ARG, bounds
        assert _code(eng.interference) == capi.GS_ERR_STATE                  # off
        eng.set_interference(())
        assert _code(eng.interference) == capi.GS_ERR_STATE                  # nothing has run
        eng.run(rows_cap=1 << 15)
        assert _code(eng.interference) == capi.GS_ERR_STATE                  # not summarised
        eng.set_interference(None)
        plain = eng.summarize()
        total_degraded = 0
        for bounds in ((), (5, 17, 65), (1, 2, 3, 4, 8, 16, 32), (2, 4)):
            eng.set_interference(bounds)
            eng.set_jobdist(bounds, ())
            assert _code(eng.interference) == capi.GS_ERR_STATE              # setting it asks for a new summary
            assert eng.summarize().tobytes() == plain.tobytes()              # the summaries do not change
            recs = eng.interference()
            assert recs.shape == (len(cases), len(bounds) + 1)
            assert eng.interference(first=2, count=3).tobytes() == recs[2:5].tobytes()
            assert eng.interference(first=4, count=0).shape == (0, len(bounds) + 1)
            assert _code(eng.interference, 3, len(cases)) == capi.GS_ERR_ARG
            assert _code(eng.interference, -1, 1) == capi.GS_ERR_ARG
            cls, _ = eng.jobdist()
            for i, (case, (table, _, _, _, _)) in enumerate(zip(cases, loaded)):
                _, _, _, hrecs, order = eng.fetch(i)
                assert_interference(recs[i], reference_interference(*job_columns_if(table, hrecs, order), bounds), f"{case} {bounds}")
                for c in range(len(bounds) + 1):                         # degraded + clean = jobdist, counts and sums
                    dg, cl, jd = recs[i][c]["degraded"], recs[i][c]["clean"], cls[i][c]
                    for f in JC_SUMS:
                        assert int(dg[f]) + int(cl[f]) == int(jd[f]), (case, c, f)
                    for q in JC_SQ:
                        u = lambda r: (int(r[q + "_sq_hi"]) << 64) | int(r[q + "_sq_lo"])   # noqa: E731
                        assert u(dg) + u(cl) == u(jd), (case, c, q)
                if bounds:
                    continue
                # scheduler_analysis.ipynb's interference cell on the reference's own job.csv
                temp = pd.read_csv(os.path.join(GOLDEN, case, "job.csv"))
                temp_degrade = temp[temp["actual_duration"] > temp["original_duration"]]
                d = summary.interference_derived(recs[i])
                kd = len(temp_degrade)
                total_degraded += kd
                assert d["degraded"][0] == kd and d["jobs"][0] == len(temp), case
                assert d["preempted_jobs"][0] == int((temp["preempt"] > 1).sum()), case
                if case.startswith("yarn_sched_"):
                    assert kd == 0, case
                if kd:
                    assert d["degraded_jct_mean"][0] == temp_degrade.jct.mean(), case
                    assert d["degraded_jct_median"][0] == temp_degrade.jct.median(), case
                    if kd > 1:
                        assert math.isclose(d["degraded_jct_std"][0], temp_degrade.jct.std(), rel_tol=1e-12), case
                else:
                    assert math.isnan(d["degraded_jct_mean"][0]) and math.isnan(d["degraded_jct_median"][0])
                assert abs(d["actual_mean"][0] - temp.actual_duration.mean()) <= 2 ** -11, case
                assert abs(d["actual_median"][0] - temp.actual_duration.median()) <= 2 ** -11, case
                assert math.isclose(d["actual_std"][0], temp.actual_duration.std(), rel_tol=1e-3), case
                assert d["degraded_share"][0] == kd / len(temp)
            if not bounds:
                assert total_degraded == 213
        # an error leaves the setting and the outputs as they were
        before = eng.interference()
        for bounds in ((0,), (4, 2), tuple(range(1, 9))):
            assert _code(eng.set_interference, bounds) == capi.GS_ERR_ARG
        assert eng.interference().tobytes() == before.tobytes()
        eng.set_interference(None)
        assert _code(eng.interference) == capi.GS_ERR_STATE
        assert eng.jobdist()[0].shape[1] == 3                              # jobdist is still on


def test_gandiva_fixtures_preempt_more_than_once(horus_emu_engine):
    cases = ["gandiva_small", "gandiva_slice"]
    loaded = [load_horus(c) for c in cases]
    with horus_emu_engine(device=0, nsims=2) as eng:
        _loaded_engine(eng, loaded)
        eng.run(rows_cap=1 << 15)
        eng.set_interference(())
        eng.summarize()
        recs = eng.interference()
    assert recs["preempted_jobs"][:, 0].tolist() == [7, 10]
    assert (recs["preempt_max"][:, 0] > 1).all()


# ---------------------------------------------------------------- summary.interference_derived / interference_spread
def test_interference_derived_matches_pandas(emu):
    import pandas as pd
    from gpuschedule_b200 import summary
    rng = np.random.default_rng(5)
    jobs = _random_jobs(rng, 3000, gpus_choice=(1, 2, 4, 8, 16, 32, 64, 128))
    jobs[1][0] = 4096                                         # the last class holds exactly one job: std NaN
    bounds = (5, 17, 65, 4096)
    rc, recs = emu_interference(emu, jobs, bounds)
    assert rc == 0
    d = summary.interference_derived(recs)
    df = pd.DataFrame(dict(gpus=jobs[1], jct=jobs[4], preempt=jobs[5], original_duration=jobs[6], actual_duration=jobs[7]))
    df["cls"] = [sum(1 for b in bounds if b <= g) for g in df["gpus"]]
    assert len(summary.interference_flat(d, 0)) == len(summary.interference_columns())
    for c in range(len(bounds) + 1):
        temp = df[df["cls"] == c]
        temp_degrade = temp[temp["actual_duration"] > temp["original_duration"]]
        assert d["jobs"][c] == len(temp) and d["degraded"][c] == len(temp_degrade)
        assert d["degraded_jct_mean"][c] == temp_degrade.jct.mean() and d["degraded_jct_median"][c] == temp_degrade.jct.median()
        assert abs(d["actual_mean"][c] - temp.actual_duration.mean()) <= 2 ** -11
        assert abs(d["actual_median"][c] - temp.actual_duration.median()) <= 2 ** -11
        if len(temp) > 1:
            assert math.isclose(d["degraded_jct_std"][c], temp_degrade.jct.std(), rel_tol=1e-12)
            assert math.isclose(d["actual_std"][c], temp.actual_duration.std(), rel_tol=1e-4)
        else:
            assert math.isnan(d["actual_std"][c]) and math.isnan(d["degraded_jct_std"][c])
        np.testing.assert_allclose(d["clean_jct_mean"][c], temp.jct[temp.index.difference(temp_degrade.index)].mean(), rtol=1e-12)
        exc = [fp(a - o)[0] for a, o in zip(temp_degrade.actual_duration, temp_degrade.original_duration)]
        assert d["excess_mean"][c] == sum(exc) / len(exc) / 1024
        assert d["lost_gpu_time"][c] == sum(g * e for g, e in zip(temp_degrade.gpus, exc)) / 1024
        assert d["preempted_share"][c] == (temp.preempt > 1).mean()
        assert d["degraded_share"][c] == len(temp_degrade) / len(temp)
    empty = np.zeros(2, dtype=recs.dtype)
    e = summary.interference_derived(empty)
    assert e["jobs"].tolist() == [0, 0] and np.isnan(e["actual_mean"]).all() and np.isnan(e["degraded_share"]).all()


def test_interference_spread_over_the_runs_that_have_jobs_in_a_class(emu):
    from gpuschedule_b200 import summary
    rng = np.random.default_rng(11)
    R, bounds = 6, (8,)
    recs = []
    for r in range(R):
        jobs = _random_jobs(rng, 50, gpus_choice=(1, 2, 4) if r % 2 else (1, 16), p_degraded=0.5)
        recs.append(emu_interference(emu, jobs, bounds)[1])
    recs = np.stack(recs)
    sp = summary.interference_spread(recs, level=0.9)
    assert sp["replicas"].tolist() == [6, 3]                               # class 1 only in the even runs
    per = [summary.interference_derived(recs[r]) for r in range(R)]
    for c, runs in ((0, range(R)), (1, range(0, R, 2))):
        for m in ("actual_mean", "degraded_jct_median", "lost_gpu_time"):
            v = np.array([per[r][m][c] for r in runs])
            ref = summary._spread_of(v, summary.Fraction("0.9"))
            assert [sp[m][s][c] for s in summary.SPREAD_STATS] == pytest.approx([ref[s] for s in summary.SPREAD_STATS], nan_ok=True)
    assert len(summary.interference_spread_flat(sp, 0)) == len(summary.interference_spread_columns())
    with pytest.raises(ValueError):
        summary.interference_spread(recs[0])
    with pytest.raises(ValueError):
        summary.interference_spread(recs, level=0)


# ---------------------------------------------------------------- sweep argument errors (before any engine exists)
def test_sweep_interference_argument_errors(tmp_path, monkeypatch):
    from gpuschedule_b200 import capi, sweep

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(capi, "Engine", no_engine)
    monkeypatch.setattr(capi, "HorusEngine", no_engine)
    fl = [sweep.make_flags(trace_file=str(tmp_path / "missing.csv"), schedule="horus", scheme="horus")]
    for bad in ((0,), (3, 3), (5, 2), tuple(range(1, 9)), (2 ** 31,), ("x",), 5):
        with pytest.raises(ValueError):
            sweep.summarize_batched(fl, interference=bad)
    assert sweep.check_interference([5, 17]) == (5, 17)
    base = ["--trace", str(tmp_path / "missing.csv")]
    for argv in (["--schedule", "horus", "--interference", "i.csv"],                                    # no --summary
                 ["--schedule", "fifo", "sjf", "--summary", "s.csv", "--interference", "i.csv"],          # nothing utilisation-aware
                 ["--schedule", "horus", "--summary", "s.csv", "--interference-ci", "c.csv", "--repeats", "3"],   # no --interference
                 ["--schedule", "horus", "--summary", "s.csv", "--interference", "i.csv", "--interference-ci", "c.csv"],  # R = 1
                 ["--schedule", "horus", "--summary", "s.csv", "--interference", "i.csv", "--gpu-classes", "5", "5"],
                 ["--schedule", "horus", "--summary", "s.csv", "--interference", "i.csv", "--gpu-classes", "0"],
                 ["--schedule", "horus", "--summary", "s.csv", "--interference", "i.csv", "--bootstrap", "4"],
                 ["--schedule", "fifo", "--summary", "s.csv", "--interference", "i.csv", "--bootstrap", "4"]):
        with pytest.raises(SystemExit) as e:
            sweep.main(base + argv)
        assert e.value.code == 2, argv
    for name in ("i.csv", "s.csv", "c.csv"):
        assert not (tmp_path / name).exists()

"""Job statistics by job size (gs_jclass and CDF counts, gpuschedule_b200/csrc/gs_summary.cuh) on a box without a GPU.

The __host__ __device__ part -- the class key, the CDF bin, the setting's validation -- and gs_jd_jobs_serial, the
kernel's steps run serially with the summary's own radix select, are compiled with g++ (tests/emu/jobdist_emu.cpp)
and compared with a numpy breakdown of job records: the fixtures' reference-made job.csv (fifo, horus), the pinned
policy oracles' records, and seeded random job sets.  gs_horus_set_jobdist / gs_horus_fetch_jobdist run through the
host-emulation build of gs_horus.cu.  summary.jobdist_derived / jobdist_spread and the sweep's argument errors too."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, REPO, golden_cases, horus_cases, load_golden, load_horus
from test_summary_cpu import PERMILLE, _policy_cases, job_columns, load_policy, reference_summary

QUANTS = ("wait", "turnaround", "jct")
DEFAULT_EDGES = tuple(2 ** i for i in range(31))


# ---------------------------------------------------------------- the numpy breakdown (shared with test_gpu_jobdist.py)
def reference_jobdist(arrive, gpus, start, end, jct, preempt, bounds, edges):
    """(per class a dict of gs_jclass fields -- sums of squares as exact ints "<q>_sq" --, CDF counts (C, 3, E + 1)) of
    the finished jobs' columns; a job's class is #(bounds <= gpus), a value's bin #(edges < value)"""
    arrive, gpus, start, end, jct, preempt = (np.asarray(a, dtype=np.int64) for a in (arrive, gpus, start, end, jct, preempt))
    cls = np.array([sum(1 for b in bounds if b <= g) for g in gpus.tolist()], dtype=np.int64)
    vals = dict(wait=start - arrive, turnaround=end - arrive, jct=jct)
    nc, ne = len(bounds) + 1, len(edges)
    e = np.asarray(edges, dtype=np.int64)
    hist = np.zeros((nc, 3, ne + 1), dtype=np.int64)
    out = []
    for c in range(nc):
        m = cls == c
        k = int(m.sum())
        d = dict(jobs=k, preempt_sum=int(preempt[m].sum()), gpu_ticks_sum=int((gpus[m] * jct[m]).sum()))
        for i, q in enumerate(QUANTS):
            v = vals[q][m]
            d[q + "_sum"] = int(v.sum())
            d[q + "_sq"] = sum(x * x for x in v.tolist())
            s = np.sort(v)
            d[q + "_q"] = [int(s[(p * k + 999) // 1000 - 1]) for p in PERMILLE] if k else [0] * 5
            cum = [int((v <= x).sum()) for x in e.tolist()] + [k]       # #(v <= e_b): the CDF counts
            hist[c, i] = np.diff([0] + cum)
        out.append(d)
    return out, hist


def jclass_fields(rec):
    """one JCLASS_DTYPE record as the dict reference_jobdist makes"""
    d = {name: (rec[name].tolist() if rec[name].shape else rec[name].item()) for name in rec.dtype.names}
    for q in QUANTS:
        d[q + "_sq"] = (int(rec[q + "_sq_hi"]) << 64) | int(rec[q + "_sq_lo"])
    return d


def assert_jobdist(classes, hist, ref, tag=""):
    want_cls, want_hist = ref
    assert len(classes) == len(want_cls), tag
    for c, (rec, want) in enumerate(zip(classes, want_cls)):
        got = jclass_fields(rec)
        for key, w in want.items():
            assert got[key] == w, (tag, c, key, got[key], w)
    assert np.array_equal(np.asarray(hist, dtype=np.int64), want_hist), tag


def csv_jobs(job_csv_path, table):
    """(arrive, gpus, start, end, jct, preempt) of the lines of a reference-made job.csv, arrive from the trace"""
    import pandas as pd
    jb = pd.read_csv(job_csv_path)
    index = {str(lab): j for j, lab in enumerate(table.label)}
    o = np.array([index[str(v)] for v in jb["job_id"].tolist()], dtype=np.int64)
    return (table.arrive_tick[o], table.gpus[o]) + tuple(jb[c].to_numpy(np.int64) for c in ("start_time", "end_time", "jct", "preempt"))


def settings_for(jobs):
    """(bounds, edges) settings that cover the cases: one class and no edge; the notebook's classes with the default
    edges; eight classes; bounds equal to the jobs' own num_gpu values; every job in one class; edges equal to the
    values; 255 edges spanning below the smallest and above the largest value; edges all below / all above"""
    arrive, gpus, start, end, jct, _ = (np.asarray(a, dtype=np.int64) for a in jobs)
    vals = np.concatenate([start - arrive, end - arrive, jct])
    lo, hi = int(vals.min()) if len(vals) else 0, int(vals.max()) if len(vals) else 1
    step = max(1, (hi - lo + 20) // 254)
    own = tuple(int(g) for g in np.unique(gpus[gpus >= 1])[:7])
    return [((), ()), ((5, 17, 65), DEFAULT_EDGES), ((1, 2, 3, 4, 8, 16, 32), (0, 10, 100, 1000)), (own, (1, 4)),
            ((10 ** 6,), (lo, hi)), ((1,), tuple(int(x) for x in np.unique(vals)[:255])),
            ((2, 4), tuple(lo - 10 + step * i for i in range(255))), ((4,), (-10, -5)), ((), (2 ** 31 - 2, 2 ** 31 - 1))]


# ---------------------------------------------------------------- host build
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("jobdist_emu") / "libjobdist_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "jobdist_emu.cpp")], check=True)
    lib = C.CDLL(out)
    for name in ("emu_jd_class", "emu_jd_bin", "emu_jd_jobs"):
        getattr(lib, name).restype = C.c_int
    return lib


def _p(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def emu_jobdist(lib, jobs, bounds, edges, nclasses=None):
    """(rc, classes, hist) of gs_jd_jobs_serial over the job columns (arrive, gpus, start, end, jct, preempt)"""
    from gpuschedule_b200.capi import JCLASS_DTYPE
    arrive, gpus, start, end, jct, preempt = (_i32(c) for c in jobs)
    nc = len(bounds) + 1 if nclasses is None else nclasses
    classes = np.zeros(max(nc, 1), dtype=JCLASS_DTYPE)
    hist = np.zeros((max(nc, 1), 3, len(edges) + 1), dtype=np.uint32)
    b, e = _i32(bounds if len(bounds) else [0]), _i32(edges if len(edges) else [0])
    rc = lib.emu_jd_jobs(_p(arrive), _p(start), _p(end), _p(jct), _p(preempt), _p(gpus), C.c_longlong(len(arrive)), C.c_int(nc),
                         _p(b) if len(bounds) else None, C.c_int(len(edges)), _p(e) if len(edges) else None, _p(classes), _p(hist))
    return rc, classes[:nc], hist[:nc]


def check_setting(lib, jobs, bounds, edges, tag):
    rc, classes, hist = emu_jobdist(lib, jobs, bounds, edges)
    assert rc == 0, tag
    ref = reference_jobdist(*jobs, bounds, edges)
    assert_jobdist(classes, hist, ref, tag)
    # the invariants: counts and sums add up to the summary's job part; every histogram row sums to its class's jobs
    s = reference_summary(np.zeros(0, dtype=_row_dtype()), *jobs)
    for f in ("wait_sum", "turnaround_sum", "jct_sum", "preempt_sum", "gpu_ticks_sum"):
        assert int(classes[f].sum()) == s[f], (tag, f)
    assert int(classes["jobs"].sum()) == s["finished"], tag
    assert (hist.astype(np.int64).sum(axis=2) == classes["jobs"][:, None]).all(), tag
    if len(bounds) == 0:                                   # one class: the summary's job part, field for field
        for f in ("wait_q", "turnaround_q", "jct_q"):
            assert classes[0][f].tolist() == s[f], (tag, f)
    return classes, hist


def _row_dtype():
    from gpuschedule_b200.log_manager import ROW_DTYPE
    return ROW_DTYPE


def test_class_and_bin_keys(emu):
    b = _i32([5, 17, 65])
    for g, want in ((0, 0), (1, 0), (4, 0), (5, 1), (16, 1), (17, 2), (64, 2), (65, 3), (1024, 3)):
        assert emu.emu_jd_class(_p(b), 3, g) == want, g
    assert emu.emu_jd_class(None, 0, 7) == 0
    e = _i32([0, 10, 20])
    for v, want in ((-5, 0), (0, 0), (1, 1), (10, 1), (11, 2), (20, 2), (21, 3), (2 ** 31 - 1, 3)):
        assert emu.emu_jd_bin(_p(e), 3, v) == want, v
    assert emu.emu_jd_bin(None, 0, 123) == 0


# ---------------------------------------------------------------- fixtures
def _fixture_jobs(kind, case):
    import oracle
    if kind == "fifo":
        table, _, _, _, _ = load_golden(case)
        return csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table)
    if kind == "horus":
        table, _, _, _, _ = load_horus(case)
        return csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table)
    table, cluster, pol = load_policy(case)
    res = oracle.run_policy(cluster, pol, table)
    return job_columns(table, res.recs, res.finish_order)


FIXTURES = [("fifo", c) for c in golden_cases()] + [("policy", c) for c in _policy_cases()] + [("horus", c) for c in horus_cases()]


@pytest.mark.parametrize("kind,case", FIXTURES)
def test_fixture_breakdown(emu, kind, case):
    jobs = _fixture_jobs(kind, case)
    assert len(jobs[0]) > 0
    for bounds, edges in settings_for(jobs):
        check_setting(emu, jobs, bounds, edges, f"{case} bounds={bounds} E={len(edges)}")


def test_fixture_settings_cover_the_edge_cases():
    """across the fixtures, the settings above meet empty classes, a class with every job, num_gpu equal to a bound,
    values equal to an edge, and E = 0 and E = 255"""
    seen = set()
    for kind, case in FIXTURES:
        jobs = _fixture_jobs(kind, case)
        gpus = np.asarray(jobs[1])
        vals = np.concatenate([np.asarray(jobs[3]) - np.asarray(jobs[0]), np.asarray(jobs[4])])
        for bounds, edges in settings_for(jobs):
            cls = np.searchsorted(np.asarray(bounds, dtype=np.int64), gpus, side="right")
            counts = np.bincount(cls, minlength=len(bounds) + 1)
            seen.add("empty class") if (counts == 0).any() else None
            seen.add("one class holds every job") if len(bounds) and counts.max() == len(gpus) else None
            seen.add("gpus equal to a bound") if np.isin(gpus, bounds).any() else None
            seen.add("value equal to an edge") if np.isin(vals, edges).any() else None
            seen.add(f"E={len(edges)}") if len(edges) in (0, 255) else None
    assert seen >= {"empty class", "one class holds every job", "gpus equal to a bound", "value equal to an edge", "E=0", "E=255"}, seen


# ---------------------------------------------------------------- seeded random job sets
def test_random_job_sets(emu):
    rng = np.random.default_rng(17)
    for k in (0, 1, 2, 3, 1000, 5000):
        for scale in (10, 2 ** 20, 2 ** 30):
            arrive = rng.integers(0, scale, k)
            start = arrive + rng.integers(0, scale, k)
            jct = rng.integers(1, scale, k)
            end = start + jct + rng.integers(0, 3, k)
            gpus = rng.choice([1, 2, 4, 5, 8, 16, 17, 32, 64, 65, 128], k)
            preempt = rng.integers(0, 4, k)
            jobs = (arrive, gpus, start, end, jct, preempt)
            for bounds, edges in (((), ()), ((5, 17, 65), DEFAULT_EDGES), ((1, 2, 4, 8, 16, 32, 64), tuple(range(0, 255 * (scale // 255 + 1), scale // 255 + 1))),
                                  ((3,), tuple(sorted(set(rng.integers(0, scale, 40).tolist()))))):
                classes, _ = check_setting(emu, jobs, bounds, edges, f"k={k} scale={scale} bounds={bounds}")
            if k >= 1000 and scale == 2 ** 30:
                assert int(classes["wait_sq_hi"].max()) > 0                  # the sums of squares need their high words


def test_setting_errors(emu):
    jobs = tuple(np.ones(4, dtype=np.int64) for _ in range(6))
    assert emu_jobdist(emu, jobs, (), ())[0] == 0
    for bounds, edges, nc in (((), (), 9), ((), (), -1), ((0,), (), None), ((3, 3), (), None), ((4, 2), (), None),
                              ((), (1, 1), None), ((), (5, 2), None), ((), tuple(range(256)), None)):
        assert emu_jobdist(emu, jobs, bounds, edges, nclasses=nc)[0] == -1, (bounds, len(edges), nc)


# ---------------------------------------------------------------- gs_horus_set_jobdist / gs_horus_fetch_jobdist, host build of gs_horus.cu
@pytest.fixture(scope="module")
def horus_emu_engine():
    import importlib.util
    import sys
    spec = importlib.util.spec_from_file_location("tests_emu_jobdist", os.path.join(REPO, "tests", "emu", "__init__.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["tests_emu_jobdist"] = mod
    spec.loader.exec_module(mod)
    out = mod._ABI_OUT
    hdr = os.path.join(REPO, "gpuschedule_b200", "csrc", "gs_summary.cuh")
    if os.path.exists(out) and os.path.getmtime(out) < os.path.getmtime(hdr) and mod._abi_lib is None:
        mod.build_abi(force=True)                 # gs_summary.cuh is not among the emu build's own dependencies
    return mod.emu_engine_class()


def _code(fn, *a):
    from gpuschedule_b200 import capi
    with pytest.raises(capi.GsError) as e:
        fn(*a)
    return e.value.code


def test_horus_jobdist_host_build_matches_reference(horus_emu_engine):
    from gpuschedule_b200 import capi
    cases = horus_cases()
    loaded = [load_horus(c) for c in cases]
    with horus_emu_engine(device=0, nsims=len(cases)) as eng:
        for i, (table, cluster, params, _, _) in enumerate(loaded):
            eng.config(i, cluster, capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"]))
            eng.load_trace(i, table)
            np.random.seed(params["seed"])
            eng.load_words(i, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))
        for bounds, edges in (((0,), ()), ((3, 3), ()), ((5, 2), ()), ((), (2, 2)), ((), (3, 1)), ((1, 2, 3, 4, 5, 6, 7, 8), ()),
                              ((), tuple(range(256))), ((), (2 ** 31,))):
            assert _code(eng.set_jobdist, bounds, edges) == capi.GS_ERR_ARG, (bounds, len(edges))
        assert _code(eng.jobdist) == capi.GS_ERR_STATE                      # off
        eng.set_jobdist((5, 17, 65), DEFAULT_EDGES)
        assert _code(eng.jobdist) == capi.GS_ERR_STATE                      # nothing has run
        eng.run(rows_cap=1 << 15)
        assert _code(eng.jobdist) == capi.GS_ERR_STATE                      # not summarised
        eng.set_jobdist(None, None)
        plain = eng.summarize()
        for bounds, edges in (((5, 17, 65), DEFAULT_EDGES), ((), ()), ((1, 2, 3, 4, 8, 16, 32), tuple(range(0, 2550, 10)))):
            eng.set_jobdist(bounds, edges)
            assert _code(eng.jobdist) == capi.GS_ERR_STATE                  # setting it asks for a new summary
            recs = eng.summarize()
            assert recs.tobytes() == plain.tobytes()                        # the summaries do not change
            classes, hist = eng.jobdist()
            assert classes.shape == (len(cases), len(bounds) + 1) and hist.shape == (len(cases), len(bounds) + 1, 3, len(edges) + 1)
            part = eng.jobdist(first=2, count=3)
            assert part[0].tobytes() == classes[2:5].tobytes() and part[1].tobytes() == hist[2:5].tobytes()
            assert _code(eng.jobdist, 3, len(cases)) == capi.GS_ERR_ARG
            assert _code(eng.jobdist, -1, 1) == capi.GS_ERR_ARG
            for i, (case, (table, _, _, _, _)) in enumerate(zip(cases, loaded)):
                _, _, _, hrecs, order = eng.fetch(i)
                jobs = job_columns(table, hrecs, order)
                assert_jobdist(classes[i], hist[i], reference_jobdist(*jobs, bounds, edges), f"{case} bounds={bounds}")
                assert_jobdist(classes[i], hist[i], reference_jobdist(*csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table), bounds, edges),
                               f"{case} job.csv bounds={bounds}")
                if not bounds:
                    for f in ("wait_sum", "turnaround_sum", "jct_sum", "preempt_sum", "gpu_ticks_sum", "wait_q", "turnaround_q", "jct_q"):
                        assert np.array_equal(classes[i][0][f], recs[i][f]), (case, f)
                    assert classes[i][0]["jobs"] == recs[i]["finished"]
        eng.set_jobdist(None, None)
        assert _code(eng.jobdist) == capi.GS_ERR_STATE


# ---------------------------------------------------------------- summary.jobdist_derived / jobdist_spread
def test_jobdist_derived_matches_pandas(emu):
    import pandas as pd
    from gpuschedule_b200 import summary
    rng = np.random.default_rng(3)
    k = 3000
    arrive = rng.integers(0, 10 ** 6, k)
    start = arrive + rng.integers(0, 2 ** 28, k)
    jct = rng.integers(1, 2 ** 29, k)
    end = start + jct
    gpus = rng.choice([1, 2, 4, 8, 16, 32, 64, 128], k)
    gpus[:1] = 200                                            # class 3 (65+) has ... exactly 1 job: std NaN
    gpus[1:] = np.where(gpus[1:] > 64, 64, gpus[1:])
    jobs = (arrive, gpus, start, end, jct, np.zeros(k, dtype=np.int64))
    bounds, edges = (5, 17, 65, 1000), (10 ** 6, 2 ** 27, 2 ** 28, 2 ** 29, 2 ** 30)
    _, classes, hist = emu_jobdist(emu, jobs, bounds, edges)
    d = summary.jobdist_derived(classes, hist, edges)
    df = pd.DataFrame(dict(wait=start - arrive, turnaround=end - arrive, jct=jct, num_gpu=gpus))
    df["cls"] = pd.cut(df["num_gpu"], [0, 4, 16, 64, 999, 10 ** 9], labels=False)
    assert d["jobs"].tolist() == [int((df["cls"] == c).sum()) for c in range(5)]
    for c in range(5):
        g = df[df["cls"] == c]
        for q in QUANTS:
            if len(g) == 0:
                assert math.isnan(d[q + "_mean"][c]) and math.isnan(d[q + "_std"][c]) and math.isnan(d[q + "_cdf"][c, 0])
                continue
            assert math.isclose(d[q + "_mean"][c], g[q].mean(), rel_tol=1e-12)
            if len(g) > 1:
                assert math.isclose(d[q + "_std"][c], g[q].std(), rel_tol=1e-12), (c, q)
            else:
                assert math.isnan(d[q + "_std"][c]) and math.isnan(g[q].std())
            s = np.sort(g[q].to_numpy())
            for p, pm in zip(summary.QUANTILES, PERMILLE):
                assert d[f"{q}_p{p}"][c] == s[(pm * len(s) + 999) // 1000 - 1]
            assert d[q + "_cdf"][c].tolist() == [float((g[q] <= e).mean()) for e in edges]
    assert len(summary.jobdist_flat(d, 0)) == len(summary.jobdist_columns())
    with pytest.raises(ValueError):
        summary.jobdist_derived(classes, hist, edges[:-1])


def _jclasses(specs):
    from gpuschedule_b200.capi import JCLASS_DTYPE
    out = np.zeros(len(specs), dtype=JCLASS_DTYPE)
    for i, d in enumerate(specs):
        for key, v in d.items():
            out[i][key] = v
    return out


def test_jobdist_spread_over_the_replicas_that_have_jobs_in_a_class():
    from gpuschedule_b200 import summary
    R, nc, edges = 5, 2, (10, 20)
    specs, hist = [], np.zeros((R, nc, 3, 3), dtype=np.uint32)
    for r in range(R):
        specs.append(dict(jobs=4, wait_sum=4 * (r + 1), wait_sq_lo=4 * (r + 1) ** 2, jct_sum=40, jct_sq_lo=400, turnaround_sum=8, turnaround_sq_lo=16,
                          wait_q=[r + 1] * 5))
        hist[r, 0, 0] = [min(r, 4), 4 - min(r, 4), 0]
        hist[r, 0, 1] = [4, 0, 0]
        hist[r, 0, 2] = [0, 4, 0]
        if r in (1, 3):                           # class 1: only replicas 1 and 3 have jobs
            specs.append(dict(jobs=1, wait_sum=7 * r, wait_sq_lo=(7 * r) ** 2, wait_q=[7 * r] * 5))
            hist[r, 1, :, 0] = 1
        else:
            specs.append(dict())
    classes = _jclasses(specs).reshape(R, nc)
    sp = summary.jobdist_spread(classes, hist, edges, level=0.8)
    assert sp["replicas"].tolist() == [5, 2]
    means = [float(r + 1) for r in range(R)]
    assert sp["wait_mean"]["mean"][0] == pytest.approx(np.mean(means))
    assert sp["wait_mean"]["std"][0] == pytest.approx(np.std(means, ddof=1))
    ref = summary._spread_of(np.array(means), summary.Fraction("0.8"))
    assert [sp["wait_mean"][s][0] for s in summary.SPREAD_STATS] == pytest.approx([ref[s] for s in summary.SPREAD_STATS])
    assert sp["wait_std"]["mean"][0] == 0.0                          # four equal values per replica
    assert sp["wait_p50"]["lo"][0] == 1.0 and sp["wait_p50"]["hi"][0] == 5.0
    assert sp["wait_mean"]["mean"][1] == pytest.approx(14.0) and sp["wait_mean"]["lo"][1] == 7.0 and sp["wait_mean"]["hi"][1] == 21.0
    assert math.isnan(sp["wait_std"]["mean"][1])                     # one job per replica: NaN std, NaN throughout
    cdf0 = [hist[r, 0, 0, 0] / 4 for r in range(R)]
    assert sp["wait_cdf"]["mean"][0, 0] == pytest.approx(np.mean(cdf0))
    assert sp["jct_cdf"]["mean"][0].tolist() == [0.0, 1.0] and sp["wait_cdf"]["mean"][1].tolist() == [1.0, 1.0]
    assert len(summary.jobdist_spread_flat(sp, 0)) == len(summary.jobdist_spread_columns())
    none = summary.jobdist_spread(_jclasses([dict()] * 2).reshape(2, 1), np.zeros((2, 1, 3, 3), dtype=np.uint32), edges)
    assert none["replicas"].tolist() == [0] and math.isnan(none["wait_mean"]["mean"][0]) and math.isnan(none["jct_cdf"]["hi"][0, 1])
    with pytest.raises(ValueError):
        summary.jobdist_spread(classes[0], hist[0], edges)
    with pytest.raises(ValueError):
        summary.jobdist_spread(classes, hist, edges, level=0)


# ---------------------------------------------------------------- sweep argument errors (before any engine exists)
def test_sweep_jobdist_argument_errors(tmp_path, monkeypatch):
    from gpuschedule_b200 import capi, sweep

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(capi, "Engine", no_engine)
    monkeypatch.setattr(capi, "HorusEngine", no_engine)
    fl = [sweep.make_flags(trace_file=str(tmp_path / "missing.csv"))]
    for bad in (((0,), ()), ((3, 3), ()), ((4, 2), ()), ((1, 2, 3, 4, 5, 6, 7, 8), ()), ((2 ** 31,), ()), ((), (1, 1)), ((), (3, 2)),
                ((), tuple(range(256))), ((), (2 ** 31,)), ((), (-2 ** 31 - 1,)), ((1,),), 5, "ab", ((1,), ("x",))):
        with pytest.raises(ValueError):
            sweep.summarize_batched(fl, jobdist=bad)
        with pytest.raises(ValueError):
            sweep.summarize_bootstrap(fl, 2, jobdist=bad)
    assert sweep.check_jobdist(([5, 17, 65], range(3))) == ((5, 17, 65), (0, 1, 2))
    assert sweep.check_jobdist(((), ())) == ((), ())
    assert sweep.DEFAULT_CDF_EDGES == DEFAULT_EDGES
    base = ["--trace", str(tmp_path / "missing.csv")]
    for argv in (["--jobdist", "j.csv"],                                                      # no --summary
                 ["--summary", "s.csv", "--gpu-classes", "5"], ["--summary", "s.csv", "--cdf-edges", "5"],   # no --jobdist
                 ["--summary", "s.csv", "--jobdist-cdf", "c.csv"],
                 ["--summary", "s.csv", "--jobdist", "j.csv", "--gpu-classes", "0"],
                 ["--summary", "s.csv", "--jobdist", "j.csv", "--gpu-classes", "5", "5"],
                 ["--summary", "s.csv", "--jobdist", "j.csv", "--gpu-classes", "1", "2", "3", "4", "5", "6", "7", "8"],
                 ["--summary", "s.csv", "--jobdist", "j.csv", "--cdf-edges", "3", "2"],
                 ["--summary", "s.csv", "--jobdist", "j.csv", "--cdf-edges"] + [str(i) for i in range(256)],
                 ["--summary", "s.csv", "--jobdist", "j.csv", "--bootstrap", "0"]):
        with pytest.raises(SystemExit) as e:
            sweep.main(base + argv)
        assert e.value.code == 2, argv
    for name in ("j.csv", "s.csv", "c.csv"):
        assert not (tmp_path / name).exists()

"""Job statistics by a chosen key with bounded slowdown (gs_sdclass and CDF counts, gpuschedule_b200/csrc/gs_summary.cuh)
on a box without a GPU.

The __host__ __device__ part -- the key, the class, the slowdown value, the setting's validation -- and gs_sd_serial,
the kernel's steps run serially with the summary's own radix select, are compiled with g++ (tests/emu/slowdown_emu.cpp)
and compared with `reference_slowdown`, a numpy / Python-int restatement of the definitions in include/gsched.h, on the
fixtures' job records and seeded random job sets.  gs_horus_set_slowdown / gs_horus_fetch_slowdown run through the
host-emulation build of gs_horus.cu.  summary.slowdown_derived / slowdown_spread and the sweep's argument errors too."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, REPO, horus_cases, load_horus
from test_jobdist_cpu import DEFAULT_EDGES, FIXTURES, QUANTS, _code, _fixture_jobs, csv_jobs, horus_emu_engine  # noqa: F401
from test_summary_cpu import PERMILLE, job_columns

KEYS = ("gpus", "length", "gpu-time")
SD_MAX = 2 ** 31 - 1
DEFAULT_SD_EDGES = tuple(1024 * 2 ** i for i in range(21))


# ---------------------------------------------------------------- the restatement (shared with test_gpu_slowdown.py)
def sd_values(turn, jct, tau):
    """bounded slowdown in units of 1/1024 as Python ints: min(2^31 - 1, max(1024, floor(1024 * turn / max(jct, tau))))"""
    return [min(SD_MAX, max(1024, (1024 * t) // max(j, tau))) for t, j in zip(turn, jct)]


def job_keys(key, gpus, jct):
    if key == "gpus":
        return [int(g) for g in gpus]
    if key == "length":
        return [int(j) for j in jct]
    return [int(g) * int(j) for g, j in zip(gpus, jct)]


def _q(vals):
    s = sorted(vals)
    k = len(s)
    return [s[(p * k + 999) // 1000 - 1] for p in PERMILLE] if k else [0] * 5


def reference_slowdown(arrive, gpus, start, end, jct, preempt, key, bounds, tau, edges, sd_edges):
    """(per class a dict of gs_sdclass fields -- gs_jclass fields flat, sums of squares and the key sum as exact ints
    "<q>_sq", "key_sum" --, CDF counts (C, 3 * (E + 1) + Esd + 1)) of the finished jobs' columns"""
    cols = [[int(x) for x in np.asarray(a, dtype=np.int64).tolist()] for a in (arrive, gpus, start, end, jct, preempt)]
    arrive, gpus, start, end, jct, preempt = cols
    keys = job_keys(key, gpus, jct)
    cls = [sum(1 for b in bounds if b <= k) for k in keys]
    wait = [s - a for s, a in zip(start, arrive)]
    turn = [e - a for e, a in zip(end, arrive)]
    sd = sd_values(turn, jct, tau)
    vals = dict(wait=wait, turnaround=turn, jct=jct, sd=sd)
    nc, ne, ns = len(bounds) + 1, len(edges), len(sd_edges)
    hist = np.zeros((nc, 3 * (ne + 1) + ns + 1), dtype=np.int64)
    out = []
    for c in range(nc):
        idx = [i for i in range(len(cls)) if cls[i] == c]
        k = len(idx)
        gt = sum(gpus[i] * jct[i] for i in idx) % 2 ** 64         # gs_jclass's int64 gpu_ticks_sum wraps; key_sum is exact
        d = dict(jobs=k, preempt_sum=sum(preempt[i] for i in idx), gpu_ticks_sum=gt - 2 ** 64 if gt >= 2 ** 63 else gt,
                 key_sum=sum(keys[i] for i in idx))
        for m, q in enumerate(QUANTS + ("sd",)):
            v = [vals[q][i] for i in idx]
            d[q + "_sum"] = sum(v)
            d[q + "_sq"] = sum(x * x for x in v)
            d[q + "_q"] = _q(v)
            ed = sd_edges if q == "sd" else edges
            lo = m * (ne + 1)
            for x in v:
                hist[c, lo + sum(1 for e in ed if e < x)] += 1
        d["sd_min"] = min(vals["sd"][i] for i in idx) if k else 0
        d["sd_clamped"] = sum(1 for i in idx if vals["sd"][i] == SD_MAX)
        out.append(d)
    return out, hist


def sdclass_fields(rec):
    """one SDCLASS_DTYPE record as the dict reference_slowdown makes"""
    jc = rec["jc"]
    d = {name: (jc[name].tolist() if jc[name].shape else jc[name].item()) for name in jc.dtype.names}
    for q in QUANTS:
        d[q + "_sq"] = (int(jc[q + "_sq_hi"]) << 64) | int(jc[q + "_sq_lo"])
    d["sd_sum"] = int(rec["sd_sum"])
    d["sd_sq"] = (int(rec["sd_sq_hi"]) << 64) | int(rec["sd_sq_lo"])
    d["sd_q"] = rec["sd_q"].tolist()
    d["sd_min"] = int(rec["sd_min"])
    d["sd_clamped"] = int(rec["sd_clamped"])
    d["key_sum"] = (int(rec["key_sum_hi"]) << 64) | int(rec["key_sum_lo"])
    return d


def assert_slowdown(recs, hist, ref, tag=""):
    want, want_hist = ref
    assert len(recs) == len(want), tag
    for c, (rec, w) in enumerate(zip(recs, want)):
        got = sdclass_fields(rec)
        for key, v in w.items():
            assert got[key] == v, (tag, c, key, got[key], v)
    assert np.array_equal(np.asarray(hist, dtype=np.int64), want_hist), tag


# ---------------------------------------------------------------- host build
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("slowdown_emu") / "libslowdown_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "slowdown_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.emu_sd_key.restype = C.c_longlong
    lib.emu_sd_key.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.emu_sd_class.argtypes = [C.c_void_p, C.c_int, C.c_longlong]
    lib.emu_sd_value.argtypes = [C.c_int, C.c_int, C.c_longlong]
    for name in ("emu_sd_class", "emu_sd_value", "emu_sd_check", "emu_sd_jobs"):
        getattr(lib, name).restype = C.c_int
    return lib


def _p(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def emu_slowdown(lib, jobs, key, bounds, tau, edges, sd_edges, cfg=None):
    """(rc, records, hist) of gs_sd_serial over the job columns (arrive, gpus, start, end, jct, preempt); outputs
    start filled with 0xAB bytes so that an untouched output can be told apart"""
    from gpuschedule_b200 import capi
    cols = [np.ascontiguousarray(c, dtype=np.int32) for c in jobs]
    if cfg is None:
        cfg, keep = capi.slowdown_cfg(key, bounds, tau, edges, sd_edges)
    nc = max(cfg.nclasses, 1)
    row = 3 * (max(cfg.nedges, 0) + 1) + max(cfg.nsd_edges, 0) + 1
    recs = np.frombuffer(b"\xab" * (nc * capi.SDCLASS_DTYPE.itemsize), dtype=capi.SDCLASS_DTYPE).copy()
    hist = np.full((nc, row), 0xABABABAB, dtype=np.uint32)
    rc = lib.emu_sd_jobs(*[_p(c) for c in (cols[0], cols[2], cols[3], cols[4], cols[5], cols[1])], C.c_longlong(len(cols[0])),
                         C.byref(cfg), _p(recs), _p(hist))
    return rc, recs[:cfg.nclasses] if cfg.nclasses > 0 else recs, hist[:cfg.nclasses] if cfg.nclasses > 0 else hist


def check(lib, jobs, key, bounds, tau, edges, sd_edges, tag):
    rc, recs, hist = emu_slowdown(lib, jobs, key, bounds, tau, edges, sd_edges)
    assert rc == 0, tag
    assert_slowdown(recs, hist, reference_slowdown(*jobs, key, bounds, tau, edges, sd_edges), tag)
    # invariants: the classes add up to all jobs; every histogram row sums to its class's jobs
    assert int(recs["jc"]["jobs"].sum()) == len(jobs[0]), tag
    n = recs["jc"]["jobs"].astype(np.int64)
    ne = len(edges) + 1
    for m in range(3):
        assert (hist[:, m * ne:(m + 1) * ne].astype(np.int64).sum(axis=1) == n).all(), tag
    assert (hist[:, 3 * ne:].astype(np.int64).sum(axis=1) == n).all(), tag
    return recs, hist


def test_key_class_and_value(emu):
    for key, code in (("gpus", 0), ("length", 1), ("gpu-time", 2)):
        assert emu.emu_sd_key(code, 8, 3600) == job_keys(key, [8], [3600])[0]
    assert emu.emu_sd_key(2, 2 ** 24 - 1, 2 ** 31 - 1) == (2 ** 24 - 1) * (2 ** 31 - 1)       # above 2^31: int64
    b = np.array([60, 720, 2880, 2 ** 40], dtype=np.int64)
    for k, want in ((0, 0), (59, 0), (60, 1), (719, 1), (720, 2), (2880, 3), (2 ** 40 - 1, 3), (2 ** 40, 4), (2 ** 50, 4)):
        assert emu.emu_sd_class(_p(b), 4, k) == want, k
    assert emu.emu_sd_class(None, 0, 5) == 0
    cases = [(0, 1, 1), (1, 1, 1), (10, 5, 1), (10, 5, 20), (7, 3, 1), (2 ** 31 - 1, 1, 1), (2 ** 21, 1, 1), (2 ** 21 - 1, 1, 1),
             (5, 0, 1), (100, 1, 2 ** 40), (2 ** 31 - 1, 2 ** 31 - 1, 1), (3, 7, 1)]
    for turn, jct, tau in cases:
        assert emu.emu_sd_value(turn, jct, tau) == sd_values([turn], [jct], tau)[0], (turn, jct, tau)
    assert emu.emu_sd_value(2 ** 21, 1, 1) == SD_MAX and emu.emu_sd_value(2 ** 21 - 1, 1, 1) == SD_MAX - 1023


# ---------------------------------------------------------------- fixtures
def settings_for(jobs):
    """(key, bounds, tau, edges, sd_edges) settings that cover: every key, one and eight classes, bounds equal to the
    jobs' own keys, GPU-time bounds above 2^31, tau = 1, tau above every turnaround (every sd = 1024), E = 0 and 255 for
    both edge lists, edges equal to values"""
    arrive, gpus, start, end, jct, _ = (np.asarray(a, dtype=np.int64) for a in jobs)
    turn = end - arrive
    sd = np.array(sd_values(turn.tolist(), jct.tolist(), 1), dtype=np.int64)
    own_len = tuple(int(x) for x in np.unique(jct)[:7])
    big = int(turn.max()) + 1 if len(turn) else 2
    sd_own = tuple(int(x) for x in np.unique(sd)[:255])
    return [("length", (), 1, (), ()), ("length", (60, 720, 2880), 1, DEFAULT_EDGES, DEFAULT_SD_EDGES),
            ("gpus", (2, 4, 8, 16, 32, 64, 128), 10, (0, 10, 100), tuple(range(1024, 1024 + 255 * 16, 16))),
            ("gpu-time", (100, 10 ** 4, 2 ** 31, 2 ** 40), 60, tuple(range(0, 2550, 10)), (1024, 2048)),
            ("length", own_len, big, (1, 4), (1023, 1024, 1025)), ("gpu-time", (1,), 1, (), sd_own)]


@pytest.mark.parametrize("kind,case", FIXTURES)
def test_fixture_slowdown(emu, kind, case):
    jobs = _fixture_jobs(kind, case)
    assert len(jobs[0]) > 0 and int(np.min(jobs[4])) >= 1          # jct >= 1 in every engine's records
    for key, bounds, tau, edges, sd_edges in settings_for(jobs):
        recs, _ = check(emu, jobs, key, bounds, tau, edges, sd_edges, f"{case} {key} bounds={bounds} tau={tau}")
        if tau > int(np.max(np.asarray(jobs[3]) - np.asarray(jobs[0]))):
            assert all(q == 1024 for r in recs if r["jc"]["jobs"] for q in r["sd_q"].tolist())


def test_gpus_key_records_equal_jobdist(emu):
    """with key = gpus and jobdist's bounds and edges, the gs_jclass part is gs_jd_jobs_serial's, byte for byte"""
    from test_jobdist_cpu import emu_jobdist
    out = os.path.join(os.path.dirname(emu._name), "libjobdist_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "jobdist_emu.cpp")], check=True)
    jd = C.CDLL(out)
    jd.emu_jd_jobs.restype = C.c_int
    for kind, case in FIXTURES[:6] + FIXTURES[-3:]:
        jobs = _fixture_jobs(kind, case)
        for bounds, edges in (((), ()), ((5, 17, 65), DEFAULT_EDGES), ((1, 2, 3, 4, 8, 16, 32), (0, 10, 100, 1000))):
            _, recs, hist = emu_slowdown(emu, jobs, "gpus", bounds, 1, edges, DEFAULT_SD_EDGES)
            _, cls, jh = emu_jobdist(jd, jobs, bounds, edges)
            assert recs["jc"].tobytes() == cls.tobytes(), case
            ne = len(edges) + 1
            assert hist[:, :3 * ne].tobytes() == jh.reshape(len(cls), 3 * ne).tobytes(), case


# ---------------------------------------------------------------- seeded random job sets
def test_random_job_sets(emu):
    rng = np.random.default_rng(29)
    for k in (0, 1, 2, 3, 1000, 4000):
        for scale in (10, 2 ** 16, 2 ** 29):
            arrive = rng.integers(0, scale, k)
            start = arrive + rng.integers(0, scale, k)
            jct = rng.integers(1, max(2, scale // 64), k)
            jct[: k // 3] = rng.integers(1, 4, k // 3)                            # ties, and short jobs that saturate
            end = start + jct + rng.integers(0, 3, k)
            gpus = rng.choice([1, 2, 4, 8, 64, 2 ** 20, 2 ** 24 - 1], k)
            preempt = rng.integers(0, 4, k)
            jobs = (arrive, gpus, start, end, jct, preempt)
            for key, bounds, tau in (("length", (), 1), ("length", (60, 720, 2880), 1), ("gpus", (2, 8, 2 ** 20), 5),
                                     ("gpu-time", (2 ** 10, 2 ** 31, 2 ** 33, 2 ** 40, 2 ** 44, 2 ** 48, 2 ** 50), 1),
                                     ("length", (1, 2, 3, 5, 8, 13, 21), scale * 4)):
                recs, _ = check(emu, jobs, key, bounds, tau, DEFAULT_EDGES, DEFAULT_SD_EDGES, f"k={k} scale={scale} {key} tau={tau}")
            if k >= 1000 and scale == 2 ** 29:
                r, _ = check(emu, jobs, "gpu-time", (), 1, (), (), f"k={k} one class")
                assert int(r["sd_clamped"][0]) > 0 and int(r["sd_q"][0][4]) == SD_MAX    # saturation is counted
                assert int(r["sd_sq_hi"][0]) > 0


def test_gpu_time_key_sum_needs_128_bits(emu):
    """600 jobs of (2^24 - 1) GPUs x (2^31 - 1) ticks: a key sum above 2^64"""
    k = 600
    z = np.zeros(k, dtype=np.int64)
    jct = np.full(k, 2 ** 31 - 1, dtype=np.int64)
    jobs = (z, np.full(k, 2 ** 24 - 1, dtype=np.int64), z, jct, jct, z)
    recs, _ = check(emu, jobs, "gpu-time", (2 ** 54, 2 ** 55), 1, (), (), "huge keys")
    assert [int(x) for x in recs["jc"]["jobs"]] == [0, 600, 0] and int(recs["key_sum_hi"][1]) > 0


def test_setting_errors_leave_outputs_untouched(emu):
    from gpuschedule_b200 import capi
    jobs = tuple(np.ones(4, dtype=np.int64) for _ in range(6))
    assert emu_slowdown(emu, jobs, "length", (), 1, (), ())[0] == 0
    bad = []
    for bounds, tau, edges, sd_edges in (((0,), 1, (), ()), ((3, 3), 1, (), ()), ((4, 2), 1, (), ()), ((), 0, (), ()), ((), -5, (), ()),
                                         ((), 1, (1, 1), ()), ((), 1, (5, 2), ()), ((), 1, (), (9, 9)), ((), 1, (), (4, 3))):
        bad.append(capi.slowdown_cfg("length", bounds, tau, edges, sd_edges))
    for mut in ("key", "nclasses_hi", "nclasses_lo", "nedges", "nsd", "null_edges", "null_sd"):
        cfg, keep = capi.slowdown_cfg("length", (), 1, (1, 2), (1024,))
        if mut == "key":
            cfg.key = 3
        elif mut == "nclasses_hi":
            cfg.nclasses = 9
        elif mut == "nclasses_lo":
            cfg.nclasses = -1
        elif mut == "nedges":
            cfg.nedges = 256
        elif mut == "nsd":
            cfg.nsd_edges = 256
        elif mut == "null_edges":
            cfg.edges = None
        else:
            cfg.sd_edges = None
        bad.append((cfg, keep))
    for cfg, keep in bad:
        assert emu.emu_sd_check(C.byref(cfg)) == -1
        rc, recs, hist = emu_slowdown(emu, jobs, None, None, None, None, None, cfg=cfg)
        assert rc == -1
        assert recs.tobytes() == b"\xab" * len(recs.tobytes()) and (hist == 0xABABABAB).all()
    assert emu.emu_sd_check(None) == 0                                       # NULL: off
    with pytest.raises(capi.GsError):
        capi.slowdown_cfg("size", (), 1, (), ())
    with pytest.raises(capi.GsError):
        capi.slowdown_cfg("length", (), 1, (2 ** 31,), ())


# ---------------------------------------------------------------- gs_horus_set_slowdown / gs_horus_fetch_slowdown, host build of gs_horus.cu
def test_horus_slowdown_host_build_matches_reference(horus_emu_engine):
    from gpuschedule_b200 import capi
    cases = horus_cases()
    loaded = [load_horus(c) for c in cases]
    with horus_emu_engine(device=0, nsims=len(cases)) as eng:
        for i, (table, cluster, params, _, _) in enumerate(loaded):
            eng.config(i, cluster, capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"]))
            eng.load_trace(i, table)
            np.random.seed(params["seed"])
            eng.load_words(i, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))
        for bounds, tau, edges, sd_edges in (((0,), 1, (), ()), ((3, 3), 1, (), ()), ((), 0, (), ()), ((), 1, (2, 2), ()), ((), 1, (), (3, 1)),
                                             ((), 1, tuple(range(256)), ()), ((), 1, (), tuple(range(256)))):
            assert _code(eng.set_slowdown, "length", bounds, tau, edges, sd_edges) == capi.GS_ERR_ARG, (bounds, tau)
        assert _code(eng.slowdown) == capi.GS_ERR_STATE                        # off
        eng.set_slowdown("length", (60, 720), 1, DEFAULT_EDGES, DEFAULT_SD_EDGES)
        assert _code(eng.slowdown) == capi.GS_ERR_STATE                        # nothing has run
        eng.run(rows_cap=1 << 15)
        assert _code(eng.slowdown) == capi.GS_ERR_STATE                        # not summarised
        eng.set_slowdown(None)
        plain = eng.summarize()
        eng.set_jobdist((5, 17, 65), DEFAULT_EDGES)                            # both on: each keeps its own state
        for key, bounds, tau, edges, sd_edges in (("length", (60, 720, 2880), 1, DEFAULT_EDGES, DEFAULT_SD_EDGES), ("gpus", (5, 17, 65), 1, DEFAULT_EDGES, ()),
                                                  ("gpu-time", (), 100, (), tuple(range(1024, 1024 * 256, 1024))), ("length", (1, 2, 3, 4, 8, 16, 32), 10 ** 9, (0, 5), (1024,))):
            eng.set_slowdown(key, bounds, tau, edges, sd_edges)
            assert _code(eng.slowdown) == capi.GS_ERR_STATE                    # setting it asks for a new summary
            jd_before = eng.jobdist() if key != "length" or bounds != (60, 720, 2880) else None
            recs_sum = eng.summarize()
            assert recs_sum.tobytes() == plain.tobytes()                       # the summaries do not change
            recs, hist = eng.slowdown()
            assert recs.shape == (len(cases), len(bounds) + 1) and hist.shape == (len(cases), len(bounds) + 1, 3 * (len(edges) + 1) + len(sd_edges) + 1)
            part = eng.slowdown(first=2, count=3)
            assert part[0].tobytes() == recs[2:5].tobytes() and part[1].tobytes() == hist[2:5].tobytes()
            assert _code(eng.slowdown, 3, len(cases)) == capi.GS_ERR_ARG
            assert _code(eng.slowdown, -1, 1) == capi.GS_ERR_ARG
            cls, _ = eng.jobdist()
            if jd_before is not None:
                assert cls.tobytes() == jd_before[0].tobytes()
            for i, (case, (table, _, _, _, _)) in enumerate(zip(cases, loaded)):
                _, _, _, hrecs, order = eng.fetch(i)
                jobs = job_columns(table, hrecs, order)
                assert_slowdown(recs[i], hist[i], reference_slowdown(*jobs, key, bounds, tau, edges, sd_edges), f"{case} {key}")
                assert_slowdown(recs[i], hist[i], reference_slowdown(*csv_jobs(os.path.join(GOLDEN, case, "job.csv"), table), key, bounds, tau,
                                                                     edges, sd_edges), f"{case} job.csv {key}")
                if key == "gpus":
                    assert recs[i]["jc"].tobytes() == cls[i].tobytes()
        eng.set_slowdown(None)
        assert _code(eng.slowdown) == capi.GS_ERR_STATE
        assert eng.jobdist()[0].shape[1] == 4                                  # jobdist is still on


# ---------------------------------------------------------------- summary.slowdown_derived / slowdown_spread
def test_slowdown_derived_matches_pandas(emu):
    import pandas as pd
    from gpuschedule_b200 import summary
    rng = np.random.default_rng(5)
    k = 3000
    arrive = rng.integers(0, 10 ** 6, k)
    start = arrive + rng.integers(0, 2 ** 20, k)
    jct = rng.integers(1, 5000, k)
    jct[0] = 10 ** 6                                          # class 3 (2880+) has ... exactly 1 job: std NaN
    end = start + jct
    gpus = rng.choice([1, 2, 4, 8, 16, 32, 64, 128], k)
    jobs = (arrive, gpus, start, end, jct, np.zeros(k, dtype=np.int64))
    bounds, tau, edges, sd_edges = (60, 720, 5000, 10 ** 7), 30, (10 ** 3, 2 ** 18, 2 ** 20), (1024, 2048, 10240, 102400)
    _, recs, hist = emu_slowdown(emu, jobs, "length", bounds, tau, edges, sd_edges)
    d = summary.slowdown_derived(recs, hist, edges, sd_edges)
    df = pd.DataFrame(dict(wait=start - arrive, turnaround=end - arrive, jct=jct))
    df["sd"] = [v / 1024 for v in sd_values(df["turnaround"].tolist(), df["jct"].tolist(), tau)]
    df["cls"] = pd.cut(df["jct"], [0, 59, 719, 4999, 10 ** 7 - 1, 10 ** 9], labels=False)
    assert d["jobs"].tolist() == [int((df["cls"] == c).sum()) for c in range(5)]
    for c in range(5):
        g = df[df["cls"] == c]
        if len(g) == 0:
            assert math.isnan(d["sd_mean"][c]) and math.isnan(d["key_mean"][c]) and math.isnan(d["sd_cdf"][c, 0])
            continue
        assert math.isclose(d["key_mean"][c], g["jct"].mean(), rel_tol=1e-12)
        assert math.isclose(d["sd_mean"][c], g["sd"].mean(), rel_tol=1e-12)
        if len(g) > 1:
            assert math.isclose(d["sd_std"][c], g["sd"].std(), rel_tol=1e-12), c
            assert math.isclose(d["wait_std"][c], g["wait"].std(), rel_tol=1e-12), c
        else:
            assert math.isnan(d["sd_std"][c]) and math.isnan(g["sd"].std())
        s = np.sort(g["sd"].to_numpy())
        for p, pm in zip(summary.QUANTILES, PERMILLE):
            assert d[f"sd_p{p}"][c] == s[(pm * len(s) + 999) // 1000 - 1]
        assert d["sd_min"][c] == s[0]
        assert d["sd_cdf"][c].tolist() == [float((g["sd"] <= e / 1024).mean()) for e in sd_edges]
        assert d["turnaround_cdf"][c].tolist() == [float((g["turnaround"] <= e).mean()) for e in edges]
    assert len(summary.slowdown_flat(d, 0)) == len(summary.slowdown_columns())
    with pytest.raises(ValueError):
        summary.slowdown_derived(recs, hist, edges, sd_edges[:-1])


def test_slowdown_spread_over_the_replicas_that_have_jobs_in_a_class(emu):
    from gpuschedule_b200 import summary
    rng = np.random.default_rng(11)
    R, bounds, edges, sd_edges = 6, (100,), (10, 1000), (1024, 4096)
    recs, hists = [], []
    for r in range(R):
        k = 50
        arrive = rng.integers(0, 1000, k)
        start = arrive + rng.integers(0, 500, k)
        jct = rng.integers(1, 99, k) if r % 2 else np.concatenate([rng.integers(1, 99, k - 3), [150, 300, 600]])
        end = start + jct
        _, rc, hs = emu_slowdown(emu, (arrive, np.ones(k), start, end, jct, np.zeros(k)), "length", bounds, 1, edges, sd_edges)
        recs.append(rc)
        hists.append(hs)
    recs, hists = np.stack(recs), np.stack(hists)
    sp = summary.slowdown_spread(recs, hists, edges, sd_edges, level=0.9)
    assert sp["replicas"].tolist() == [6, 3]                                  # class 1 only in the even replicas
    per = [summary.slowdown_derived(recs[r], hists[r], edges, sd_edges) for r in range(R)]
    for c, reps in ((0, range(R)), (1, range(0, R, 2))):
        v = np.array([per[r]["sd_mean"][c] for r in reps])
        ref = summary._spread_of(v, summary.Fraction("0.9"))
        assert [sp["sd_mean"][s][c] for s in summary.SPREAD_STATS] == pytest.approx([ref[s] for s in summary.SPREAD_STATS])
        v = np.array([per[r]["sd_cdf"][c, 1] for r in reps])
        assert sp["sd_cdf"]["mean"][c, 1] == pytest.approx(v.mean())
    assert len(summary.slowdown_spread_flat(sp, 0)) == len(summary.slowdown_spread_columns())
    with pytest.raises(ValueError):
        summary.slowdown_spread(recs[0], hists[0], edges, sd_edges)
    with pytest.raises(ValueError):
        summary.slowdown_spread(recs, hists, edges, sd_edges, level=0)


# ---------------------------------------------------------------- sweep argument errors (before any engine exists)
def test_sweep_slowdown_argument_errors(tmp_path, monkeypatch):
    from gpuschedule_b200 import capi, sweep

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(capi, "Engine", no_engine)
    monkeypatch.setattr(capi, "HorusEngine", no_engine)
    fl = [sweep.make_flags(trace_file=str(tmp_path / "missing.csv"))]
    ok = ("length", (), 1, (), ())
    bads = [("size",) + ok[1:], ("length", (0,), 1, (), ()), ("length", (3, 3), 1, (), ()), ("length", tuple(range(1, 9)), 1, (), ()),
            ("length", (2 ** 63,), 1, (), ()), ("length", (), 0, (), ()), ("length", (), 2 ** 63, (), ()), ("length", (), 1, (1, 1), ()),
            ("length", (), 1, tuple(range(256)), ()), ("length", (), 1, (), (5, 2)), ("length", (), 1, (), tuple(range(256))),
            ("length", (), 1, (), (2 ** 31,)), ("length", (), 1, ()), 5, "abcde", ("length", ("x",), 1, (), ())]
    for bad in bads:
        with pytest.raises(ValueError):
            sweep.summarize_batched(fl, slowdown=bad)
        with pytest.raises(ValueError):
            sweep.summarize_bootstrap(fl, 2, slowdown=bad)
    assert sweep.check_slowdown(("gpu-time", [2 ** 40], 60, range(3), [1024])) == ("gpu-time", (2 ** 40,), 60, (0, 1, 2), (1024,))
    assert sweep.DEFAULT_SD_EDGES == DEFAULT_SD_EDGES
    base = ["--trace", str(tmp_path / "missing.csv")]
    for argv in (["--slowdown", "d.csv"],                                                       # no --summary
                 ["--summary", "s.csv", "--job-key", "gpus"], ["--summary", "s.csv", "--key-classes", "5"],   # no --slowdown
                 ["--summary", "s.csv", "--slowdown-bound", "5"], ["--summary", "s.csv", "--slowdown-cdf", "c.csv"],
                 ["--summary", "s.csv", "--sd-edges", "1024"],
                 ["--summary", "s.csv", "--slowdown", "d.csv", "--job-key", "size"],
                 ["--summary", "s.csv", "--slowdown", "d.csv", "--key-classes", "0"],
                 ["--summary", "s.csv", "--slowdown", "d.csv", "--key-classes", "5", "5"],
                 ["--summary", "s.csv", "--slowdown", "d.csv", "--key-classes", "1", "2", "3", "4", "5", "6", "7", "8"],
                 ["--summary", "s.csv", "--slowdown", "d.csv", "--slowdown-bound", "0"],
                 ["--summary", "s.csv", "--slowdown", "d.csv", "--sd-edges", "3", "2"],
                 ["--summary", "s.csv", "--slowdown", "d.csv", "--sd-edges"] + [str(i) for i in range(256)],
                 ["--summary", "s.csv", "--slowdown", "d.csv", "--cdf-edges", "3", "2"],
                 ["--summary", "s.csv", "--slowdown", "d.csv", "--bootstrap", "0"]):
        with pytest.raises(SystemExit) as e:
            sweep.main(base + argv)
        assert e.value.code == 2, argv
    for name in ("d.csv", "s.csv", "c.csv"):
        assert not (tmp_path / name).exists()

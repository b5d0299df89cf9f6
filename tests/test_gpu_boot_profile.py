"""Profiled bootstrap replicas generated on the H100 (gs_boot_profiles / gs_boot_traces_profiled,
sweep.summarize_bootstrap(profile=...)).

Every profiled trace is compared byte for byte with the numpy mirror tracegen.bootstrap_packed(..., profile=...) on a
heterogeneous handle; unprofiled replicas of a profiled launch, a NULL profile and an all -1 profile must be
gs_boot_traces_mixed exactly; profiled arrivals must be arrive_p of the 1/1 replica's; a profiled handle must run and
summarise exactly like the same traces uploaded with gs_load_traces_packed; refused calls change nothing; and the
sweep's profiled path must keep its shapes, pairs, columns and line order."""
import csv
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN
from test_gpu_bootstrap import clusters, make_params, packed_block, policy

pytestmark = pytest.mark.gpu

SURGE = ([(0, 1, 1), (20000, 1, 3), (22000, 1, 1)], 0)
DAILY = ([(0, 5, 3), (480, 5, 7), (1200, 5, 3)], 1440)
LONG = ([(k * 1000, 1 + k % 4, 1 + (k * 7) % 5) for k in range(64)], 64 * 1000 + 17)
PROFILES = [SURGE, DAILY, LONG, ([(0, 1, 2)], 0)]


@pytest.fixture(scope="module")
def pop():
    from gpuschedule_b200 import ingest, tracegen
    return ingest.table_from_columns(tracegen.synth_columns(3000, seed=3))


def mirror(packed, p, L=1, w=None, prof=None):
    from gpuschedule_b200 import tracegen
    return tracegen.bootstrap_packed(packed, int(p["seed"]), int(p["stream"]), int(p["n"]), int(p["gap_num"]), int(p["gap_den"]),
                                     block_len=int(L), weights=w, profile=prof)[0]


def hetero(R):
    """params, block lengths, mixes and profiles of a heterogeneous handle: profiled replicas at 1/1, others scaled"""
    params = make_params(R, ns=(0, 1, 257, 1000, 3000, 7001, 256, 2999), scales=((1, 1), (1, 2), (7, 3)))
    Ls = np.array([(1, 16)[(i // 2) % 2] for i in range(R)], dtype=np.uint32)
    mix = np.array([(-1, 0, 1)[(i // 3) % 3] for i in range(R)], dtype=np.int32)
    prof = np.array([(-1, 0, 1, 2, 3)[i % 5] for i in range(R)], dtype=np.int32)
    params["gap_num"][prof >= 0] = 1
    params["gap_den"][prof >= 0] = 1
    return params, Ls, mix, prof


def mixes(table):
    from gpuschedule_b200 import tracegen
    return np.stack([np.full(table.n, 2, dtype=np.uint32), tracegen.class_weights(table.gpus, (2, 8), (1, 0, 5))])


def test_fetch_trace_equals_mirror_heterogeneous(pop):
    from gpuschedule_b200 import capi
    R = 120
    params, Ls, mix, prof = hetero(R)
    W = mixes(pop)
    shapes = clusters()
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, shapes[i % 2])
        eng.boot_population(pop)
        eng.boot_mixes(W)
        eng.boot_profiles(PROFILES)
        before = eng.launch_count()
        ms = eng.boot_traces(params, with_time=True, block_len=Ls, mix=mix, profile=prof)
        assert ms > 0 and eng.launch_count() - before == 1
        got = [eng.fetch_trace(i) for i in range(R)]
        for i in range(R):
            want = mirror(pop.packed(), params[i], Ls[i], None if mix[i] < 0 else W[mix[i]], None if prof[i] < 0 else PROFILES[prof[i]])
            assert got[i].tobytes() == want.tobytes(), (i, int(Ls[i]), int(mix[i]), int(prof[i]))
        # the unprofiled replicas of that launch are those of gs_boot_traces_mixed
        eng.boot_traces(params, block_len=Ls, mix=mix)
        for i in np.flatnonzero(prof < 0):
            assert eng.fetch_trace(i).tobytes() == got[i].tobytes(), i
        # profiled arrivals are arrive_p of the 1/1 replica's arrivals, every other field unchanged
        from gpuschedule_b200 import tracegen
        ones = params.copy()
        ones["gap_num"] = ones["gap_den"] = 1
        eng.boot_traces(ones, block_len=Ls, mix=mix)
        for i in np.flatnonzero(prof >= 0):
            base = eng.fetch_trace(i)
            for f in ("gpus", "gpu_per_task", "ps_count", "mem_bytes", "duration"):
                assert np.array_equal(base[f], got[i][f])
            arr = tracegen.profile_arrive(base["arrive_tick"].astype(np.int64), *PROFILES[prof[i]])
            assert arr.tolist() == got[i]["arrive_tick"].tolist(), i
        # a new population keeps the profiles
        eng.boot_population(pop.packed()[:500].copy())
        eng.boot_traces(params, block_len=Ls, profile=prof)
        for i in range(0, R, 7):
            want = mirror(pop.packed()[:500].copy(), params[i], Ls[i], None, None if prof[i] < 0 else PROFILES[prof[i]])
            assert eng.fetch_trace(i).tobytes() == want.tobytes(), i


def test_null_and_all_minus_one_are_the_mixed_call(pop):
    from gpuschedule_b200 import capi
    lib = capi.load_library()
    R = 20
    params = make_params(R, ns=(0, 1, 257, 2000), scales=((1, 1), (7, 3)), seed=4)
    minus = np.full(R, -1, dtype=np.int32)
    mix = np.array([(-1, 0, 1)[i % 3] for i in range(R)], dtype=np.int32)
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, clusters()[i % 2])
        eng.boot_population(pop)
        eng.boot_mixes(mixes(pop))
        eng.boot_profiles(PROFILES)
        p = params.ctypes.data_as(C.c_void_p)
        for Ls in (None, np.array([(1, 16, 300)[i % 3] for i in range(R)], dtype=np.uint32)):
            lp = None if Ls is None else Ls.ctypes.data_as(C.c_void_p)
            for mp in (None, mix.ctypes.data_as(C.c_void_p)):
                got = {}
                for name, call in (("mixed", lambda: lib.gs_boot_traces_mixed(eng.h, p, lp, mp, None)),
                                   ("null", lambda: lib.gs_boot_traces_profiled(eng.h, p, lp, mp, None, None)),
                                   ("minus", lambda: lib.gs_boot_traces_profiled(eng.h, p, lp, mp, minus.ctypes.data_as(C.c_void_p), None))):
                    eng._n = [int(k) for k in params["n"].tolist()]
                    before = eng.launch_count()
                    assert call() == capi.GS_OK
                    got[name] = (eng.launch_count() - before, [eng.fetch_trace(i).tobytes() for i in range(R)])
                assert got["mixed"][0] == 1
                assert got["null"] == got["mixed"] and got["minus"] == got["mixed"]


@pytest.mark.parametrize("name", ["fifo", "dlas-gpu"])
def test_profiled_handle_runs_like_uploaded_traces(pop, name):
    from gpuschedule_b200 import capi
    R = 24
    params = make_params(R, ns=(600, 1500, 2500), scales=((1, 1),), seed=8)
    Ls = np.array([(1, 16)[i % 2] for i in range(R)], dtype=np.uint32)
    prof = np.array([(-1, 0, 1, 2)[i % 4] for i in range(R)], dtype=np.int32)
    profiles = [([(0, 1, 1), (3000, 1, 3), (6000, 1, 1)], 0), DAILY, LONG]
    traces = [mirror(pop.packed(), params[i], Ls[i], None, None if prof[i] < 0 else profiles[prof[i]]) for i in range(R)]
    shapes = clusters()
    pol = policy(name, pop)
    with capi.Engine(device=0, nsims=R) as gen, capi.Engine(device=0, nsims=R) as ref:
        for i in range(R):
            gen.config(i, shapes[i % 2], pol)
            ref.config(i, shapes[i % 2], pol)
        gen.boot_population(pop)
        gen.boot_profiles(profiles)
        gen.boot_traces(params, block_len=Ls, profile=prof)
        ref.load_traces_packed(*packed_block(traces))
        for eng in (gen, ref):
            eng.set_timeline(500, 64)
        a, b = gen.run_summarized(rows_cap=1 << 14), ref.run_summarized(rows_cap=1 << 14)
        assert a.tobytes() == b.tobytes()
        assert a["done"].all() and (a["finished"] > 0).any()
        assert gen.timeline().tobytes() == ref.timeline().tobytes()


def test_refused_calls_change_nothing(pop):
    from gpuschedule_b200 import capi
    lib = capi.load_library()
    R = 8
    params = make_params(R, ns=(500, 1000), scales=((1, 1),), seed=2)
    prof = np.array([0, 1, -1, 0, 1, -1, 0, 1], dtype=np.int32)
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, clusters()[0])
        eng.boot_population(pop)
        eng.boot_profiles([SURGE, DAILY])
        eng.boot_traces(params, profile=prof)
        before = [eng.fetch_trace(i).tobytes() for i in range(R)]
        seg = lambda rows: np.array([(t, n, d, 0) for t, n, d in rows], dtype=np.int32).view(capi.BOOT_SEG_DTYPE).reshape(-1)
        one = np.array([1], dtype=np.int32)
        zero = np.array([0], dtype=np.int32)
        ok = seg([(0, 1, 1)])
        bad_profiles = [(-1, one, zero, ok), (1, None, zero, ok), (1, one, None, ok), (1, one, zero, None),
                        (1, np.array([0], np.int32), zero, ok), (1, np.array([65], np.int32), zero, seg([(k, 1, 1) for k in range(65)])),
                        (1, one, zero, seg([(1, 1, 1)])), (2, np.array([1, 2], np.int32), np.zeros(2, np.int32), seg([(0, 1, 1), (0, 1, 1), (0, 1, 1)])),
                        (1, np.array([2], np.int32), zero, seg([(0, 1, 1), (2 ** 31 - 1, 1, 1)])), (1, one, zero, seg([(0, 0, 1)])),
                        (1, one, zero, seg([(0, 1, 0)])), (1, one, np.array([-1], np.int32), ok),
                        (1, np.array([2], np.int32), np.array([10], np.int32), seg([(0, 1, 1), (10, 1, 1)]))]
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        for nprof, nseg, per, segs in bad_profiles:
            assert lib.gs_boot_profiles(eng.h, nprof, ptr(nseg), ptr(per), ptr(segs)) == capi.GS_ERR_ARG, (nprof, nseg, per)
        # the profiles are still SURGE and DAILY: the same call gives the same bytes
        eng.boot_traces(params, profile=prof)
        assert [eng.fetch_trace(i).tobytes() for i in range(R)] == before
        p = params.ctypes.data_as(C.c_void_p)
        for bad in (np.array([2] + [0] * 7, np.int32), np.array([-2] + [0] * 7, np.int32)):
            assert lib.gs_boot_traces_profiled(eng.h, p, None, None, bad.ctypes.data_as(C.c_void_p), None) == capi.GS_ERR_ARG
        scaled = params.copy()
        scaled["gap_den"][0] = 2
        assert lib.gs_boot_traces_profiled(eng.h, scaled.ctypes.data_as(C.c_void_p), None, None, prof.ctypes.data_as(C.c_void_p), None) == capi.GS_ERR_ARG
        big = params.copy()                                   # a surge at 1/1 of 3000-job gaps cannot fit 2^31 - 1 with this n
        big["n"][0] = 2 ** 31 - 100
        assert lib.gs_boot_traces_profiled(eng.h, big.ctypes.data_as(C.c_void_p), None, None, prof.ctypes.data_as(C.c_void_p), None) == capi.GS_ERR_ARG
        assert [eng.fetch_trace(i).tobytes() for i in range(R)] == before
        eng.boot_profiles([])                                 # nprof = 0 clears them
        with pytest.raises(capi.GsError) as e:
            eng.boot_traces(params, profile=prof)
        assert e.value.code == capi.GS_ERR_ARG


def test_summarize_bootstrap_with_profiles():
    from gpuschedule_b200 import capi, sweep
    trace = os.path.join(GOLDEN, "kat0", "trace.csv")
    sets = [sweep.make_flags(trace_file=trace, schedule=s) for s in ("fifo", "dlas-gpu")]
    profs = [(((0, 1.0),), 0), (((0, 1.0), (200, 3.0), (400, 1.0)), 0), (((0, 0.5), (100, 1.5)), 300)]
    loads, R = [1.0, 1.5], 3
    recs, bins, (prec, phist) = sweep.summarize_bootstrap(sets, R, loads, seed=5, timeline=(100, 16), compare=([(0, 1)], (4,), (-10, 0, 10)),
                                                          profile=profs)
    assert recs.shape == (2, 2, 3, R) and bins.shape == (2, 2, 3, R, 16)
    assert prec.shape == (1, 2, 3, R, 2)
    plain, pbins, (pp, ph) = sweep.summarize_bootstrap(sets, R, loads, seed=5, timeline=(100, 16), compare=([(0, 1)], (4,), (-10, 0, 10)))
    # a one-segment factor-1 profile is the unprofiled run
    assert recs[:, :, 0].tobytes() == plain.tobytes()
    assert bins[:, :, 0].tobytes() == pbins.tobytes()
    assert prec[:, :, 0].tobytes() == pp.tobytes() and phist[:, :, 0].tobytes() == ph.tobytes()
    assert recs["done"].all()
    # compare pairs within a profile: each profile's pair is the pair of that profile alone
    for q in range(3):
        one = sweep.summarize_bootstrap(sets, R, loads, seed=5, compare=([(0, 1)], (4,), (-10, 0, 10)), profile=[profs[q]])
        assert one[0][:, :, 0].tobytes() == recs[:, :, q].tobytes()
        assert one[1][0][:, :, 0].tobytes() == prec[:, :, q].tobytes()
    mixed = sweep.summarize_bootstrap(sets, R, loads, seed=5, mix=((4,), [(1, 1), (1, 3)]), profile=profs)
    assert mixed.shape == (2, 2, 2, 3, R)


def test_cli_profile_column(tmp_path):
    from gpuschedule_b200 import sweep
    trace = os.path.join(GOLDEN, "kat0", "trace.csv")
    out, tl = str(tmp_path / "s.csv"), str(tmp_path / "t.csv")
    specs = ["0:1", "0:1,200:3,400:1", "0:0.5,100:1.5@300"]
    sweep.main(["--trace", trace, "--schedule", "fifo", "dlas-gpu", "--summary", out, "--bootstrap", "2", "--load", "1", "1.5",
                "--load-profile", *specs, "--timeline", tl, "--bin-width", "100", "--bins", "8"])
    with open(out, newline="") as f:
        rows = list(csv.reader(f))
    head = rows[0]
    assert head[:3] == ["replica", "load", "profile"]
    keys = [(r[1], r[2]) for r in rows[1:]]
    assert len(keys) == 2 * 2 * 3 * 2
    per_conf = keys[:12]
    assert per_conf == [(L, p) for L in ("1.0", "1.5") for p in specs for _ in range(2)]
    with open(tl, newline="") as f:
        trows = list(csv.reader(f))
    at = trows[0].index("load")
    assert trows[0][at + 1] == "profile"
    plain = str(tmp_path / "p.csv")
    sweep.main(["--trace", trace, "--schedule", "fifo", "dlas-gpu", "--summary", plain, "--bootstrap", "2", "--load", "1", "1.5"])
    with open(plain, newline="") as f:
        prow = list(csv.reader(f))
    assert prow[0] == head[:2] + head[3:]
    assert [r[:2] + r[3:] for r in rows[1:] if r[2] == "0:1"] == prow[1:]

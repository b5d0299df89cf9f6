"""Mixed bootstrap replicas generated on the H100 (gs_boot_mixes / gs_boot_traces_mixed,
sweep.summarize_bootstrap(mix=...)).

Every mixed trace is compared byte for byte with the numpy mirror tracegen.bootstrap_packed(..., weights=w); a NULL or
all -1 mix must be gs_boot_traces_blocked exactly, and a uniform mix the unweighted replica; a handle that generates
mixed traces must compute exactly what a handle computes when it is given the mirror's traces through
gs_load_traces_packed (summaries, timelines, job statistics and paired comparisons); refused calls change nothing;
and the sweep's mixed path must return the records of the ordinary path run on bootstrap_table's weighted replicas."""
import csv
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN
from test_gpu_bootstrap import clusters, compare_handles, make_params, packed_block, policy

pytestmark = pytest.mark.gpu

LMAX = 2 ** 32 - 1
WMAX = 2 ** 32 - 1


@pytest.fixture(scope="module")
def pop():
    from gpuschedule_b200 import ingest, tracegen
    return ingest.table_from_columns(tracegen.synth_columns(3000, seed=3))


def make_mixes(table):
    """four mixes of the population: uniform, by size class, random with zeros, and one row"""
    from gpuschedule_b200 import tracegen
    k = table.n
    rng = np.random.default_rng(5)
    by_class = tracegen.class_weights(table.gpus, (2, 5, 17), (0, 1, 3, WMAX))
    assert by_class.any()
    rand = rng.integers(0, 4, size=k).astype(np.uint32)
    one = np.zeros(k, dtype=np.uint32)
    one[k // 3] = 2
    return np.stack([np.full(k, 9, dtype=np.uint32), by_class, rand, one])


def mirror(packed, p, L=1, w=None):
    from gpuschedule_b200 import tracegen
    return tracegen.bootstrap_packed(packed, int(p["seed"]), int(p["stream"]), int(p["n"]), int(p["gap_num"]), int(p["gap_den"]),
                                     block_len=int(L), weights=w)[0]


def test_fetch_trace_equals_mirror_heterogeneous(pop):
    from gpuschedule_b200 import capi
    R = 100
    params = make_params(R, ns=(0, 1, 257, 1000, 3000, 7001, 256, 2999), scales=((1, 1), (1, 2), (2, 1), (7, 3), (0, 1)))
    Ls = np.array([(1, 16, LMAX)[i % 3] for i in range(R)], dtype=np.uint32)
    mix = np.array([(-1, 0, 1, 2, 3)[i % 5] for i in range(R)], dtype=np.int32)
    W = make_mixes(pop)
    shapes = clusters()
    max_need = int(max(1.0, float(pop.duration.max()))) + 2
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, shapes[i % 2])
        eng.boot_population(pop)
        eng.boot_mixes(W)
        before = eng.launch_count()
        ms = eng.boot_traces(params, with_time=True, block_len=Ls, mix=mix)
        assert ms > 0 and eng.launch_count() - before == 1
        want = [mirror(pop.packed(), params[i], Ls[i], None if mix[i] < 0 else W[mix[i]]) for i in range(R)]
        for i in range(R):
            assert eng.fetch_trace(i).tobytes() == want[i].tobytes(), (i, int(Ls[i]), int(mix[i]))
        eng.run(max_ticks=1, rows_cap=0)
        for i in range(R):
            lay, w, M = eng.result_layout(i), want[i], shapes[i % 2].n_nodes
            last = int(w["arrive_tick"][-1]) if len(w) else 0
            assert lay.cap_ev == last + 2 * max_need + 4096, i                # last arrival tick from the kernel
            assert lay.cap_spans == max(int(np.minimum(w["gpus"] // w["gpu_per_task"], M).sum()), 1), i
        iid_only = np.where(mix >= 0, mix, 0).astype(np.int32)               # the iid mixed instantiation alone
        eng.boot_traces(params, mix=iid_only)
        for i in range(R):
            assert eng.fetch_trace(i).tobytes() == mirror(pop.packed(), params[i], 1, W[iid_only[i]]).tobytes(), i
        one = pop.packed()[17:18].copy()                                      # a new population clears the mixes
        one["arrive_tick"] = 0
        eng.boot_population(one)
        with pytest.raises(capi.GsError) as e:
            eng.boot_traces(params, mix=mix)
        assert e.value.code == capi.GS_ERR_ARG
        eng.boot_mixes(np.full((2, 1), 3, dtype=np.uint32))
        eng.boot_traces(params, block_len=Ls, mix=np.array([(-1, 0, 1)[i % 3] for i in range(R)], dtype=np.int32))
        for i in range(R):
            got = eng.fetch_trace(i)
            assert got.tobytes() == mirror(one, params[i], Ls[i]).tobytes(), i
            assert (got["arrive_tick"] == 0).all() and (got["gpus"] == one["gpus"][0]).all()


def test_null_and_all_minus_one_are_the_blocked_call(pop):
    from gpuschedule_b200 import capi
    lib = capi.load_library()
    R = 20
    params = make_params(R, ns=(0, 1, 257, 2000), scales=((1, 1), (7, 3)), seed=4)
    minus = np.full(R, -1, dtype=np.int32)
    W = make_mixes(pop)
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, clusters()[i % 2])
        eng.boot_population(pop)
        eng.boot_mixes(W)
        p = params.ctypes.data_as(C.c_void_p)
        for Ls in (None, np.array([(1, 16, 300)[i % 3] for i in range(R)], dtype=np.uint32)):
            lp = None if Ls is None else Ls.ctypes.data_as(C.c_void_p)
            got = {}
            for name, call in (("blocked", lambda: lib.gs_boot_traces_blocked(eng.h, p, lp, None)),
                               ("null", lambda: lib.gs_boot_traces_mixed(eng.h, p, lp, None, None)),
                               ("minus", lambda: lib.gs_boot_traces_mixed(eng.h, p, lp, minus.ctypes.data_as(C.c_void_p), None))):
                eng._n = [int(k) for k in params["n"].tolist()]
                before = eng.launch_count()
                assert call() == capi.GS_OK
                got[name] = (eng.launch_count() - before, [eng.fetch_trace(i).tobytes() for i in range(R)])
            assert got["blocked"][0] == 1
            assert got["null"] == got["blocked"] and got["minus"] == got["blocked"]
            Lr = np.ones(R, dtype=np.uint32) if Ls is None else Ls
            assert got["blocked"][1] == [mirror(pop.packed(), params[i], Lr[i]).tobytes() for i in range(R)]
            eng.boot_traces(params, block_len=Ls, mix=0)                       # the uniform mix: the unweighted bytes
            assert [eng.fetch_trace(i).tobytes() for i in range(R)] == got["blocked"][1]


@pytest.mark.parametrize("name", ["fifo", "sjf", "dlas-gpu", "gittins"])
def test_mixed_handle_runs_like_packed_upload(pop, name):
    """summaries, a timeline, job statistics and the paired comparison of replicas that share a trace"""
    from gpuschedule_b200 import capi
    H = 12
    R = 2 * H                                                                # replica i + H repeats replica i on the other cluster
    params = make_params(H, ns=(1500, 700, 2000, 1), scales=((1, 1), (1, 2), (3, 2)), seed=5)
    params = np.concatenate([params, params])
    shapes = clusters()
    pol = policy(name, pop)
    W = make_mixes(pop)
    bounds, edges = (2, 8), (0, 100, 10000)
    with capi.Engine(device=0, nsims=R) as gen, capi.Engine(device=0, nsims=R) as ref:
        for i in range(R):
            gen.config(i, shapes[(i // H + i) % 2], pol)
            ref.config(i, shapes[(i // H + i) % 2], pol)
        gen.boot_population(pop)
        gen.boot_mixes(W)
        results = []
        for Ls, mix in ((None, np.array([(1, 2, 3, -1)[i % 4] for i in range(R)], dtype=np.int32)),
                        (np.array([(16, 1, 300)[i % 3] for i in range(R)], dtype=np.uint32), np.int32(1))):
            gen.boot_traces(params, block_len=Ls, mix=mix)
            Lr = np.broadcast_to(1 if Ls is None else Ls, (R,))
            Mr = np.broadcast_to(mix, (R,))
            block, pitch, n_each = packed_block([mirror(pop.packed(), params[i], Lr[i], None if Mr[i] < 0 else W[Mr[i]]) for i in range(R)])
            ref.load_traces_packed(block, pitch, n_each)
            for eng in (gen, ref):
                eng.set_timeline(500, 64)
                eng.set_jobdist(bounds, edges)
            first = compare_handles(gen, ref, name, R)
            assert gen.timeline().tobytes() == ref.timeline().tobytes()
            for x, y in zip(gen.jobdist(), ref.jobdist()):
                assert x.tobytes() == y.tobytes()
            a, b = np.arange(H), np.arange(H) + H
            for x, y in zip(gen.compare(a, b, bounds, edges), ref.compare(a, b, bounds, edges)):
                assert x.tobytes() == y.tobytes()
            results.append(first)
        assert results[0].tobytes() != results[1].tobytes()                  # another mix gave other traces


def test_refused_calls_change_nothing(pop):
    from gpuschedule_b200 import capi
    lib = capi.load_library()
    R = 4
    good = make_params(R, ns=(400,), scales=((1, 1),), seed=2)
    W = make_mixes(pop)
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, clusters()[0])
        wp = W.ctypes.data_as(C.c_void_p)
        assert lib.gs_boot_mixes(eng.h, 4, wp) == capi.GS_ERR_STATE        # no population yet
        assert lib.gs_boot_mixes(eng.h, 0, None) == capi.GS_ERR_STATE
        eng.boot_population(pop)
        eng.boot_mixes(W)
        eng.boot_traces(good, mix=np.array([0, 1, 2, 3], dtype=np.int32))
        before = [eng.fetch_trace(i).tobytes() for i in range(R)]
        zero_row = W.copy()
        zero_row[2] = 0
        assert lib.gs_boot_mixes(eng.h, -1, wp) == capi.GS_ERR_ARG
        assert lib.gs_boot_mixes(eng.h, 2, None) == capi.GS_ERR_ARG
        assert lib.gs_boot_mixes(eng.h, 4, zero_row.ctypes.data_as(C.c_void_p)) == capi.GS_ERR_ARG
        for mix in ([0, 1, 2, 4], [-2, 0, 0, 0], [0, 0, 0, 2 ** 31 - 1]):
            with pytest.raises(capi.GsError) as e:
                eng.boot_traces(good, mix=np.array(mix, dtype=np.int32))
            assert e.value.code == capi.GS_ERR_ARG
        with pytest.raises(capi.GsError) as e:                               # the block length is checked first, as before
            eng.boot_traces(good, block_len=np.array([1, 0, 1, 1]), mix=np.array([0, 9, 0, 0], dtype=np.int32))
        assert e.value.code == capi.GS_ERR_ARG and "block_len" in str(e.value)
        for bad in (1.5, [0, 0], 2 ** 31):
            with pytest.raises(ValueError):
                eng.boot_traces(good, mix=bad)
        with pytest.raises(ValueError):
            eng.boot_mixes(W[:, :-1])
        assert [eng.fetch_trace(i).tobytes() for i in range(R)] == before      # refused calls changed nothing
        eng.boot_traces(good, mix=np.array([0, 1, 2, 3], dtype=np.int32))       # the tables are the ones uploaded first
        assert [eng.fetch_trace(i).tobytes() for i in range(R)] == before
        assert before[3] == mirror(pop.packed(), good[3], 1, W[3]).tobytes()
        assert eng.run_summarized()["done"].all()
        eng.boot_mixes(np.zeros((0, pop.n), dtype=np.uint32))                   # nmix = 0 clears the tables
        with pytest.raises(capi.GsError):
            eng.boot_traces(good, mix=0)
        eng.boot_traces(good, mix=-1)
        assert eng.fetch_trace(1).tobytes() == mirror(pop.packed(), good[1]).tobytes()


def test_summarize_bootstrap_mix_equals_the_ordinary_path():
    from gpuschedule_b200 import capi, sweep, tracegen
    trace = os.path.join(GOLDEN, "n64", "trace.csv")
    flag_sets = [sweep.make_flags(trace_file=trace, schedule=s, num_queue=2) for s in ("fifo", "sjf", "dlas-gpu", "gittins")]
    loads, R, seed, n = (1.0, 2.0), 2, 7, 150
    base = sweep._plain_setup(flag_sets[:1])[0][2].table
    bounds = (int(np.median(base.gpus)) + 1,)
    mults = [(1, 1), (1, 4), (3, 0)]
    for L in (1, 8):
        recs = sweep.summarize_bootstrap(flag_sets, R, loads, seed=seed, n=n, block_len=L, mix=(bounds, mults))
        assert recs.shape == (len(flag_sets), len(loads), len(mults), R)
        for c, (fl, infra, jm, pol) in enumerate(sweep._plain_setup(flag_sets)):
            for li, load in enumerate(loads):
                num, den = sweep.load_gap_scale(load)
                for m, mult in enumerate(mults):
                    w = tracegen.class_weights(jm.table.gpus, bounds, mult)
                    for r in range(R):
                        table = tracegen.bootstrap_table(jm.table, seed, r, n, num, den, block_len=L, weights=w)
                        with capi.Engine(device=0, nsims=1) as eng:
                            eng.config(0, infra.gs_cluster(), pol)
                            eng.load_trace(0, table)
                            want = eng.run_summarized()
                        assert recs[c, li, m, r].tobytes() == want[0].tobytes(), (fl.schedule, load, mult, r, L)
        assert (recs["finished"] > 0).all()
        plain = sweep.summarize_bootstrap(flag_sets, R, loads, seed=seed, n=n, block_len=L)
        assert recs[:, :, 0].tobytes() == plain.tobytes()                     # the uniform mix is the unweighted bootstrap


def test_summarize_bootstrap_mix_shapes_and_compare():
    from gpuschedule_b200 import sweep
    trace = os.path.join(GOLDEN, "n64", "trace.csv")
    flag_sets = [sweep.make_flags(trace_file=trace, schedule=s, num_queue=2) for s in ("fifo", "dlas-gpu")]
    loads, R, n = (1.0, 1.5), 3, 120
    mix = ((4,), [(1, 1), (1, 5)])
    recs, tl, (cls, hist), (prec, phist) = sweep.summarize_bootstrap(flag_sets, R, loads, seed=3, n=n, timeline=(500, 16),
                                                                     jobdist=((4,), (0, 1000)), compare=([(0, 1)], (4,), (0,)), mix=mix)
    assert recs.shape == (2, 2, 2, R) and tl.shape == (2, 2, 2, R, 16)
    assert cls.shape == (2, 2, 2, R, 2) and hist.shape == (2, 2, 2, R, 2, 3, 3)
    assert prec.shape == (1, 2, 2, R, 2) and phist.shape == (1, 2, 2, R, 2, 3, 2)
    assert (prec["jobs"].sum(axis=-1) == n).all()                            # (a, L, mix, r) and (b, L, mix, r) share a trace
    assert (cls["jobs"].sum(axis=-1) == n).all()
    plain = sweep.summarize_bootstrap(flag_sets, R, loads, seed=3, n=n, timeline=(500, 16), jobdist=((4,), (0, 1000)),
                                      compare=([(0, 1)], (4,), (0,)))
    assert plain[0].tobytes() == recs[:, :, 0].tobytes() and plain[1].tobytes() == tl[:, :, 0].tobytes()
    assert plain[3][0].tobytes() == prec[:, :, 0].tobytes()
    with pytest.raises(ValueError):
        sweep.summarize_bootstrap(flag_sets, R, loads, n=n, mix=((10 ** 6,), [(1, 1), (0, 1)]))


def test_sweep_cli_mix(tmp_path):
    """the README example, shrunk: fifo vs dlas-gpu at load 1.2 under two mixes, with job statistics and paired output"""
    from gpuschedule_b200 import sweep
    trace = os.path.join(GOLDEN, "n64", "trace.csv")
    out, ci, jd, pr, ps = (str(tmp_path / f) for f in ("s.csv", "ci.csv", "jd.csv", "p.csv", "ps.csv"))
    sweep.main(["--trace", trace, "--schedule", "fifo", "dlas-gpu", "--bootstrap", "4", "--load", "1.2", "--jobs", "100",
                "--mix", "1:1:1:1", "1:1:1:4", "--mix-classes", "2", "5", "17", "--jobdist", jd, "--gpu-classes", "2", "5", "17",
                "--summary", out, "--summary-ci", ci, "--compare", "fifo", "--paired", pr, "--paired-summary", ps])
    for path, lines in ((out, 2 * 2 * 4), (ci, 2 * 2), (jd, 2 * 2 * 4), (pr, 2 * 4 * 3), (ps, 2)):
        with open(path) as f:
            rows = list(csv.reader(f))
        head = rows[0]
        assert head[head.index("load") + 1] == "mix" and len(rows) == 1 + lines, path
        assert {r[head.index("mix")] for r in rows[1:]} == {"1:1:1:1", "1:1:1:4"}
    with open(ci) as f:
        rows = list(csv.DictReader(f))
    assert [(r["schedule"], r["mix"]) for r in rows] == [("fifo", "1:1:1:1"), ("fifo", "1:1:1:4"),
                                                          ("dlas-gpu", "1:1:1:1"), ("dlas-gpu", "1:1:1:4")]

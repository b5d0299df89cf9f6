"""Block bootstrap replicas generated on the H100 (gs_boot_traces_blocked, sweep.summarize_bootstrap(block_len=L)).

Every blocked trace is compared byte for byte with the numpy mirror tracegen.bootstrap_packed(..., block_len=L); NULL
and all-ones block lengths must be gs_boot_traces exactly; a handle that generates blocked traces must compute exactly
what a handle computes when it is given the mirror's traces through gs_load_traces_packed; a zero block length is
refused without changing anything; and the sweep's blocked path must return the records of the ordinary path run on
bootstrap_table's blocked replicas."""
import csv
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN
from test_gpu_bootstrap import clusters, compare_handles, make_params, packed_block, policy

pytestmark = pytest.mark.gpu

LMAX = 2 ** 32 - 1


@pytest.fixture(scope="module")
def pop():
    from gpuschedule_b200 import ingest, tracegen
    return ingest.table_from_columns(tracegen.synth_columns(3000, seed=3))


def mirror(packed, p, L):
    from gpuschedule_b200 import tracegen
    return tracegen.bootstrap_packed(packed, int(p["seed"]), int(p["stream"]), int(p["n"]), int(p["gap_num"]), int(p["gap_den"]),
                                     block_len=int(L))[0]


def test_fetch_trace_equals_mirror_mixed_handle(pop):
    from gpuschedule_b200 import capi
    R = 96
    params = make_params(R, ns=(0, 1, 257, 1000, 3000, 7001, 256, 2999), scales=((1, 1), (1, 2), (2, 1), (7, 3), (0, 1)))
    Ls = np.array([(1, 2, 3, 16, 1000, LMAX, 32)[i % 7] for i in range(R)], dtype=np.uint32)
    shapes = clusters()
    max_need = int(max(1.0, float(pop.duration.max()))) + 2
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, shapes[i % 2])
        eng.boot_population(pop)
        ms = eng.boot_traces(params, with_time=True, block_len=Ls)
        assert ms > 0
        want = [mirror(pop.packed(), params[i], Ls[i]) for i in range(R)]
        for i in range(R):
            assert eng.fetch_trace(i).tobytes() == want[i].tobytes(), (i, int(Ls[i]))
        eng.run(max_ticks=1, rows_cap=0)
        for i in range(R):
            lay, w, M = eng.result_layout(i), want[i], shapes[i % 2].n_nodes
            last = int(w["arrive_tick"][-1]) if len(w) else 0
            assert lay.cap_ev == last + 2 * max_need + 4096, i                # last arrival tick from the kernel
            assert lay.cap_spans == max(int(np.minimum(w["gpus"] // w["gpu_per_task"], M).sum()), 1), i
        one = pop.packed()[17:18].copy()                                      # a population of K = 1
        one["arrive_tick"] = 0
        eng.boot_population(one)
        eng.boot_traces(params, block_len=Ls)
        for i in range(R):
            got = eng.fetch_trace(i)
            assert got.tobytes() == mirror(one, params[i], Ls[i]).tobytes(), i
            assert (got["arrive_tick"] == 0).all() and (got["gpus"] == one["gpus"][0]).all()


def test_null_and_ones_are_the_iid_call(pop):
    from gpuschedule_b200 import capi
    lib = capi.load_library()
    R = 20
    params = make_params(R, ns=(0, 1, 257, 2000), scales=((1, 1), (7, 3)), seed=4)
    ones = np.ones(R, dtype=np.uint32)
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, clusters()[i % 2])
        eng.boot_population(pop)
        p = params.ctypes.data_as(C.c_void_p)
        got = {}
        for name, call in (("iid", lambda: lib.gs_boot_traces(eng.h, p, None)),
                           ("null", lambda: lib.gs_boot_traces_blocked(eng.h, p, None, None)),
                           ("ones", lambda: lib.gs_boot_traces_blocked(eng.h, p, ones.ctypes.data_as(C.c_void_p), None))):
            eng._n = [int(k) for k in params["n"].tolist()]
            before = eng.launch_count()
            assert call() == capi.GS_OK
            got[name] = (eng.launch_count() - before, [eng.fetch_trace(i).tobytes() for i in range(R)])
        assert got["iid"][0] == 1
        assert got["null"] == got["iid"] and got["ones"] == got["iid"]
        assert got["iid"][1] == [mirror(pop.packed(), params[i], 1).tobytes() for i in range(R)]
        before = eng.launch_count()
        eng.boot_traces(params, block_len=16)
        assert eng.launch_count() - before == 1


@pytest.mark.parametrize("name", ["fifo", "sjf", "dlas-gpu", "gittins"])
def test_blocked_handle_runs_like_packed_upload(pop, name):
    from gpuschedule_b200 import capi
    R = 24
    params = make_params(R, ns=(1500, 700, 2000, 1), scales=((1, 1), (1, 2), (3, 2)), seed=5)
    shapes = clusters()
    pol = policy(name, pop)
    with capi.Engine(device=0, nsims=R) as gen, capi.Engine(device=0, nsims=R) as ref:
        for i in range(R):
            gen.config(i, shapes[i % 2], pol)
            ref.config(i, shapes[i % 2], pol)
        gen.boot_population(pop)
        results = []
        for Ls in (np.array([(16, 1, 300, 2)[i % 4] for i in range(R)], dtype=np.uint32), 64):
            gen.boot_traces(params, block_len=Ls)
            Lr = np.broadcast_to(Ls, (R,))
            block, pitch, n_each = packed_block([mirror(pop.packed(), params[i], Lr[i]) for i in range(R)])
            ref.load_traces_packed(block, pitch, n_each)
            first = compare_handles(gen, ref, name, R)
            gen.reset()
            ref.reset()
            second = compare_handles(gen, ref, name, R)
            assert first.tobytes() == second.tobytes()
            results.append(first)
        assert results[0].tobytes() != results[1].tobytes()              # a different L gave different traces


def test_zero_block_len_is_refused_and_changes_nothing(pop):
    from gpuschedule_b200 import capi
    lib = capi.load_library()
    R = 4
    good = make_params(R, ns=(400,), scales=((1, 1),), seed=2)
    with capi.Engine(device=0, nsims=R) as eng:
        for i in range(R):
            eng.config(i, clusters()[0])
        eng.boot_population(pop)
        eng.boot_traces(good, block_len=8)
        before = [eng.fetch_trace(i).tobytes() for i in range(R)]
        for Ls in ([8, 0, 8, 8], [0, 0, 0, 0], [1, 1, 1, 0]):
            with pytest.raises(capi.GsError) as e:
                eng.boot_traces(good, block_len=np.array(Ls))
            assert e.value.code == capi.GS_ERR_ARG
        zero = np.zeros(R, dtype=np.uint32)
        assert lib.gs_boot_traces_blocked(eng.h, good.ctypes.data_as(C.c_void_p), zero.ctypes.data_as(C.c_void_p), None) == capi.GS_ERR_ARG
        assert lib.gs_boot_traces_blocked(eng.h, None, zero.ctypes.data_as(C.c_void_p), None) == capi.GS_ERR_ARG
        for bad in (-1, 2 ** 32, 1.5, [8, 8]):
            with pytest.raises(ValueError):
                eng.boot_traces(good, block_len=bad)
        assert [eng.fetch_trace(i).tobytes() for i in range(R)] == before      # refused calls changed nothing
        out = eng.run_summarized()
        assert out["done"].all() and out["n"].tolist() == [400] * R
        eng.boot_traces(good, block_len=3)
        assert eng.fetch_trace(2).tobytes() == mirror(pop.packed(), good[2], 3).tobytes()
        assert eng.run_summarized()["done"].all()


def test_summarize_bootstrap_blocked_equals_the_ordinary_path():
    from gpuschedule_b200 import capi, sweep, tracegen
    trace = os.path.join(GOLDEN, "n64", "trace.csv")
    flag_sets = [sweep.make_flags(trace_file=trace, schedule=s, num_queue=2) for s in ("fifo", "sjf", "dlas-gpu", "gittins")]
    loads, R, seed, L, n = (1.0, 2.0), 3, 7, 8, 150
    recs = sweep.summarize_bootstrap(flag_sets, R, loads, seed=seed, n=n, block_len=L)
    assert recs.shape == (len(flag_sets), len(loads), R)
    for c, (fl, infra, jm, pol) in enumerate(sweep._plain_setup(flag_sets)):
        for li, load in enumerate(loads):
            num, den = sweep.load_gap_scale(load)
            for r in range(R):
                table = tracegen.bootstrap_table(jm.table, seed, r, n, num, den, block_len=L)
                with capi.Engine(device=0, nsims=1) as eng:
                    eng.config(0, infra.gs_cluster(), pol)
                    eng.load_trace(0, table)
                    want = eng.run_summarized()
                assert recs[c, li, r].tobytes() == want[0].tobytes(), (fl.schedule, load, r)
    assert (recs["finished"] > 0).all()
    iid = sweep.summarize_bootstrap(flag_sets, R, loads, seed=seed, n=n)
    assert sweep.summarize_bootstrap(flag_sets, R, loads, seed=seed, n=n, block_len=1).tobytes() == iid.tobytes()


def test_sweep_cli_block_len(tmp_path):
    from gpuschedule_b200 import sweep
    trace = os.path.join(GOLDEN, "n64", "trace.csv")
    out, ci, tl, jd = (str(tmp_path / f) for f in ("s.csv", "ci.csv", "tl.csv", "jd.csv"))
    sweep.main(["--trace", trace, "--schedule", "fifo", "sjf", "--bootstrap", "4", "--block-len", "8", "--load", "1", "1.5",
                "--jobs", "80", "--seed", "3", "--summary", out, "--summary-ci", ci, "--timeline", tl, "--bin-width", "500",
                "--jobdist", jd])
    for path, lines in ((out, 2 * 2 * 4), (ci, 2 * 2)):
        with open(path) as f:
            rows = list(csv.reader(f))
        head = rows[0]
        assert head[head.index("load") + 1] == "block_len" and len(rows) == 1 + lines
        assert {r[head.index("block_len")] for r in rows[1:]} == {"8"}
    for path in (tl, jd):
        with open(path) as f:
            head = next(csv.reader(f))
        assert head[head.index("load") + 1] == "block_len"
    with open(out) as f:
        recs = list(csv.DictReader(f))
    assert {r["n"] for r in recs} == {"80"}

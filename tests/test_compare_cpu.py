"""Paired per-job comparisons (gs_jpair, gpuschedule_b200/csrc/gs_summary.cuh) on a box without a GPU.

gs_cmp_pair_serial, the kernel's steps run serially with the summary's own radix select, is compiled with g++
(tests/emu/compare_emu.cpp) and compared with `reference_pair`, a numpy restatement of the definition in
include/gsched.h that keeps sums and squares in Python integers.  Job values come from the oracles (gsched_oracle's
fifo against policy_oracle's sjf / dlas / dlas-gpu / gittins on the same fixture traces) and from seeded random job
sets.  gs_horus_compare runs through the host-emulation build of gs_horus.cu.  summary.pair_derived / pair_spread /
paired_spread and the sweep's argument errors too."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import REPO, horus_cases, load_horus
from test_summary_cpu import PERMILLE, _policy_cases, load_policy

QUANTS = ("wait", "turnaround", "jct")
DIFF_EDGES = tuple(-2 ** i for i in range(30, -1, -1)) + (0,) + tuple(2 ** i for i in range(31))
BIG = 2 ** 31 - 1


# ---------------------------------------------------------------- the numpy restatement (shared with test_gpu_compare.py)
def reference_pair(arrive, gpus, run_a, fin_a, run_b, fin_b, bounds, edges):
    """(per class a dict of gs_jpair fields -- "d_sq" as exact ints --, CDF counts (C, 3, E + 1)) of runs a and b of one
    trace.  run_x: (start, end, jct) by trace index; fin_x: the finish order.  d = x_b - x_a over the jobs in both
    finish orders; a job's class is #(bounds <= gpus), a value's bin #(edges < d)."""
    arrive, gpus = np.asarray(arrive, dtype=np.int64), np.asarray(gpus, dtype=np.int64)
    n = len(arrive)
    va = [np.asarray(x, dtype=np.int64) for x in run_a]
    vb = [np.asarray(x, dtype=np.int64) for x in run_b]
    qa = (va[0] - arrive, va[1] - arrive, va[2])
    qb = (vb[0] - arrive, vb[1] - arrive, vb[2])
    in_a, in_b = np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
    in_a[np.asarray(fin_a, dtype=np.int64)] = True
    in_b[np.asarray(fin_b, dtype=np.int64)] = True
    cls = np.searchsorted(np.asarray(bounds, dtype=np.int64), gpus, side="right")
    nc, ne = len(bounds) + 1, len(edges)
    e = np.asarray(edges, dtype=np.int64)
    hist = np.zeros((nc, 3, ne + 1), dtype=np.int64)
    out = []
    for c in range(nc):
        both = (cls == c) & in_a & in_b
        k = int(both.sum())
        rec = dict(jobs=k, only_a=int(((cls == c) & in_a & ~in_b).sum()), only_b=int(((cls == c) & ~in_a & in_b).sum()),
                   lt=[], eq=[], gt=[], d_sum=[], d_sq=[], q_hi=[], q_lo=[])
        for m in range(3):
            d = (qb[m] - qa[m])[both]
            rec["lt"].append(int((d < 0).sum())); rec["eq"].append(int((d == 0).sum())); rec["gt"].append(int((d > 0).sum()))
            rec["d_sum"].append(sum(d.tolist())); rec["d_sq"].append(sum(x * x for x in d.tolist()))
            s = sorted(d.tolist())
            ranks = [(p * k + 999) // 1000 - 1 for p in PERMILLE]
            rec["q_hi"].append([s[r] for r in ranks] if k else [0] * 5)
            rec["q_lo"].append([s[k - 1 - r] for r in ranks] if k else [0] * 5)
            hist[c, m] = np.bincount(np.searchsorted(e, d, side="left"), minlength=ne + 1)
        out.append(rec)
    return out, hist


def jpair_fields(rec):
    """one JPAIR_DTYPE record as the dict reference_pair makes"""
    d = {k: int(rec[k]) for k in ("jobs", "only_a", "only_b")}
    for k in ("lt", "eq", "gt", "d_sum"):
        d[k] = [int(x) for x in rec[k]]
    d["d_sq"] = [(int(h) << 64) | int(lo) for lo, h in zip(rec["d_sq_lo"], rec["d_sq_hi"])]
    d["q_hi"], d["q_lo"] = rec["q_hi"].tolist(), rec["q_lo"].tolist()
    return d


def assert_pair(recs, hist, ref, tag=""):
    want, want_hist = ref
    assert len(recs) == len(want), tag
    for c, (rec, w) in enumerate(zip(recs, want)):
        got = jpair_fields(rec)
        for key, v in w.items():
            assert got[key] == v, (tag, c, key, got[key], v)
    assert np.array_equal(np.asarray(hist, dtype=np.int64), want_hist), tag


def run_cols(recs):
    """(start, end, jct) of job records by trace index"""
    return recs["start"], recs["end"], recs["jct"]


def settings_for(values):
    """(bounds, edges) settings: one class and no edge; the notebook's classes with the default signed edges; eight
    classes with 255 edges spanning the differences (negative ones among them, hit exactly); edges equal to values"""
    v = np.unique(np.asarray(values, dtype=np.int64))
    lo, hi = (int(v.min()), int(v.max())) if len(v) else (-1, 1)
    step = max(1, (hi - lo + 20) // 254)
    own = tuple(int(x) for x in v[:255]) if len(v) else ()
    return [((), ()), ((5, 17, 65), DIFF_EDGES), ((1, 2, 3, 4, 8, 16, 32), tuple(lo - 10 + step * i for i in range(255))),
            ((2,), own), ((10 ** 6,), (-5, 0, 5))]


# ---------------------------------------------------------------- host build
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("compare_emu") / "libcompare_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "compare_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.emu_cmp_pair.restype = C.c_int
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def emu_pair(lib, arrive, gpus, run_a, fin_a, run_b, fin_b, bounds, edges, nclasses=None):
    """(rc, recs (C,), hist (C, 3, E + 1)) of gs_cmp_pair_serial"""
    from gpuschedule_b200.capi import JPAIR_DTYPE
    arrive, gpus, fin_a, fin_b = _i32(arrive), _i32(gpus), _i32(fin_a), _i32(fin_b)
    ra, rb = [_i32(x) for x in run_a], [_i32(x) for x in run_b]
    nc = len(bounds) + 1 if nclasses is None else nclasses
    recs = np.zeros(max(nc, 1), dtype=JPAIR_DTYPE)
    hist = np.zeros((max(nc, 1), 3, len(edges) + 1), dtype=np.uint32)
    b, e = _i32(bounds if len(bounds) else [0]), _i32(edges if len(edges) else [0])
    rc = lib.emu_cmp_pair(_p(arrive), _p(gpus), C.c_longlong(len(arrive)), _p(ra[0]), _p(ra[1]), _p(ra[2]), _p(fin_a),
                          C.c_longlong(len(fin_a)), _p(rb[0]), _p(rb[1]), _p(rb[2]), _p(fin_b), C.c_longlong(len(fin_b)),
                          C.c_int(nc), _p(b) if len(bounds) else None, C.c_int(len(edges)), _p(e) if len(edges) else None, _p(recs), _p(hist))
    return rc, recs[:nc], hist[:nc]


def check_pair(lib, arrive, gpus, run_a, fin_a, run_b, fin_b, bounds, edges, tag):
    rc, recs, hist = emu_pair(lib, arrive, gpus, run_a, fin_a, run_b, fin_b, bounds, edges)
    assert rc == 0, tag
    assert_pair(recs, hist, reference_pair(arrive, gpus, run_a, fin_a, run_b, fin_b, bounds, edges), tag)
    # swapping the pair: lt / gt and only_a / only_b swap, sums negate, squares stay, q_hi(b, a) = -q_lo(a, b)
    _, sw, sw_hist = emu_pair(lib, arrive, gpus, run_b, fin_b, run_a, fin_a, bounds, edges)
    assert (sw["only_a"] == recs["only_b"]).all() and (sw["lt"] == recs["gt"]).all() and (sw["eq"] == recs["eq"]).all(), tag
    assert (sw["d_sum"] == -recs["d_sum"]).all() and (sw["d_sq_lo"] == recs["d_sq_lo"]).all() and (sw["q_hi"] == -recs["q_lo"]).all(), tag
    return recs, hist


def test_emu_matches_definition_hand_worked(emu):
    """three jobs, job 2 finished in b only: d = (b - a) of wait / turnaround / jct for jobs 0 and 1"""
    arrive, gpus = [0, 0, 5], [1, 8, 1]
    run_a = ([1, 4, 0], [3, 10, 0], [2, 6, 0])
    run_b = ([0, 9, 7], [5, 11, 8], [5, 2, 1])
    rc, recs, hist = emu_pair(emu, arrive, gpus, run_a, [0, 1], run_b, [1, 0, 2], (), (-1, 0, 1))
    assert rc == 0
    r = recs[0]
    assert (int(r["jobs"]), int(r["only_a"]), int(r["only_b"])) == (2, 0, 1)
    assert r["d_sum"].tolist() == [-1 + 5, 2 + 1, 3 - 4]                         # waits -1, 5; turnarounds 2, 1; jcts 3, -4
    assert r["d_sq_lo"].tolist() == [1 + 25, 4 + 1, 9 + 16]
    assert r["lt"].tolist() == [1, 0, 1] and r["gt"].tolist() == [1, 2, 1] and r["eq"].tolist() == [0, 0, 0]
    assert r["q_hi"][0].tolist() == [-1, 5, 5, 5, 5] and r["q_lo"][0].tolist() == [5, -1, -1, -1, -1]
    assert hist[0, 0].tolist() == [1, 0, 0, 1] and hist[0, 2].tolist() == [1, 0, 0, 1]


def test_fixture_oracles_fifo_against_policies(emu):
    import oracle
    for case in _policy_cases():
        table, cluster, pol = load_policy(case)
        f = oracle.run_fifo(cluster, table)
        p = oracle.run_policy(cluster, pol, table)
        ra, rb = run_cols(f.recs), run_cols(p.recs)
        d = np.concatenate([(np.asarray(rb[i], dtype=np.int64) - np.asarray(ra[i], dtype=np.int64)) for i in range(3)])
        for bounds, edges in settings_for(d):
            check_pair(emu, table.arrive_tick, table.gpus, ra, f.finish_order, rb, p.finish_order, bounds, edges, f"{case} {bounds}")
            # a prefix of each finish order: the state after some window, with only-a and only-b jobs
            check_pair(emu, table.arrive_tick, table.gpus, ra, f.finish_order[:len(f.finish_order) // 2], rb,
                       p.finish_order[:len(p.finish_order) // 3], bounds, edges, f"{case} partial {bounds}")


def _random_case(rng, n, scale, tie_frac=0.0):
    arrive = np.sort(rng.integers(0, scale, n))
    gpus = rng.choice([1, 2, 4, 5, 8, 16, 17, 32, 64, 65, 128], n)

    def run():
        start = arrive + rng.integers(0, scale, n)
        jct = rng.integers(1, scale, n)
        return start, start + jct + rng.integers(0, 3, n), jct
    ra, rb = run(), run()
    if tie_frac:
        tie = rng.random(n) < tie_frac
        rb = tuple(np.where(tie, x, y) for x, y in zip(ra, rb))
    return arrive, gpus, ra, rb


def test_random_job_sets(emu):
    rng = np.random.default_rng(29)
    for n in (0, 1, 2, 3, 257, 3000):
        for scale, ties in ((10, 0.5), (2 ** 20, 0.1), (2 ** 29, 0.0)):
            arrive, gpus, ra, rb = _random_case(rng, n, scale, ties)
            fa, fb = rng.permutation(n), rng.permutation(n)
            for cut_a, cut_b in ((n, n), (n // 2, n), (n, n // 3), (0, n)):
                d = np.concatenate([rb[i][:cut_a] - ra[i][:cut_a] for i in range(3)]) if n else np.zeros(0)
                for bounds, edges in settings_for(d)[:3]:
                    check_pair(emu, arrive, gpus, ra, fa[:cut_a], rb, fb[:cut_b], bounds, edges, f"n={n} scale={scale} cut={cut_a},{cut_b}")


def test_small_counts_ties_and_empty_classes(emu):
    arrive, gpus = np.zeros(4, dtype=np.int64), np.array([1, 1, 100, 100])
    same = (np.array([3, 3, 3, 3]), np.array([9, 9, 9, 9]), np.array([6, 6, 6, 6]))
    later = tuple(x + 2 for x in same)
    for fa, fb, tag in (([0], [0], "k=1"), ([0, 1], [1, 0], "k=2"), ([0, 1, 2, 3], [3, 2, 1, 0], "all"), ([], [2, 3], "only b"), ([2, 3], [], "only a")):
        for run_b in (same, later):
            recs, hist = check_pair(emu, arrive, gpus, same, fa, run_b, fb, (5, 50, 1000), (-2, 0, 2), tag)
            assert recs["jobs"][3] == 0 and recs["q_hi"][3].tolist() == [[0] * 5] * 3       # the class 1000+ is empty
    rc, recs, _ = emu_pair(emu, arrive, gpus, same, [0, 1, 2, 3], same, [0, 1, 2, 3], (), ())
    assert recs["eq"][0].tolist() == [4, 4, 4] and recs["d_sum"][0].tolist() == [0, 0, 0] and not recs["q_hi"].any()


def test_extreme_differences(emu):
    """d = +-(2^31 - 1): x_a = 0 and x_b = 2^31 - 1 and the reverse; the points and squares need every bit"""
    arrive, gpus = np.zeros(4, dtype=np.int64), np.array([1, 2, 3, 4])
    ra = (np.array([0, BIG, 0, BIG]), np.array([0, BIG, BIG, 0]), np.array([0, BIG, 5, 6]))
    rb = (np.array([BIG, 0, 0, BIG]), np.array([BIG, 0, BIG, 0]), np.array([BIG, 0, 5, 6]))
    for bounds, edges in (((), ()), ((), (-BIG, 0, BIG - 1)), ((), (-2 ** 31, -BIG + 1, BIG)), ((3,), DIFF_EDGES)):
        recs, hist = check_pair(emu, arrive, gpus, ra, [0, 1, 2, 3], rb, [3, 2, 1, 0], bounds, edges, f"extreme {edges}")
    assert recs["q_hi"][0][0][4] == BIG and recs["q_lo"][0][0][4] == -BIG


def test_setting_errors(emu):
    arrive, gpus = np.zeros(2), np.ones(2)
    run = (np.zeros(2), np.zeros(2), np.zeros(2))
    for bounds, edges, nc in (((), (), 0), ((), (), 9), ((0,), (), None), ((3, 3), (), None), ((), (1, 1), None), ((), tuple(range(256)), None)):
        assert emu_pair(emu, arrive, gpus, run, [0], run, [1], bounds, edges, nclasses=nc)[0] == -1, (bounds, len(edges), nc)


# ---------------------------------------------------------------- gs_horus_compare, host build of gs_horus.cu
@pytest.fixture(scope="module")
def horus_emu_engine():
    import importlib.util
    import sys
    spec = importlib.util.spec_from_file_location("tests_emu_compare", os.path.join(REPO, "tests", "emu", "__init__.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["tests_emu_compare"] = mod
    spec.loader.exec_module(mod)
    out = mod._ABI_OUT
    hdr = os.path.join(REPO, "gpuschedule_b200", "csrc", "gs_summary.cuh")
    if os.path.exists(out) and os.path.getmtime(out) < os.path.getmtime(hdr) and mod._abi_lib is None:
        mod.build_abi(force=True)                 # gs_summary.cuh is not among the emu build's own dependencies
    return mod.emu_engine_class()


def _code(fn, *a, **k):
    from gpuschedule_b200 import capi
    with pytest.raises(capi.GsError) as e:
        fn(*a, **k)
    return e.value.code


def horus_pairs_setup(eng, cases):
    """replica 2i: fixture i as recorded; replica 2i + 1: the same trace, cluster and words under another schedule"""
    from gpuschedule_b200 import capi
    other = {"horus": ("gandiva", "gandiva"), "horus+": ("horus", "horus"), "gandiva": ("horus", "horus")}
    loaded = []
    for i, case in enumerate(cases):
        table, cluster, params, _, _ = load_horus(case)
        scheme, sched = other[params["schedule"]]
        np.random.seed(params["seed"])
        words = np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32)
        for k, (sc, sh) in enumerate(((params["scheme"], params["schedule"]), (scheme, sched))):
            eng.config(2 * i + k, cluster, capi.make_horus_params(sc, sh, params["num_buffer"], params["num_queue"]))
            eng.load_trace(2 * i + k, table)
            eng.load_words(2 * i + k, words)
        loaded.append(table)
    return loaded


def test_horus_compare_host_build(horus_emu_engine):
    from gpuschedule_b200 import capi
    cases = horus_cases()[:4]
    with horus_emu_engine(device=0, nsims=2 * len(cases)) as eng:
        tables = horus_pairs_setup(eng, cases)
        assert _code(eng.compare, [0], [1]) == capi.GS_ERR_STATE                 # nothing has run
        eng.run(rows_cap=1 << 15)
        n0 = eng.lib.gs_horus_launch_count(eng.h)
        for a, b, bounds, edges in (([0], [2 * len(cases)], (), ()), ([-1], [0], (), ()), ([0], [1], (0,), ()), ([0], [1], (3, 3), ()),
                                    ([0], [1], (), (1, 1)), ([0], [1], (), tuple(range(256))), ([0], [1], tuple(range(1, 9)), ())):
            assert _code(eng.compare, a, b, bounds, edges) == capi.GS_ERR_ARG, (a, b, bounds, len(edges))
        assert _code(eng.compare, [0, 1], [1, 2]) == capi.GS_ERR_ARG                  # pair 1 holds two different traces
        assert b"pair 1" in eng.lib.gs_horus_last_error(eng.h)
        assert eng.compare([], [])[0].shape == (0, 1)
        assert eng.lib.gs_horus_launch_count(eng.h) == n0 + 1                                          # only the refused pair launched
        for bounds, edges in (((), ()), ((5, 17, 65), DIFF_EDGES), ((2,), (-100, -1, 0, 1, 100))):
            pa = [2 * i for i in range(len(cases))] + [2 * i + 1 for i in range(len(cases))] + [0]
            pb = [2 * i + 1 for i in range(len(cases))] + [2 * i for i in range(len(cases))] + [0]
            recs, hist = eng.compare(pa, pb, bounds, edges)
            for p, (a, b) in enumerate(zip(pa, pb)):
                table = tables[a // 2]
                _, _, _, ra, fa = eng.fetch(a)
                _, _, _, rb, fb = eng.fetch(b)
                assert_pair(recs[p], hist[p], reference_pair(table.arrive_tick, table.gpus, run_cols(ra), fa, run_cols(rb), fb, bounds, edges),
                            f"{cases[a // 2]} {a},{b} {bounds}")


# ---------------------------------------------------------------- summary.pair_derived / pair_spread / paired_spread
def test_pair_derived_matches_pandas(emu):
    import pandas as pd
    from gpuschedule_b200 import summary
    rng = np.random.default_rng(5)
    arrive, gpus, ra, rb = _random_case(rng, 3000, 2 ** 28, 0.2)
    gpus[0] = 200
    gpus[1:] = np.where(gpus[1:] > 64, 64, gpus[1:])
    fa, fb = np.arange(3000), np.arange(2900)
    bounds, edges = (5, 17, 65, 1000), (-2 ** 27, -1, 0, 1, 2 ** 27)
    _, recs, hist = emu_pair(emu, arrive, gpus, ra, fa, rb, fb, bounds, edges)
    d = summary.pair_derived(recs, hist, edges)
    df = pd.DataFrame(dict(wait=(rb[0] - arrive) - (ra[0] - arrive), turnaround=rb[1] - ra[1], jct=rb[2] - ra[2], g=gpus))[:2900]
    df["cls"] = pd.cut(df["g"], [0, 4, 16, 64, 999, 10 ** 9], labels=False)
    assert d["jobs"].tolist() == [int((df["cls"] == c).sum()) for c in range(5)]
    assert d["only_a"].sum() == 100 and d["only_b"].sum() == 0
    for c in range(5):
        g = df[df["cls"] == c]
        for q in QUANTS:
            if len(g) == 0:
                assert math.isnan(d[q + "_d_mean"][c]) and math.isnan(d[q + "_d_p50"][c]) and math.isnan(d[q + "_cdf"][c, 0])
                continue
            assert math.isclose(d[q + "_d_mean"][c], g[q].mean(), rel_tol=1e-12)
            if len(g) > 1:
                assert math.isclose(d[q + "_d_std"][c], g[q].std(), rel_tol=1e-12), (c, q)
            assert d[q + "_lt_share"][c] == (g[q] < 0).mean() and d[q + "_gt_share"][c] == (g[q] > 0).mean()
            s = np.sort(g[q].to_numpy())
            assert d[q + "_d_p100"][c] == s[-1] and d[q + "_d_p0"][c] == s[0]
            assert d[q + "_d_p90"][c] == s[(900 * len(s) + 999) // 1000 - 1] and d[q + "_d_p10"][c] == s[len(s) - 1 - ((900 * len(s) + 999) // 1000 - 1)]
            assert d[q + "_cdf"][c].tolist() == [float((g[q] <= e).mean()) for e in edges]
    assert len(summary.pair_flat(d, 0, "jct")) == len(summary.pair_columns())
    with pytest.raises(ValueError):
        summary.pair_derived(recs, hist, edges[:-1])


def _jpairs(specs):
    from gpuschedule_b200.capi import JPAIR_DTYPE
    out = np.zeros(len(specs), dtype=JPAIR_DTYPE)
    for i, d in enumerate(specs):
        for key, v in d.items():
            out[i][key] = v
    return out


def test_pair_derived_hand_worked_and_spread():
    from gpuschedule_b200 import summary
    # two jobs with wait differences -3 and 5: mean 1, std sqrt(32), shares 1/2 below and above
    rec = _jpairs([dict(jobs=2, lt=[1, 0, 0], gt=[1, 0, 0], eq=[0, 2, 2], d_sum=[2, 0, 0], d_sq_lo=[34, 0, 0],
                        q_hi=[[-3, 5, 5, 5, 5], [0] * 5, [0] * 5], q_lo=[[5, -3, -3, -3, -3], [0] * 5, [0] * 5])])
    hist = np.zeros((1, 3, 2), dtype=np.uint32)
    hist[0, 0] = [1, 1]
    hist[0, 1:, 0] = 2
    d = summary.pair_derived(rec, hist, (0,))
    assert d["wait_d_mean"][0] == 1.0 and d["wait_d_std"][0] == math.sqrt(32.0)
    assert d["wait_lt_share"][0] == 0.5 and d["wait_eq_share"][0] == 0.0 and d["jct_eq_share"][0] == 1.0
    assert d["wait_d_p0"][0] == -3 and d["wait_d_p100"][0] == 5 and d["wait_d_p50"][0] == -3 and d["wait_d_p50_lo"][0] == 5
    assert d["wait_cdf"][0].tolist() == [0.5] and d["jct_cdf"][0].tolist() == [1.0]
    # spread over three replicas; class 1 has jobs in one replica only
    R = 3
    specs = []
    for r in range(R):
        specs.append(dict(jobs=1, d_sum=[r, 0, 0], d_sq_lo=[r * r, 0, 0], gt=[int(r > 0), 0, 0], eq=[int(r == 0), 1, 1], q_hi=[[r] * 5, [0] * 5, [0] * 5]))
        specs.append(dict(jobs=2 if r == 1 else 0, only_a=4, d_sum=[8, 0, 0], d_sq_lo=[32, 0, 0], gt=[2, 0, 0]))
    recs = _jpairs(specs).reshape(R, 2)
    hs = np.zeros((R, 2, 3, 2), dtype=np.uint32)
    sp = summary.pair_spread(recs, hs, (0,), level=0.8)
    assert sp["replicas"].tolist() == [3, 1]
    assert sp["wait_d_mean"]["mean"][0] == 1.0 and sp["wait_d_mean"]["lo"][0] == 0.0 and sp["wait_d_mean"]["hi"][0] == 2.0
    assert sp["wait_d_mean"]["std"][0] == 1.0 and sp["wait_gt_share"]["mean"][0] == pytest.approx(2 / 3)
    assert sp["wait_d_mean"]["mean"][1] == 4.0 and math.isnan(sp["wait_d_mean"]["std"][1]) and sp["only_a"]["mean"][1] == 4.0
    assert len(summary.pair_spread_flat(sp, 0, "wait")) == len(summary.pair_spread_columns())
    with pytest.raises(ValueError):
        summary.pair_spread(recs[0], hs[0], (0,))


def test_paired_spread_against_pandas():
    import pandas as pd
    from gpuschedule_b200 import capi, summary
    rng = np.random.default_rng(11)
    R = 9
    ra, rb = np.zeros(R, dtype=capi.SUMMARY_DTYPE), np.zeros(R, dtype=capi.SUMMARY_DTYPE)
    for recs in (ra, rb):
        recs["rows"] = rng.integers(100, 200, R)
        recs["makespan"] = rng.integers(1000, 2000, R)
        recs["busy_gpus_sum"] = rng.integers(0, 10 ** 6, R)
        recs["finished"] = 50
        recs["wait_sum"] = rng.integers(0, 10 ** 5, R)
        recs["jct_sum"] = rng.integers(0, 10 ** 5, R)
        recs["pending_rows"] = 10
        recs["avg_pending_sum"] = rng.random(R) * 100
    rb["makespan"][:3] = ra["makespan"][:3]                       # three ties
    ca, cb = (128, 8, 32), (64, 8, 32)
    sp = summary.paired_spread(ra, rb, ca, cb, level=0.8)
    da = pd.DataFrame([summary.derived(r, *ca) for r in ra])
    db = pd.DataFrame([summary.derived(r, *cb) for r in rb])
    diff = db - da
    diff["makespan"] = rb["makespan"].astype(float) - ra["makespan"].astype(float)
    for m in ("makespan", "gpu_share", "wait_mean", "pending_mean"):
        assert sp[m]["mean"] == pytest.approx(diff[m].mean(), rel=1e-12) and sp[m]["std"] == pytest.approx(diff[m].std(), rel=1e-12)
        s = np.sort(diff[m].to_numpy())
        assert sp[m]["lo"] == s[0] and sp[m]["hi"] == s[-1]                         # level 0.8 of 9: ranks 0 and 8
        assert (sp[m]["b_lt_a"], sp[m]["b_eq_a"], sp[m]["b_gt_a"]) == (int((diff[m] < 0).sum()), int((diff[m] == 0).sum()), int((diff[m] > 0).sum()))
    assert sp["makespan"]["b_eq_a"] >= 3
    assert len(summary.paired_flat(sp)) == len(summary.paired_columns())
    with pytest.raises(ValueError):
        summary.paired_spread(ra, rb[:-1], ca, cb)


# ---------------------------------------------------------------- sweep argument errors (before any engine exists)
def test_sweep_compare_argument_errors(tmp_path, monkeypatch):
    from gpuschedule_b200 import capi, sweep

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(capi, "Engine", no_engine)
    monkeypatch.setattr(capi, "HorusEngine", no_engine)
    t1, t2 = str(tmp_path / "missing1.csv"), str(tmp_path / "missing2.csv")
    fl = [sweep.make_flags(trace_file=t1), sweep.make_flags(trace_file=t1, schedule="sjf"), sweep.make_flags(trace_file=t2),
          sweep.make_flags(trace_file=t1, schedule="horus", scheme="horus")]
    for bad in ((((0, 2),), (), ()), (((0, 3),), (), ()), (((0, 4),), (), ()), (((0, 1),), (0,), ()), (((0, 1),), (), (2, 1)),
                (((0, 1),), (), tuple(range(256))), (((0,),), (), ()), 5, (((0, 1),), ())):
        with pytest.raises(ValueError):
            sweep.summarize_batched(fl, compare=bad)
        with pytest.raises(ValueError):
            sweep.summarize_bootstrap(fl[:3], 2, compare=bad)
    with pytest.raises(ValueError, match="different engines"):
        sweep.check_compare((((0, 3),), (), ()), fl)
    assert sweep.check_compare((((0, 1),), [5], [-1, 0]), fl) == (((0, 1),), (5,), (-1, 0))
    assert sweep.DEFAULT_DIFF_EDGES == DIFF_EDGES and len(DIFF_EDGES) == 63
    base = ["--trace", t1, "--summary", "s.csv"]
    for argv in (["--trace", t1, "--compare", "fifo", "--schedule", "fifo", "sjf"],                       # no --summary
                 base + ["--schedule", "fifo", "sjf", "--compare", "dlas"],                             # not a schedule
                 base + ["--schedule", "fifo", "sjf", "fifo", "--compare", "fifo"],                     # listed twice
                 base + ["--schedule", "fifo", "horus", "--compare", "fifo"],                           # different engines
                 base + ["--schedule", "fifo", "sjf", "--paired", "p.csv"],                             # no --compare
                 base + ["--schedule", "fifo", "sjf", "--paired-summary", "p.csv"],
                 base + ["--schedule", "fifo", "sjf", "--diff-edges", "1"],
                 base + ["--schedule", "fifo", "sjf", "--paired-cdf", "c.csv"],
                 base + ["--schedule", "fifo", "sjf", "--compare", "fifo", "--paired-cdf", "c.csv"],   # no --paired
                 base + ["--schedule", "fifo", "sjf", "--compare", "fifo", "--paired", "p.csv", "--diff-edges", "2", "1"],
                 base + ["--schedule", "fifo", "sjf", "--compare", "fifo", "--paired", "p.csv", "--gpu-classes", "0"],
                 base + ["--schedule", "fifo", "sjf", "--gpu-classes", "5"]):                          # neither --jobdist nor --paired
        with pytest.raises(SystemExit) as e:
            sweep.main(argv)
        assert e.value.code == 2, argv
    for name in ("s.csv", "p.csv", "c.csv"):
        assert not (tmp_path / name).exists()

"""Timelines (gs_tbin: a run's rows binned by `delta`, gpuschedule_b200/csrc/gs_summary.cuh) on a box without a GPU.

The __host__ __device__ part -- the bin key, the per-bin fold of rows and of the fifo engine's compact records, the
serial row fold -- is compiled with g++ (tests/emu/timeline_emu.cpp, whose loops restate the kernels' range logic) and
compared with a numpy binning of rows: the pinned oracles' rows on every fixture, the fifo records folded window by
window, the event-driven policies' rows in their own order and shuffled, and the host-emulation build of gs_horus.cu
through gs_horus_summarize itself.  summary.timeline_derived / timeline_spread and the sweep's argument errors too."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import REPO, golden_cases, horus_cases, load_golden, load_horus
from test_summary_cpu import _policy_cases, load_policy

INT_FIELDS = ("rows", "busy_gpus_sum", "running_sum", "queued_sum", "busy_gpus_max", "running_max", "queued_max", "pend_max_max",
              "pend_sum_sum", "mem_busy_sum", "pending_rows", "delta_min", "delta_max", "finished_last")
FLOAT_FIELDS = ("avg_pending_sum", "util_sum")
GRID_B = (1, 2, 1024)


# ---------------------------------------------------------------- the numpy binning (shared with test_gpu_timeline.py)
def bin_of(delta, W, B):
    return np.minimum(np.maximum(np.asarray(delta, dtype=np.int64), 0) // W, B - 1)


def reference_bins(rows, W, B, util=None):
    """per bin, the gs_tbin fields of cluster.csv-style rows (ROW_DTYPE, in row order) as a dict; 128-bit fields as
    exact ints, util_sum only when `util` is given (NaN counted as 0); a bin without rows is all zero"""
    key = bin_of(rows["now"], W, B)
    out = []
    for b in range(B):
        m = key == b
        r = rows[m]
        d = dict.fromkeys(INT_FIELDS, 0)
        d["avg_pending_sum"] = 0.0
        if util is not None:
            d["util_sum"] = 0.0
        if len(r):
            d["rows"] = len(r)
            for f in ("busy_gpus", "running", "queued"):
                d[f + "_sum"] = int(r[f].astype(np.int64).sum())
                d[f + "_max"] = int(r[f].max())
            d["pend_max_max"] = int(r["pend_max"].max())
            d["pend_sum_sum"] = sum(r["pend_sum"].tolist())
            d["mem_busy_sum"] = sum(r["mem_busy_bytes"].tolist())
            nz = (r["queued"] > 0) & (r["pend_sum"] != 0)
            d["pending_rows"] = int(nz.sum())
            d["avg_pending_sum"] = math.fsum((r["pend_sum"][nz].astype(np.float64) / (r["queued"][nz].astype(np.float64) + 1e-9)).tolist())
            d["delta_min"], d["delta_max"] = int(r["now"].min()), int(r["now"].max())
            d["finished_last"] = int(r["finished"][-1])
            if util is not None:
                d["util_sum"] = math.fsum(np.nan_to_num(np.asarray(util, dtype=np.float64)[m], nan=0.0).tolist())
        out.append(d)
    return out


def bin_fields(t):
    """one TBIN_DTYPE record as the dict reference_bins makes"""
    d = {name: t[name].item() for name in t.dtype.names}
    d["pend_sum_sum"] = (int(t["pend_sum_hi"]) << 64) | int(t["pend_sum_lo"])
    d["mem_busy_sum"] = (int(t["mem_busy_hi"]) << 64) | int(t["mem_busy_lo"])
    return d


def assert_bins(got, ref, tag="", rel=1e-12, skip=()):
    assert len(got) == len(ref), (tag, len(got), len(ref))
    for b, (t, want) in enumerate(zip(got, ref)):
        g = bin_fields(t)
        for key, w in want.items():
            if key in skip:
                continue
            if key in FLOAT_FIELDS:
                assert math.isclose(g[key], w, rel_tol=rel, abs_tol=1e-12), (tag, b, key, g[key], w)
            else:
                assert g[key] == w, (tag, b, key, g[key], w)


def widths(makespan):
    return (1, 3, 64, int(makespan) + 5)


# ---------------------------------------------------------------- host build of the timeline fold
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("timeline_emu") / "libtimeline_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "timeline_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.emu_tl_rows.restype = C.c_int
    lib.emu_tl_bin.restype = C.c_int
    return lib


def _p(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def emu_rows(lib, rows, W, B, util=None, serial=False):
    """(bins, 1 if the serial path was taken)"""
    from gpuschedule_b200.capi import TBIN_DTYPE
    bins = np.zeros(B, dtype=TBIN_DTYPE)
    rows = np.ascontiguousarray(rows)
    u = None if util is None else np.ascontiguousarray(util, dtype=np.float64)
    args = (_p(rows), _p(u), C.c_longlong(0), C.c_longlong(len(rows)), C.c_longlong(W), C.c_int(B), _p(bins))
    if serial:
        lib.emu_tl_rows_serial(*args)
        return bins, 1
    return bins, lib.emu_tl_rows(*args)


def test_bin_key(emu):
    for delta, W, B, want in ((0, 1, 1, 0), (5, 1, 1024, 5), (5, 3, 1024, 1), (2000, 1, 1024, 1023), (-4, 2, 8, 0),
                              (63, 64, 2, 0), (64, 64, 2, 1), (10 ** 9, 64, 2, 1), (10 ** 9, 2 ** 40, 1024, 0)):
        assert emu.emu_tl_bin(C.c_longlong(delta), C.c_longlong(W), C.c_int(B)) == want, (delta, W, B)
        assert int(bin_of([delta], W, B)[0]) == want


# ---------------------------------------------------------------- rows of the oracles
@pytest.mark.parametrize("case", golden_cases())
def test_fifo_fixture_rows_fold(emu, case):
    import oracle
    table, cluster, _, _, _ = load_golden(case)
    rows = oracle.run_fifo(cluster, table).rows
    for W in widths(rows["now"][-1]):
        for B in GRID_B:
            got, serial = emu_rows(emu, rows, W, B)
            assert serial == 0
            assert_bins(got, reference_bins(rows, W, B), f"{case} W={W} B={B}")


@pytest.mark.parametrize("case", _policy_cases())
def test_policy_fixture_rows_fold_in_any_order(emu, case):
    """the rows of the event-driven policies, binned by their own delta: in the engine's row order (whatever it is),
    and shuffled so that delta goes back and forth (the kernel's serial path)"""
    import oracle
    table, cluster, pol = load_policy(case)
    rows = oracle.run_policy(cluster, pol, table).rows
    shuffled = rows[np.random.default_rng(5).permutation(len(rows))]
    assert (np.diff(shuffled["now"]) < 0).any()
    for W in widths(rows["now"].max()):
        for B in GRID_B:
            for tag, rr in (("row order", rows), ("shuffled", shuffled)):
                ref = reference_bins(rr, W, B)
                for serial in (False, True):
                    got, _ = emu_rows(emu, rr, W, B, serial=serial)
                    assert_bins(got, ref, f"{case} {tag} W={W} B={B} serial={serial}")


@pytest.mark.parametrize("case", horus_cases())
def test_horus_fixture_rows_fold_with_utilisation(emu, case):
    import oracle
    table, cluster, params, _, _ = load_horus(case)
    res = oracle.run_horus(cluster, table, **params)
    for W in widths(res.rows["now"][-1]):
        for B in GRID_B:
            got, serial = emu_rows(emu, res.rows, W, B, util=res.util)
            assert serial == 0
            assert_bins(got, reference_bins(res.rows, W, B, util=res.util), f"{case} W={W} B={B}")


# ---------------------------------------------------------------- the fifo engine's compact records, window by window
def fold_windows(lib, t2, W, B, **run_kw):
    """restart the Tight2 yardstick and fold the records of every window as gs_summarize does after every gs_run"""
    from gpuschedule_b200.capi import TBIN_DTYPE
    bins = np.zeros(B, dtype=TBIN_DTYPE)
    t2.restart()
    wm, windows, records = 0, 0, []
    while True:
        rc, w, _, _, done = t2.run_window(**run_kw)
        assert rc == 0
        ev, qr = t2.ev[:w.ev_rows].copy(), t2.qr[:w.q_rows].copy()
        for _ in range(2):                     # a second fold of the same window adds nothing
            lib.emu_tl_compact(_p(ev), C.c_int(len(ev)), _p(qr), C.c_int(len(qr)), C.c_longlong(w.ticks), C.c_longlong(wm),
                               C.c_longlong(W), C.c_int(B), _p(bins))
            wm = max(wm, int(w.ticks))
        records.append((ev, qr, int(w.ticks)))
        windows += 1
        if done or t2.n == 0:
            return bins, windows, records


def _straddles(records, W, B):
    """(records with a queue whose rows cross a bin boundary, such records whose zero-pending row lies inside)"""
    n_split = n_zero = 0
    for ev, qr, ticks in records:
        qi = 0
        for k in range(len(ev)):
            e = ev[k]
            t_last = int(ev[k + 1]["now"]) - 1 if k + 1 < len(ev) else ticks
            if e["queued"] <= 0:
                continue
            while qr[qi]["now"] < e["now"]:
                qi += 1
            if bin_of([e["now"]], W, B)[0] != bin_of([t_last], W, B)[0]:
                n_split += 1
                a, q = int(qr[qi]["arrive_sum"]), int(e["queued"])
                n_zero += a % q == 0 and int(e["now"]) <= a // q <= t_last
    return n_split, n_zero


@pytest.mark.parametrize("case", golden_cases())
def test_fifo_records_fold_window_by_window(emu, case):
    import oracle
    table, cluster, _, _, _ = load_golden(case)
    if cluster.enable_network_costs:
        pytest.skip("the record yardstick runs the plain fifo + yarn tick only (no network-cost branch)")
    rows = oracle.run_fifo(cluster, table).rows
    t2 = oracle.Tight2(cluster, table)
    for W in widths(rows["now"][-1]):
        for B in GRID_B:
            ref = reference_bins(rows, W, B)
            whole, n1, _ = fold_windows(emu, t2, W, B)
            assert n1 == 1
            assert_bins(whole, ref, f"{case} W={W} B={B}")
            for kw, tag in ((dict(max_ticks=7), "7-tick windows"), (dict(cap_a=1, cap_b=1), "one record per window")):
                got, nw, _ = fold_windows(emu, t2, W, B, **kw)
                assert nw > 1, tag
                assert_bins(got, ref, f"{case} {tag} W={W} B={B}")
                for a, b in zip(got, whole):
                    fa, fb = bin_fields(a), bin_fields(b)
                    assert all(fa[k] == fb[k] for k in INT_FIELDS), (case, tag, W, B)


def test_fixtures_have_records_that_straddle_bin_boundaries():
    """the window-by-window test above meets many records with a queue that straddle a bin boundary"""
    import oracle
    n_split = 0
    for case in golden_cases():
        table, cluster, _, _, _ = load_golden(case)
        if cluster.enable_network_costs:
            continue
        t2 = oracle.Tight2(cluster, table)
        t2.restart()
        rc, w, _, _, _ = t2.run_window()
        assert rc == 0
        recs = [(t2.ev[:w.ev_rows].copy(), t2.qr[:w.q_rows].copy(), int(w.ticks))]
        for W in (3, 64):
            n_split += _straddles(recs, W, 1024)[0]
    assert n_split > 100, n_split


def test_split_record_with_a_zero_pending_row(emu):
    """hand-made records (the fixtures never queue a job on its arrival row): record 1 covers ticks 6 .. 17 with two
    jobs queued that both arrived at 6, so its pending sum 2v - 12 is zero on its first row, 6 -- the only row of a
    record where it can be zero.  The widths below split the record in many ways, with row 6 at the start, in the
    middle or at the end of a piece"""
    from gpuschedule_b200.capi import EVROW_DTYPE, QROW_DTYPE
    from gpuschedule_b200.log_manager import ROW_DTYPE
    ev = np.zeros(3, dtype=EVROW_DTYPE)
    ev[0] = (1, 0, 0, 8, 2, 1000)
    ev[1] = (6, 2, 1, 16, 3, 5000)
    ev[2] = (18, 1, 4, 4, 1, 7)
    qr = np.zeros(2, dtype=QROW_DTYPE)
    qr[0] = (6, 6, 6, 6, 12)
    qr[1] = (18, 15, 15, 15, 15)
    ticks = 25
    rows = np.zeros(ticks, dtype=ROW_DTYPE)
    for v in range(1, ticks + 1):
        k = 0 if v < 6 else 1 if v < 18 else 2
        e = ev[k]
        r = rows[v - 1]
        r["now"], r["queued"], r["finished"], r["busy_gpus"], r["running"], r["mem_busy_bytes"] = v, e["queued"], e["finished"], e["busy_gpus"], e["running"], e["mem_busy_bytes"]
        if e["queued"]:
            q = qr[k - 1]
            r["pend_sum"], r["pend_max"] = int(e["queued"]) * v - int(q["arrive_sum"]), v - int(q["oldest_arrive"])
    assert (rows["pend_sum"][(rows["queued"] > 0)] == 0).sum() == 1
    from gpuschedule_b200.capi import TBIN_DTYPE
    for W in (1, 2, 3, 4, 5, 6, 7, 30):
        for B in (1, 2, 3, 1024):
            ref = reference_bins(rows, W, B)
            for wm_steps in ((ticks,), (4, 5, 11, ticks), tuple(range(1, ticks + 1))):
                bins, wm = np.zeros(B, dtype=TBIN_DTYPE), 0
                for t in wm_steps:                 # a run paused at tick t: the records up to t, rows up to wm folded before
                    ne, nq = int((ev["now"] <= t).sum()), int((qr["now"] <= t).sum())
                    emu.emu_tl_compact(_p(ev[:ne]), C.c_int(ne), _p(qr[:nq]), C.c_int(nq), C.c_longlong(t), C.c_longlong(wm),
                                       C.c_longlong(W), C.c_int(B), _p(bins))
                    wm = t
                assert_bins(bins, ref, f"W={W} B={B} steps={len(wm_steps)}")


# ---------------------------------------------------------------- gs_horus_summarize's timeline through the host build of gs_horus.cu
@pytest.fixture(scope="module")
def horus_emu_engine():
    import importlib.util
    import sys
    spec = importlib.util.spec_from_file_location("tests_emu_timeline", os.path.join(REPO, "tests", "emu", "__init__.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["tests_emu_timeline"] = mod
    spec.loader.exec_module(mod)
    out = mod._ABI_OUT
    hdr = os.path.join(REPO, "gpuschedule_b200", "csrc", "gs_summary.cuh")
    if os.path.exists(out) and os.path.getmtime(out) < os.path.getmtime(hdr) and mod._abi_lib is None:
        mod.build_abi(force=True)                 # gs_summary.cuh is not among the emu build's own dependencies
    return mod.emu_engine_class()


def test_horus_timeline_host_build_matches_reference(horus_emu_engine):
    from gpuschedule_b200 import capi
    cases = horus_cases()
    loaded = [load_horus(c) for c in cases]
    with horus_emu_engine(device=0, nsims=len(cases)) as eng:
        for i, (table, cluster, params, _, _) in enumerate(loaded):
            eng.config(i, cluster, capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"]))
            eng.load_trace(i, table)
            np.random.seed(params["seed"])
            eng.load_words(i, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))
        for width, nbins in ((0, -1), (0, 4), (5, 1025), (2 ** 41, 4)):
            with pytest.raises(capi.GsError) as e:
                eng.set_timeline(width, nbins)
            assert e.value.code == capi.GS_ERR_ARG, (width, nbins)
        with pytest.raises(capi.GsError) as e:
            eng.timeline()
        assert e.value.code == capi.GS_ERR_STATE                      # off
        eng.set_timeline(7, 16)
        with pytest.raises(capi.GsError) as e:
            eng.timeline()
        assert e.value.code == capi.GS_ERR_STATE                      # nothing has run
        eng.run(rows_cap=1 << 15)
        with pytest.raises(capi.GsError) as e:
            eng.timeline()
        assert e.value.code == capi.GS_ERR_STATE                      # not summarised
        recs = eng.summarize()
        for width, nbins in ((7, 16), (3, 1024)):
            if nbins != 16:
                eng.set_timeline(width, nbins)
                with pytest.raises(capi.GsError) as e:
                    eng.timeline()
                assert e.value.code == capi.GS_ERR_STATE              # setting it asks for a new summary
                recs = eng.summarize()
            tl = eng.timeline()
            assert tl.shape == (len(cases), nbins)
            assert eng.timeline(first=2, count=3).tobytes() == tl[2:5].tobytes()
            for i, case in enumerate(cases):
                rows, util, _, _, _ = eng.fetch(i)
                assert_bins(tl[i], reference_bins(rows, width, nbins, util=util), f"{case} W={width} B={nbins}")
                assert int(tl[i]["rows"].sum()) == int(recs[i]["rows"])
                assert math.isclose(math.fsum(tl[i]["util_sum"].tolist()), float(recs[i]["util_sum"]), rel_tol=1e-12)
        eng.set_timeline(0, 0)
        with pytest.raises(capi.GsError) as e:
            eng.timeline()
        assert e.value.code == capi.GS_ERR_STATE


# ---------------------------------------------------------------- summary.timeline_derived / timeline_spread
def _bins(specs):
    """TBIN_DTYPE records from dicts (fields not given are 0)"""
    from gpuschedule_b200.capi import TBIN_DTYPE
    out = np.zeros(len(specs), dtype=TBIN_DTYPE)
    for i, d in enumerate(specs):
        for k, v in d.items():
            out[i][k] = v
    return out


def test_timeline_derived_on_hand_made_bins():
    from gpuschedule_b200 import summary
    M, G, cap = 4, 8, 32768
    b = _bins([dict(rows=4, busy_gpus_sum=64, running_sum=10, queued_sum=6, pending_rows=2, avg_pending_sum=9.0, util_sum=1.5,
                    delta_min=0, delta_max=3, finished_last=7, pend_max_max=12, mem_busy_lo=4 * 1048576 * 32 * cap // 2),
               dict(),
               dict(rows=2, busy_gpus_sum=32, pending_rows=0, delta_min=8, delta_max=9, finished_last=9, mem_busy_lo=5, mem_busy_hi=1,
                    util_sum=float("nan"))])
    d = summary.timeline_derived(b, M, G, cap)
    assert d["rows"].tolist() == [4, 0, 2]
    assert d["gpu_share"][0] == 64 / (4 * 32) and d["gpu_share"][2] == 32 / (2 * 32)
    assert d["running_mean"][0] == 2.5 and d["queued_mean"][0] == 1.5
    assert d["pending_mean_all"][0] == 9.0 / 4 and d["pending_mean_nz"][0] == 9.0 / 2
    assert math.isnan(d["pending_mean_nz"][2]) and d["pending_mean_all"][2] == 0.0
    assert d["mem_mean"][0] == 0.5
    assert d["mem_mean"][2] == float((1 << 64) + 5) / 1048576.0 / (32 * cap) / 2
    assert d["util_mean"][0] == 1.5 / 4 and math.isnan(d["util_mean"][2])
    assert d["pend_max"][0] == 12 and d["finished_last"].tolist()[0::2] == [7, 9]
    assert d["delta_min"].tolist()[0::2] == [0, 8] and d["delta_max"].tolist()[0::2] == [3, 9]
    for k, v in d.items():
        if k != "rows":
            assert math.isnan(v[1]), k                                   # the empty bin
    assert summary.timeline_flat(d, 0)[:3] == [0, 3, 4]


def test_timeline_spread_over_the_replicas_that_reach_a_bin():
    from gpuschedule_b200 import summary
    M, G, cap = 1, 4, 1024
    R, B = 5, 3
    specs = []
    for r in range(R):
        for b in range(B):
            if b == 2 and r >= 2:                # bin 2: only replicas 0 and 1 reach it
                specs.append(dict())
            elif b == 1 and r == 4:              # bin 1: replica 4 has rows but nothing pending
                specs.append(dict(rows=2, busy_gpus_sum=4, finished_last=3))
            else:
                specs.append(dict(rows=2, busy_gpus_sum=2 * (r + 1), pending_rows=1, avg_pending_sum=float(r + b), finished_last=r + b))
    bins = _bins(specs).reshape(R, B)
    sp = summary.timeline_spread(bins, M, G, cap, level=0.8)
    assert sp["replicas"].tolist() == [5, 5, 2]
    share = [(r + 1) / 4 for r in range(R)]
    assert math.isclose(sp["gpu_share"]["mean"][0], float(np.mean(share)))
    assert math.isclose(sp["gpu_share"]["std"][0], float(np.std(share, ddof=1)))
    ref = summary.spread([dict(makespan=0, rows=2, busy_gpus_sum=2 * (r + 1), mem_busy_lo=0, mem_busy_hi=0, avg_pending_sum=0.0,
                               pending_rows=1, wait_sum=0, turnaround_sum=0, jct_sum=0, finished=1, util_sum=0.0) for r in range(R)],
                         M, G, cap, level=0.8)["gpu_share"]
    assert [sp["gpu_share"][s][0] for s in ("mean", "std", "lo", "hi")] == pytest.approx([ref[s] for s in ("mean", "std", "lo", "hi")])
    assert sp["gpu_share"]["lo"][0] == share[0] and sp["gpu_share"]["hi"][0] == share[-1]
    assert math.isnan(sp["pending_mean_nz"]["mean"][1])                 # NaN for one reaching replica: NaN throughout
    assert sp["pending_mean_all"]["mean"][2] == pytest.approx(np.mean([2 / 2, 3 / 2]))
    assert sp["finished_last"]["mean"][2] == 2.5 and sp["finished_last"]["lo"][2] == 2 and sp["finished_last"]["hi"][2] == 3
    one = summary.timeline_spread(bins[:1], M, G, cap)
    assert one["replicas"].tolist() == [1, 1, 1] and math.isnan(one["gpu_share"]["std"][0])
    none = summary.timeline_spread(_bins([dict()] * 2).reshape(2, 1), M, G, cap)
    assert none["replicas"].tolist() == [0] and math.isnan(none["gpu_share"]["mean"][0])
    with pytest.raises(ValueError):
        summary.timeline_spread(bins[0], M, G, cap)
    with pytest.raises(ValueError):
        summary.timeline_spread(bins, M, G, cap, level=0)


# ---------------------------------------------------------------- sweep argument errors (before any engine exists)
def test_sweep_timeline_argument_errors(tmp_path, monkeypatch):
    from gpuschedule_b200 import capi, sweep

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(capi, "Engine", no_engine)
    monkeypatch.setattr(capi, "HorusEngine", no_engine)
    fl = [sweep.make_flags(trace_file=str(tmp_path / "missing.csv"))]
    for bad in ((0, 4), (4, 0), (4, 1025), (2 ** 41, 4), (4,), None.__class__, "ab"):
        with pytest.raises(ValueError):
            sweep.summarize_batched(fl, timeline=bad)
        with pytest.raises(ValueError):
            sweep.summarize_bootstrap(fl, 2, timeline=bad)
    assert sweep.check_timeline((3, 1024)) == (3, 1024)
    base = ["--trace", str(tmp_path / "missing.csv")]
    for argv in (["--timeline", "t.csv", "--bin-width", "4"],                                   # no --summary
                 ["--summary", "s.csv", "--timeline", "t.csv"],                                 # no --bin-width
                 ["--summary", "s.csv", "--bin-width", "4"], ["--summary", "s.csv", "--bins", "4"],   # no --timeline
                 ["--summary", "s.csv", "--timeline", "t.csv", "--bin-width", "0"],
                 ["--summary", "s.csv", "--timeline", "t.csv", "--bin-width", "4", "--bins", "0"],
                 ["--summary", "s.csv", "--timeline", "t.csv", "--bin-width", "4", "--bins", "1025"]):
        with pytest.raises(SystemExit) as e:
            sweep.main(base + argv)
        assert e.value.code == 2, argv
    assert not (tmp_path / "t.csv").exists() and not (tmp_path / "s.csv").exists()

"""Time-weighted occupancy (gs_occ and its histograms, gpuschedule_b200/csrc/gs_summary.cuh) on a box without a GPU.

The serial folds gs_occ_serial / gs_occ_records_serial are compiled with g++ (tests/emu/occupancy_emu.cpp) and compared
with `reference`, a restatement in Python ints over a run's rows: the pinned fifo oracle's rows, folded from the
compact records window by window; the event-driven policies' rows cut into windows at every position (the carry);
synthetic rows with equal and decreasing deltas; the horus fixtures through the host-emulation build of
gs_horus_summarize, with every error code.  summary.occupancy_derived against pandas, and the sweep's argument errors."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import REPO, golden_cases, horus_cases, load_golden, load_horus
from test_summary_cpu import _policy_cases, load_policy

EDGES = (0, 1, 2, 4, 8, 16, 64, 1024)
FIELDS = ("rows", "ticks", "busy_sum", "running_sum", "queued_sum", "wait_ticks", "idle_wait_sum", "running_max", "queued_max",
          "total_gpus")


# ---------------------------------------------------------------- the restatement (shared with test_gpu_occupancy.py)
def weights(rows, done, per_tick=False):
    """(weight of every row that has one, as Python ints; rows weighed) -- one tick each for fifo / horus rows, else
    max(0, delta_(i+1) - delta_i), the last row 1 when the run is done and not weighed yet otherwise"""
    n = len(rows)
    if per_tick:
        return [1] * n, n
    d = [int(x) for x in rows["now"]]
    w = [max(0, d[i + 1] - d[i]) for i in range(n - 1)]
    if n and done:
        w.append(1)
    return w, len(w)


def reference(rows, G, edges, done, per_tick=False):
    """(record dict, busy histograms [H_all, H_wait] (2, G + 1), queue histogram (E + 1)) of a run's rows"""
    w, k = weights(rows, done, per_tick)
    rec = dict.fromkeys(FIELDS, 0)
    rec["rows"], rec["total_gpus"] = k, G
    hb = np.zeros((2, G + 1), dtype=object)
    hb[:] = 0
    hq = [0] * (len(edges) + 1)
    for i in range(k):
        wi = w[i]
        if wi <= 0:
            continue
        b, r, q = int(rows["busy_gpus"][i]), int(rows["running"][i]), int(rows["queued"][i])
        rec["ticks"] += wi
        rec["busy_sum"] += wi * b
        rec["running_sum"] += wi * r
        rec["queued_sum"] += wi * q
        rec["running_max"] = max(rec["running_max"], r)
        rec["queued_max"] = max(rec["queued_max"], q)
        hb[0, b] += wi
        if q > 0:
            rec["wait_ticks"] += wi
            rec["idle_wait_sum"] += wi * (G - b)
            hb[1, b] += wi
        hq[sum(1 for e in edges if e < q)] += wi
    return rec, hb.astype(np.uint64), np.array(hq, dtype=np.uint64)


def assert_occ(rec, busy, queue, ref, tag=""):
    """a device / host-build record and histograms (busy: (2, >= G + 1)) against reference(...), and the invariants"""
    want, hb, hq = ref
    for f in FIELDS:
        assert int(rec[f]) == want[f], (tag, f, int(rec[f]), want[f])
    G = want["total_gpus"]
    assert np.array_equal(np.asarray(busy)[:, :G + 1], hb), tag
    assert not np.asarray(busy)[:, G + 1:].any(), tag
    assert np.array_equal(np.asarray(queue), hq), tag
    check_invariants(rec, busy, queue, tag)


def check_invariants(rec, busy, queue, tag=""):
    """the redundant fields equal the histogram sums"""
    T, G = int(rec["ticks"]), int(rec["total_gpus"])
    b = np.asarray(busy, dtype=np.uint64)[:, :G + 1].astype(object)
    vals = np.arange(G + 1, dtype=object)
    assert int(b[0].sum()) == T and int(np.asarray(queue, dtype=np.uint64).sum()) == T, tag
    assert int(b[1].sum()) == int(rec["wait_ticks"]), tag
    assert int((b[0] * vals).sum()) == int(rec["busy_sum"]), tag
    assert int((b[1] * (G - vals)).sum()) == int(rec["idle_wait_sum"]), tag


# ---------------------------------------------------------------- host build of the folds
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("occupancy_emu") / "liboccupancy_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "occupancy_emu.cpp")], check=True)
    return C.CDLL(out)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class HostFold:
    """one replica's record, carry and histograms in the host build"""

    def __init__(self, lib, G, edges=EDGES):
        from gpuschedule_b200.capi import OCC_DTYPE
        self.lib, self.G = lib, G
        self.edges = np.ascontiguousarray(edges, dtype=np.int32)
        self.rec = np.zeros(1, dtype=OCC_DTYPE)
        self.carry = np.zeros(24, dtype=np.uint8)
        self.busy = np.zeros((2, G + 1), dtype=np.uint64)
        self.queue = np.zeros(len(edges) + 1, dtype=np.uint64)

    def rows(self, rows, lo, hi, done, per_tick=False):
        rows = np.ascontiguousarray(rows)
        self.lib.emu_occ_rows(_p(self.rec), _p(self.carry), _p(self.busy), _p(self.queue), C.c_int(len(self.edges)), _p(self.edges),
                              _p(rows), C.c_longlong(lo), C.c_longlong(hi), C.c_int(int(done)), C.c_int(int(per_tick)), C.c_int(self.G))

    def records(self, ev, ticks, wm):
        self.lib.emu_occ_records(_p(self.rec), _p(self.busy), _p(self.queue), C.c_int(len(self.edges)), _p(self.edges), _p(ev),
                                 C.c_int(len(ev)), C.c_longlong(ticks), C.c_longlong(wm), C.c_int(self.G))

    def check(self, ref, tag=""):
        assert_occ(self.rec[0], self.busy, self.queue, ref, tag)


def test_queue_edge_setting(emu):
    ok = lambda e: emu.emu_occ_cfg(C.c_int(len(e)), _p(np.ascontiguousarray(e, dtype=np.int32)) if len(e) else None)
    assert ok([]) == 1 and ok([0]) == 1 and ok(list(range(255))) == 1 and ok([0, 1, 2 ** 31 - 1]) == 1
    assert ok([-1, 0]) == 0 and ok([1, 1]) == 0 and ok([2, 1]) == 0 and ok(list(range(256))) == 0
    assert emu.emu_occ_cfg(C.c_int(2), None) == 0


def _gpus(cluster):
    return cluster.num_switch * cluster.num_node_p_switch * cluster.num_gpu_p_node


# ---------------------------------------------------------------- fifo: the compact records, window by window
def fold_fifo_windows(lib, t2, G, **run_kw):
    """restart the Tight2 yardstick and fold every window's records as gs_summarize does after every gs_run (twice:
    the second fold adds nothing)"""
    f = HostFold(lib, G)
    t2.restart()
    wm, windows = 0, 0
    while True:
        rc, w, _, _, done = t2.run_window(**run_kw)
        assert rc == 0
        ev = t2.ev[:w.ev_rows].copy()
        for _ in range(2):
            f.records(ev, int(w.ticks), wm)
            wm = max(wm, int(w.ticks))
        windows += 1
        if done or t2.n == 0:
            return f, windows


@pytest.mark.parametrize("case", golden_cases())
def test_fifo_records_window_by_window(emu, case):
    import oracle
    table, cluster, _, _, _ = load_golden(case)
    if cluster.enable_network_costs:
        pytest.skip("the record yardstick runs the plain fifo + yarn tick only (no network-cost branch)")
    G = _gpus(cluster)
    res = oracle.run_fifo(cluster, table, want_spans=False)
    ref = reference(res.rows, G, EDGES, True, per_tick=True)
    t2 = oracle.Tight2(cluster, table)
    for kw, tag in ((dict(), "one window"), (dict(max_ticks=7), "7-tick windows"), (dict(max_ticks=1), "1-tick windows"),
                    (dict(cap_a=1, cap_b=1), "one record per window")):
        f, nw = fold_fifo_windows(emu, t2, G, **kw)
        assert (nw == 1) == (tag == "one window"), (tag, nw)
        f.check(ref, f"{case} {tag}")
    # the Little's-law identity of the fifo rows: a job is queued on the rows arrive + 1 .. start (or .. ticks)
    st = res.recs["start"].astype(np.int64)
    a = np.asarray(table.arrive_tick, dtype=np.int64)
    T = int(res.ticks)
    want = int(np.maximum(0, np.where(st >= 0, np.minimum(st, T), T) - a).sum())
    assert ref[0]["queued_sum"] == want, case


# ---------------------------------------------------------------- event-driven policies: windows cut at every row
@pytest.mark.parametrize("case", _policy_cases())
def test_policy_rows_in_windows(emu, case):
    import oracle
    table, cluster, pol = load_policy(case)
    rows = oracle.run_policy(cluster, pol, table).rows
    G = _gpus(cluster)
    whole = reference(rows, G, EDGES, True)
    n = len(rows)
    cuts_list = [(n,), (n // 3, n), tuple(range(1, n + 1))] if n <= 400 else [(n,), (n // 3, n), tuple(range(1, n + 1, 7)) + (n,)]
    for cuts in cuts_list:
        f, lo = HostFold(emu, G), 0
        for k in cuts:
            f.rows(rows, lo, k, done=k == n)
            f.rows(rows, k, k, done=k == n)              # a second summarize of the same window adds nothing
            if k < n and len(cuts) < 10:
                f.check(reference(rows[:k], G, EDGES, False), f"{case} prefix {k}")
            lo = k
        f.check(whole, f"{case} {len(cuts)} windows")


def _rows(deltas, busy, queued, running=None):
    from gpuschedule_b200.log_manager import ROW_DTYPE
    r = np.zeros(len(deltas), dtype=ROW_DTYPE)
    r["now"], r["busy_gpus"], r["queued"] = deltas, busy, queued
    r["running"] = running if running is not None else np.minimum(busy, 3)
    return r


def test_synthetic_equal_and_decreasing_deltas(emu):
    """dlas can emit rows whose delta goes backwards: such a row, and a row followed by one with the same delta, weigh 0"""
    rows = _rows([1, 4, 4, 9, 7, 8, 8, 20, 15, 30], [0, 8, 6, 16, 16, 3, 16, 0, 5, 2], [0, 2, 0, 5, 1, 0, 3, 0, 7, 4])
    w, _ = weights(rows, True)
    assert w == [3, 0, 5, 0, 1, 0, 12, 0, 15, 1]
    ref = reference(rows, 16, EDGES, True)
    assert ref[0]["ticks"] == 37 and ref[0]["rows"] == 10
    for cuts in [(10,), tuple(range(1, 11)), (2, 3, 5, 10), (0, 4, 4, 10)]:
        f, lo = HostFold(emu, 16), 0
        for k in cuts:
            f.rows(rows, lo, k, done=k == 10)
            lo = k
        f.check(ref, f"cuts {cuts}")
    f = HostFold(emu, 16)
    f.rows(rows, 0, 10, done=False)                       # unfinished: the last row waits in the carry
    f.check(reference(rows, 16, EDGES, False), "unfinished")
    f.rows(rows, 10, 10, done=True)                       # the run ends without a new row: the carry weighs 1
    f.check(ref, "done later")
    f.rows(rows, 10, 10, done=True)
    f.check(ref, "done twice")


def test_per_tick_rows_and_saturation(emu):
    rows = _rows(np.arange(1, 9), [4, 4, 4, 4, 2, 4, 0, 4], [0, 3, 3, 9, 1, 0, 0, 2])
    f = HostFold(emu, 4)
    f.rows(rows, 0, 8, done=True, per_tick=True)
    ref = reference(rows, 4, EDGES, True, per_tick=True)
    f.check(ref)
    assert int(f.busy[0, 4]) == 6 and ref[0]["idle_wait_sum"] == 2


# ---------------------------------------------------------------- gs_horus_summarize through the host build of gs_horus.cu
@pytest.fixture(scope="module")
def horus_emu_engine():
    import importlib.util
    import sys
    spec = importlib.util.spec_from_file_location("tests_emu_occupancy", os.path.join(REPO, "tests", "emu", "__init__.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["tests_emu_occupancy"] = mod
    spec.loader.exec_module(mod)
    out = mod._ABI_OUT
    hdr = os.path.join(REPO, "gpuschedule_b200", "csrc", "gs_summary.cuh")
    if os.path.exists(out) and os.path.getmtime(out) < os.path.getmtime(hdr) and mod._abi_lib is None:
        mod.build_abi(force=True)                 # gs_summary.cuh is not among the emu build's own dependencies
    return mod.emu_engine_class()


def _horus_engine(cls, case, nsims=1):
    from gpuschedule_b200 import capi
    table, cluster, params, _, _ = load_horus(case)
    eng = cls(device=0, nsims=nsims)
    hp = capi.make_horus_params(params["scheme"], params["schedule"], params["num_buffer"], params["num_queue"])
    for s in range(nsims):
        eng.config(s, cluster, hp)
        eng.load_trace(s, table)
        np.random.seed(params["seed"])
        eng.load_words(s, np.random.randint(0, 2 ** 32, size=6 << 20, dtype=np.uint32))
    return eng, table, cluster, params


@pytest.mark.parametrize("case", horus_cases())
def test_horus_host_build(horus_emu_engine, case):
    eng, table, cluster, params = _horus_engine(horus_emu_engine, case)
    eng.set_occupancy(EDGES)
    eng.run(rows_cap=1 << 15)
    s1 = eng.summarize()
    rec, busy, queue = eng.occupancy()
    rows = eng.fetch(0)[0]
    assert len(rows) == int(s1[0]["rows"]) > 0
    assert_occ(rec[0], busy[0], queue[0], reference(rows, _gpus(cluster), EDGES, True, per_tick=True), case)
    assert int(rec[0]["ticks"]) == int(s1[0]["rows"]) and int(rec[0]["busy_sum"]) == int(s1[0]["busy_gpus_sum"])
    s2 = eng.summarize()
    again = eng.occupancy()
    assert s1.tobytes() == s2.tobytes() and rec.tobytes() == again[0].tobytes() and busy.tobytes() == again[1].tobytes()
    eng.close()


def test_horus_error_codes(horus_emu_engine):
    from gpuschedule_b200 import capi
    case = horus_cases()[0]
    eng, table, cluster, params = _horus_engine(horus_emu_engine, case, nsims=2)
    for bad in ([1, 1], [-1], list(range(256))):
        with pytest.raises(capi.GsError) as e:
            eng.set_occupancy(bad)
        assert e.value.code == capi.GS_ERR_ARG
    assert eng.lib.gs_horus_set_occupancy(eng.h, 1, 3, None) == capi.GS_ERR_ARG
    with pytest.raises(capi.GsError) as e:
        eng.occupancy()
    assert e.value.code == capi.GS_ERR_STATE                  # off
    eng.set_occupancy(EDGES)
    with pytest.raises(capi.GsError) as e:
        eng.occupancy()
    assert e.value.code == capi.GS_ERR_STATE                  # not run
    eng.run(rows_cap=1 << 15)
    with pytest.raises(capi.GsError) as e:
        eng.occupancy()
    assert e.value.code == capi.GS_ERR_STATE                  # not summarised
    eng.summarize()
    G = _gpus(cluster)
    busy = np.zeros((2, 2, G + 1), dtype=np.uint64)
    assert eng.lib.gs_horus_fetch_occupancy(eng.h, 0, 2, None, busy.ctypes.data_as(C.c_void_p), G, None) == capi.GS_ERR_CAPACITY
    assert eng.lib.gs_horus_fetch_occupancy(eng.h, 0, 3, None, None, 0, None) == capi.GS_ERR_ARG
    assert eng.lib.gs_horus_fetch_occupancy(eng.h, 0, 2, None, busy.ctypes.data_as(C.c_void_p), G + 1, None) == 0
    eng.set_occupancy(None)
    with pytest.raises(capi.GsError) as e:
        eng.occupancy()
    assert e.value.code == capi.GS_ERR_STATE
    eng.close()


# ---------------------------------------------------------------- derived numbers against pandas
@pytest.mark.parametrize("case", _policy_cases()[:3] + ["fifo:" + c for c in golden_cases()[:3]])
def test_derived_matches_pandas(emu, case):
    import pandas as pd

    import oracle
    from gpuschedule_b200 import summary
    if case.startswith("fifo:"):
        table, cluster, _, _, _ = load_golden(case[5:])
        rows = oracle.run_fifo(cluster, table, want_spans=False).rows
        per_tick = True
    else:
        table, cluster, pol = load_policy(case)
        rows = oracle.run_policy(cluster, pol, table).rows
        per_tick = False
    G = _gpus(cluster)
    f = HostFold(emu, G)
    f.rows(rows, 0, len(rows), done=True, per_tick=per_tick)
    d = summary.occupancy_derived(f.rec[0], f.busy, f.queue, EDGES)
    df = pd.DataFrame({"delta": rows["now"], "busy": rows["busy_gpus"], "running": rows["running"], "queued": rows["queued"]})
    w = pd.Series(1, index=df.index) if per_tick else (-df.delta.diff(-1)).clip(lower=0).fillna(1)
    T = w.sum()
    assert d["gpu_share"] == pytest.approx((w * df.busy).sum() / (T * G), rel=1e-12)
    assert d["running_mean"] == pytest.approx((w * df.running).sum() / T, rel=1e-12)
    assert d["queued_mean"] == pytest.approx((w * df.queued).sum() / T, rel=1e-12)
    assert d["saturated_share"] == pytest.approx(w[df.busy == G].sum() / T, rel=1e-12, abs=1e-15)
    wq = w[df.queued > 0]
    assert d["wait_share"] == pytest.approx(wq.sum() / T, rel=1e-12, abs=1e-15)
    idle = (w * (G - df.busy))[df.queued > 0].sum()
    assert d["idle_wait_share"] == pytest.approx(idle / (T * G), rel=1e-12, abs=1e-15)
    if wq.sum() > 0:
        assert d["idle_in_wait_share"] == pytest.approx(idle / (wq.sum() * G), rel=1e-12)
    expanded = np.repeat(df.busy.to_numpy(), w.astype(int).to_numpy())
    srt = np.sort(expanded)
    for q in summary.QUANTILES:
        assert d[f"busy_p{q}"] == srt[summary.nearest_rank(q / 100, len(srt))], q
    for i, e in enumerate(EDGES):
        assert d["queue_cdf"][i] == pytest.approx(w[df.queued <= e].sum() / T, rel=1e-12, abs=1e-15)
    sp = summary.occupancy_spread(np.stack([f.rec[0]] * 3), np.stack([f.busy] * 3), np.stack([f.queue] * 3), EDGES)
    assert sp["gpu_share"]["mean"] == pytest.approx(d["gpu_share"]) and sp["gpu_share"]["lo"] == pytest.approx(d["gpu_share"])


# ---------------------------------------------------------------- the sweep's argument errors
@pytest.mark.parametrize("argv", [
    ["--occupancy", "o.csv"],                                               # needs --summary
    ["--summary", "s.csv", "--queue-edges", "0", "1"],                       # needs --occupancy
    ["--summary", "s.csv", "--occupancy-cdf", "c.csv"],
    ["--summary", "s.csv", "--occupancy", "o.csv", "--queue-edges", "2", "1"],
    ["--summary", "s.csv", "--occupancy", "o.csv", "--queue-edges", "-1", "1"],
    ["--summary", "s.csv", "--occupancy", "o.csv", "--queue-edges"] + [str(i) for i in range(256)],
])
def test_cli_argument_errors(argv, tmp_path, capsys):
    from gpuschedule_b200 import sweep
    with pytest.raises(SystemExit) as e:
        sweep.main(["--trace", str(tmp_path / "missing.csv")] + argv)
    assert e.value.code == 2
    assert "missing.csv" not in capsys.readouterr().err

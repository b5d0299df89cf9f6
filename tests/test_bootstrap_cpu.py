"""Bootstrap replicas (gs_boot_traces, gpuschedule_b200/csrc/gs_boot.cuh) on a box without a GPU.

The numpy mirror in tracegen is checked against numpy's own Philox4x64-10, the __host__ __device__ part of gs_boot.cuh
is compiled with g++ (tests/emu/boot_emu.cpp) and must make byte-identical traces, and summary.spread and the sweep's
argument checks are checked on the host."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, REPO

U64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("boot_emu") / "libboot_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "boot_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.emu_boot_mulhi.restype = C.c_ulonglong
    lib.emu_boot_mulhi.argtypes = [C.c_ulonglong, C.c_ulonglong]
    lib.emu_boot_philox.argtypes = [C.c_ulonglong, C.c_ulonglong, C.c_void_p, C.c_void_p]
    lib.emu_boot_arrive_bound.restype = C.c_longlong
    lib.emu_boot_arrive_bound.argtypes = [C.c_longlong, C.c_longlong, C.c_int, C.c_int]
    lib.emu_boot_trace.restype = C.c_int
    lib.emu_boot_trace.argtypes = [C.c_void_p, C.c_longlong, C.c_ulonglong, C.c_ulonglong, C.c_longlong, C.c_int, C.c_int, C.c_int,
                                   C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    return lib


def make_population(k, seed, zero_gaps=False):
    """k records under the load rules: arrivals non-decreasing from 0 (many equal ticks), gpus a multiple of gpu_per_task"""
    from gpuschedule_b200.capi import JOBIN_DTYPE
    rng = np.random.default_rng(seed)
    p = np.zeros(k, dtype=JOBIN_DTYPE)
    gaps = np.zeros(k, dtype=np.int64) if zero_gaps else rng.choice([0, 0, 0, 1, 2, 7], size=k)
    gaps[0] = 0
    p["arrive_tick"] = np.cumsum(gaps)
    gpc = rng.choice([1, 2, 4], size=k)
    p["gpu_per_task"] = gpc
    p["gpus"] = gpc * rng.choice([1, 2, 3, 8, 40], size=k)
    p["mem_bytes"] = rng.integers(0, 1 << 34, size=k)
    p["duration"] = np.round(rng.uniform(0.5, 5000.0, size=k), 3)
    return p


# ---------------------------------------------------------------- the generator and the high-word multiply
def test_philox_matches_numpy():
    from gpuschedule_b200 import tracegen
    rng = np.random.default_rng(5)
    edge = [0, 1, 2, U64, U64 - 1, 1 << 63, (1 << 32) - 1, 1 << 32]
    cases = 0
    for t in range(1200):
        key = [int(x) for x in rng.integers(0, 1 << 64, size=2, dtype=np.uint64)]
        ctr = [int(x) for x in rng.integers(0, 1 << 64, size=4, dtype=np.uint64)]
        if t < 64:                                     # words 0 and 2^64 - 1 (and their neighbours) in keys and counters
            key = [edge[t % 8], edge[(t // 8) % 8]]
            ctr = [edge[(t + i) % 8] for i in range(4)]
        want = np.random.Philox(key=np.array(key, dtype=np.uint64), counter=np.array(ctr, dtype=np.uint64)).random_raw(4)
        c = sum(v << (64 * i) for i, v in enumerate(ctr)) + 1      # numpy increments the 256-bit counter first
        nxt = [(c >> (64 * i)) & U64 for i in range(4)]
        got = tracegen.philox4x64(key[0], key[1], np.array([nxt], dtype=np.uint64))[0]
        assert got.tolist() == want.tolist(), (key, ctr)
        cases += 1
    assert cases >= 1000


def test_philox_host_build_matches_mirror(emu):
    from gpuschedule_b200 import tracegen
    rng = np.random.default_rng(6)
    ctr = rng.integers(0, 1 << 64, size=(300, 4), dtype=np.uint64)
    ctr[:8] = [[0, 0, 0, 0], [U64] * 4, [U64, 0, U64, 0], [0, U64, 0, U64], [1, 0, 0, 0], [U64, U64, 0, 0], [0, 0, U64, U64], [1, 2, 3, 4]]
    for i, c in enumerate(ctr):
        k0, k1 = (0, U64) if i % 3 == 0 else (int(c[3]) ^ 12345, int(c[0]))
        out = np.zeros(4, dtype=np.uint64)
        emu.emu_boot_philox(k0, k1, np.ascontiguousarray(c).ctypes.data, out.ctypes.data)
        assert out.tolist() == tracegen.philox4x64(k0, k1, c[None, :])[0].tolist()


def test_mulhi_edge_values(emu):
    from gpuschedule_b200 import tracegen
    vals = [0, 1, 2, 3, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, (1 << 63) - 1, 1 << 63, U64 - 1, U64, 0xD2E7470EE14C6C93, 0xCA5A826395121157]
    rng = np.random.default_rng(7)
    vals += [int(x) for x in rng.integers(0, 1 << 64, size=20, dtype=np.uint64)]
    a = np.array([x for x in vals for _ in vals], dtype=np.uint64)
    b = np.array([y for _ in vals for y in vals], dtype=np.uint64)
    want = [(int(x) * int(y)) >> 64 for x, y in zip(a.tolist(), b.tolist())]
    assert tracegen.mulhi64(a, b).tolist() == want
    assert [emu.emu_boot_mulhi(int(x), int(y)) for x, y in zip(a.tolist(), b.tolist())] == want


def test_arrive_bound_is_exact(emu):
    for n, g, num, den in ((0, 5, 1, 1), (1, 10 ** 9, 65535, 1), (2, 2 ** 31 - 1, 1, 1), (2 ** 31 - 65, 2 ** 31 - 1, 2 ** 31 - 1, 1),
                           (100000, 3, 7, 3), (100000, 21475, 1, 1), (100000, 21475, 65535, 65534)):
        want = (n - 1) * g * num // den if n > 1 else 0
        assert emu.emu_boot_arrive_bound(n, g, num, den) == min(want, 2 ** 63 - 1)


# ---------------------------------------------------------------- host build of the trace generator vs the numpy mirror
POPULATIONS = [(1, False), (2, False), (3, False), (1000, False), (1000, True), ((1 << 20) + 7, False)]
NS = (0, 1, 255, 256, 257, 100000)
SCALES = ((0, 1), (1, 1), (1, 2), (7, 3), (65535, 1))


@pytest.mark.parametrize("k,zero_gaps", POPULATIONS)
def test_host_build_traces_match_mirror(emu, k, zero_gaps):
    from gpuschedule_b200 import tracegen
    from gpuschedule_b200.capi import JOBIN_DTYPE
    pop = make_population(k, seed=k, zero_gaps=zero_gaps)
    gaps = np.diff(pop["arrive_tick"].astype(np.int64))
    max_gap = int(gaps.max()) if len(gaps) else 0
    checked = 0
    for n in NS:
        for num, den in SCALES:
            seed, stream = (k * 7919 + n) & U64, U64 - n
            out = np.zeros(max(n, 1), dtype=JOBIN_DTYPE)
            spans, last = C.c_longlong(0), C.c_longlong(0)
            rc = emu.emu_boot_trace(pop.ctypes.data, k, seed, stream, n, num, den, 16, out.ctypes.data, C.byref(spans), C.byref(last))
            if n > 1 and (n - 1) * max_gap * num // den >= 2 ** 31 - 1:
                assert rc == -1
                with pytest.raises(ValueError):
                    tracegen.bootstrap_packed(pop, seed, stream, n, num, den)
                continue
            assert rc == 0
            want, rows = tracegen.bootstrap_packed(pop, seed, stream, n, num, den)
            assert out[:n].tobytes() == want.tobytes(), (k, n, num, den)
            assert spans.value == int(np.minimum(want["gpus"] // want["gpu_per_task"], 16).sum())
            assert last.value == (int(want["arrive_tick"][-1]) if n else 0)
            assert (np.diff(want["arrive_tick"].astype(np.int64)) >= 0).all()
            checked += 1
    assert checked >= 20


def test_mirror_definition():
    """the mirror against the definition written out with Python integers"""
    from gpuschedule_b200 import tracegen
    pop = make_population(37, seed=3)
    seed, stream, n, num, den = 99, 4, 300, 7, 3
    recs, rows = tracegen.bootstrap_packed(pop, seed, stream, n, num, den)
    S = 0
    for j in range(n):
        w = np.random.Philox(key=[seed, stream], counter=[j, 0, 0, 0]).random_raw(4).tolist()
        r = (w[0] * 37) >> 64
        if j:
            i = (w[1] * 36) >> 64
            S += int(pop["arrive_tick"][i + 1]) - int(pop["arrive_tick"][i])
        assert rows[j] == r
        assert recs["arrive_tick"][j] == S * num // den
        for f in ("gpus", "gpu_per_task", "mem_bytes", "duration"):
            assert recs[f][j] == pop[f][r]
        assert recs["ps_count"][j] == 0


def test_common_random_numbers_across_loads():
    from gpuschedule_b200 import tracegen
    pop = make_population(500, seed=8)
    a, ra = tracegen.bootstrap_packed(pop, 1, 2, 1000, 1, 1)
    b, rb = tracegen.bootstrap_packed(pop, 1, 2, 1000, 1, 2)
    c, rc = tracegen.bootstrap_packed(pop, 1, 3, 1000, 1, 1)
    assert np.array_equal(ra, rb) and np.array_equal(a["arrive_tick"] // 2, b["arrive_tick"])
    assert not np.array_equal(ra, rc)


def test_bootstrap_table_packs_to_the_mirror():
    from gpuschedule_b200 import ingest, tracegen
    base = ingest.JobTraceReader(os.path.join(GOLDEN, "kat0", "trace.csv")).prepare_jobs().table(0.5)
    for n, num, den in ((0, 1, 1), (1, 1, 1), (257, 1, 2), (1000, 7, 3)):
        t = tracegen.bootstrap_table(base, 5, n, n, num, den)
        want, rows = tracegen.bootstrap_packed(base.packed(), 5, n, n, num, den)
        assert t.n == n and t.packed().tobytes() == want.tobytes()
        assert t.label == [str(i) for i in range(n)]
        assert t.num_gpu_text == [base.num_gpu_text[r] for r in rows.tolist()]
        assert np.array_equal(t.submit, t.arrive_tick)
        assert np.array_equal(t.util_avg, base.util_avg[rows]) and np.array_equal(t.util_max, base.util_max[rows])


# ---------------------------------------------------------------- summary.spread
def synthetic_records(k, seed):
    from gpuschedule_b200.capi import SUMMARY_DTYPE
    rng = np.random.default_rng(seed)
    r = np.zeros(k, dtype=SUMMARY_DTYPE)
    r["rows"] = rng.integers(100, 10000, size=k)
    r["makespan"] = r["rows"]
    r["busy_gpus_sum"] = rng.integers(0, 1 << 40, size=k)
    r["mem_busy_lo"] = rng.integers(0, 1 << 63, size=k, dtype=np.uint64)
    r["mem_busy_hi"] = rng.integers(0, 4, size=k, dtype=np.uint64)
    r["pending_rows"] = rng.integers(1, 100, size=k)
    r["avg_pending_sum"] = rng.uniform(0, 1e6, size=k)
    r["finished"] = rng.integers(1, 1000, size=k)
    for f in ("wait_sum", "turnaround_sum", "jct_sum"):
        r[f] = rng.integers(0, 1 << 30, size=k)
    r["util_sum"] = rng.uniform(0, 1e4, size=k)
    return r


@pytest.mark.parametrize("k", [1, 2, 3, 7, 40, 100, 1000])
def test_spread_matches_numpy(k):
    from gpuschedule_b200 import summary
    recs = synthetic_records(k, seed=k)
    shape = (128, 8, 32 * 1024)
    for level in (0.95, 0.9, 0.5, 1.0):
        sp = summary.spread(recs, *shape, level=level)
        assert set(sp) == set(summary.SPREAD_METRICS)
        for m in summary.SPREAD_METRICS:
            v = np.array([float(r["makespan"]) if m == "makespan" else summary.derived(r, *shape)[m] for r in recs])
            s = np.sort(v)
            lo_q, hi_q = round((1 - level) / 2 * 1000), round((1 + level) / 2 * 1000)
            lo = s[max((lo_q * k + 999) // 1000 - 1, 0)]             # gs_summary's nearest rank, per mille
            hi = s[max((hi_q * k + 999) // 1000 - 1, 0)]
            assert sp[m]["mean"] == pytest.approx(v.mean(), rel=1e-12)
            if k > 1:
                assert sp[m]["std"] == pytest.approx(np.std(v, ddof=1), rel=1e-9)
            else:
                assert math.isnan(sp[m]["std"])
            assert (sp[m]["lo"], sp[m]["hi"]) == (lo, hi), (m, level)
    flat = summary.spread_flat(sp)
    assert len(flat) == len(summary.spread_columns()) == 4 * len(summary.SPREAD_METRICS)
    assert dict(zip(summary.spread_columns(), flat))["jct_mean_hi"] == sp["jct_mean"]["hi"]


def test_spread_nan_metric():
    from gpuschedule_b200 import summary
    recs = synthetic_records(5, seed=1)
    recs["util_sum"][2] = np.nan
    recs["finished"][0] = 0
    sp = summary.spread(recs, 128, 8, 32 * 1024)
    assert all(math.isnan(sp["util_mean"][s]) for s in summary.SPREAD_STATS)
    assert all(math.isnan(sp["wait_mean"][s]) for s in summary.SPREAD_STATS)
    assert not math.isnan(sp["makespan"]["mean"])


# ---------------------------------------------------------------- the sweep's argument errors come before any engine
def test_bootstrap_argument_errors_before_any_engine(monkeypatch, tmp_path):
    from gpuschedule_b200 import capi, sweep

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(capi, "Engine", no_engine)
    monkeypatch.setattr(capi, "HorusEngine", no_engine)
    monkeypatch.setattr(sweep, "_plain_setup", no_engine)
    trace = os.path.join(GOLDEN, "kat0", "trace.csv")
    fifo = sweep.make_flags(trace_file=trace)
    horus = sweep.make_flags(trace_file=trace, scheme="horus", schedule="horus")
    for args, kw in (([fifo, horus], {}), ([fifo], dict(replicas=0)), ([fifo], dict(loads=[])), ([fifo], dict(loads=[0.0])),
                     ([fifo], dict(loads=[-1.0])), ([fifo], dict(loads=[float("nan")])), ([fifo], dict(n=-1))):
        kw = {"replicas": 2, **kw}
        with pytest.raises(ValueError):
            sweep.summarize_bootstrap(args, **kw)
    out = str(tmp_path / "s.csv")
    for argv in (["--trace", trace, "--bootstrap", "4"],
                 ["--trace", trace, "--bootstrap", "4", "--summary", out, "--schedule", "fifo", "horus"],
                 ["--trace", trace, "--bootstrap", "0", "--summary", out],
                 ["--trace", trace, "--bootstrap", "4", "--summary", out, "--load", "0"],
                 ["--trace", trace, "--bootstrap", "4", "--summary", out, "--repeats", "3"],
                 ["--trace", trace, "--load", "2", "--summary", out],
                 ["--trace", trace, "--summary-ci", out]):
        with pytest.raises(SystemExit) as e:
            sweep.main(argv)
        assert e.value.code == 2, argv
    assert not os.path.exists(out)


def test_load_gap_scale():
    from gpuschedule_b200 import sweep
    assert sweep.load_gap_scale(1.0) == (1, 1)
    assert sweep.load_gap_scale(2.0) == (1, 2)
    assert sweep.load_gap_scale(0.5) == (2, 1)
    assert sweep.load_gap_scale(1.5) == (2, 3)
    num, den = sweep.load_gap_scale(0.7)
    assert den <= 65535 and abs(num / den - 1 / 0.7) < 1e-8

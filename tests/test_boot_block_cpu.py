"""Block bootstrap replicas (gs_boot_traces_blocked, gpuschedule_b200/csrc/gs_boot.cuh) on a box without a GPU.

The numpy mirror tracegen.bootstrap_packed(..., block_len=L) is checked against the definition written out with Python
integers and against hand-worked cases; with L = 1 it must give today's iid replicas byte for byte; the blocked path of
gs_boot.cuh, compiled with g++ in the kernel's chunked structure (tests/emu/boot_block_emu.cpp), must make
byte-identical traces; and the sweep's --block-len argument checks and output columns are checked on the host."""
import csv
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, REPO

U64 = (1 << 64) - 1
LMAX = 2 ** 32 - 1


def _compile(tmp_path_factory, name):
    out = str(tmp_path_factory.mktemp(name) / f"lib{name}.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", f"{name}.cpp")], check=True)
    return C.CDLL(out)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = _compile(tmp_path_factory, "boot_block_emu")
    lib.emu_boot_block_trace.restype = C.c_int
    lib.emu_boot_block_trace.argtypes = [C.c_void_p, C.c_longlong, C.c_ulonglong, C.c_ulonglong, C.c_longlong, C.c_int, C.c_int,
                                         C.c_uint, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    return lib


@pytest.fixture(scope="module")
def iid_emu(tmp_path_factory):
    """the host build of today's iid kernel path"""
    lib = _compile(tmp_path_factory, "boot_emu")
    lib.emu_boot_trace.restype = C.c_int
    lib.emu_boot_trace.argtypes = [C.c_void_p, C.c_longlong, C.c_ulonglong, C.c_ulonglong, C.c_longlong, C.c_int, C.c_int, C.c_int,
                                   C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    return lib


def make_population(k, seed, zero_gaps=False):
    """k records under the load rules: arrivals non-decreasing from 0, gaps of distinct sizes so a wrong gap shows"""
    from gpuschedule_b200.capi import JOBIN_DTYPE
    rng = np.random.default_rng(seed)
    p = np.zeros(k, dtype=JOBIN_DTYPE)
    gaps = np.zeros(k, dtype=np.int64) if zero_gaps else rng.choice([0, 0, 1, 2, 7, 30, 411], size=k)
    gaps[0] = 0
    p["arrive_tick"] = np.cumsum(gaps)
    gpc = rng.choice([1, 2, 4], size=k)
    p["gpu_per_task"] = gpc
    p["gpus"] = gpc * rng.choice([1, 2, 3, 8, 40], size=k)
    p["mem_bytes"] = rng.integers(0, 1 << 34, size=k)
    p["duration"] = np.round(rng.uniform(0.5, 5000.0, size=k), 3)
    return p


def words(seed, stream, j):
    key = np.array([seed, stream], dtype=np.uint64)
    return np.random.Philox(key=key, counter=np.array([j, 0, 0, 0], dtype=np.uint64)).random_raw(4).tolist()


def definition(pop, seed, stream, n, num, den, L):
    """the block bootstrap written out with Python integers: (arrivals, rows)"""
    K = len(pop)
    D = [int(pop["arrive_tick"][i + 1]) - int(pop["arrive_tick"][i]) for i in range(K - 1)]
    S, b, arrivals, rows = 0, 0, [], []
    for j in range(n):
        w = words(seed, stream, j)
        start = j == 0 or (w[2] * L) >> 64 == 0
        if start:
            b = j
            s = (w[0] * K) >> 64
        r = (s + (j - b)) % K
        if j > 0:
            S += D[(w[1] * (K - 1)) >> 64] if (start or r == 0) and K > 1 else (D[r - 1] if K > 1 else 0)
        arrivals.append(S * num // den)
        rows.append(r)
    return arrivals, rows


def iid_reference(population, seed, stream, n, gap_num=1, gap_den=1):
    """tracegen.bootstrap_packed as it was before block lengths: every job draws its row and its gap independently"""
    from gpuschedule_b200 import tracegen
    from gpuschedule_b200.capi import JOBIN_DTYPE
    pop = np.ascontiguousarray(population, dtype=JOBIN_DTYPE)
    k = len(pop)
    gaps = np.diff(pop["arrive_tick"].astype(np.int64))
    ctr = np.zeros((n, 4), dtype=np.uint64)
    ctr[:, 0] = np.arange(1, n + 1, dtype=np.uint64)
    w = tracegen.philox4x64(seed, stream, ctr)
    rows = tracegen.mulhi64(w[:, 0], np.uint64(k)).astype(np.int64)
    g = np.zeros(n, dtype=np.int64)
    if k > 1 and n > 1:
        g[1:] = gaps[tracegen.mulhi64(w[1:, 1], np.uint64(k - 1)).astype(np.int64)]
    out = np.zeros(n, dtype=JOBIN_DTYPE)
    out["arrive_tick"] = np.cumsum(g) * gap_num // gap_den
    src = pop[rows]
    for f in ("gpus", "gpu_per_task", "mem_bytes", "duration"):
        out[f] = src[f]
    return out, rows


def block_starts(seed, stream, n, L):
    from gpuschedule_b200 import tracegen
    ctr = np.zeros((n, 4), dtype=np.uint64)
    ctr[:, 0] = np.arange(1, n + 1, dtype=np.uint64)
    w = tracegen.philox4x64(seed, stream, ctr)
    st = tracegen.mulhi64(w[:, 2], np.uint64(L)) == 0
    st[:1] = True
    return st


# ---------------------------------------------------------------- the mirror against the definition and hand-worked cases
@pytest.mark.parametrize("k,n,num,den,L", [(1, 300, 1, 1, 16), (2, 600, 1, 1, 3), (2, 40, 3, 2, LMAX), (7, 300, 7, 3, 16),
                                           (37, 700, 1, 1, 1000), (37, 300, 1, 1, 1), (5, 0, 1, 1, 4), (5, 1, 1, 1, 4),
                                           (50, 400, 0, 1, 8)])
def test_mirror_matches_definition(k, n, num, den, L):
    from gpuschedule_b200 import tracegen
    pop = make_population(k, seed=k + 1)
    for seed, stream in ((99, 4), (0, U64), (U64, 0)):
        recs, rows = tracegen.bootstrap_packed(pop, seed, stream, n, num, den, block_len=L)
        arr, want_rows = definition(pop, seed, stream, n, num, den, L)
        assert rows.tolist() == want_rows
        assert recs["arrive_tick"].tolist() == arr
        for f in ("gpus", "gpu_per_task", "mem_bytes", "duration"):
            assert recs[f].tolist() == pop[f][want_rows].tolist()
        assert (recs["ps_count"] == 0).all()


def test_population_of_one():
    """K = 1: every job copies the only row at tick 0, whatever L"""
    from gpuschedule_b200 import tracegen
    pop = make_population(1, seed=1)
    for L in (1, 2, 16, LMAX):
        recs, rows = tracegen.bootstrap_packed(pop, 3, 4, 1000, 1, 1, block_len=L)
        assert (rows == 0).all() and (recs["arrive_tick"] == 0).all()
        assert (recs["gpus"] == pop["gpus"][0]).all()


def test_two_rows_one_block_wraps():
    """K = 2, one block (L = 2^32 - 1): rows alternate from s_0, every gap is D[0] (continuing from row 0 to row 1,
    and the iid gap on each wrap, since D has one element), so arrivals are j * D[0] scaled"""
    from gpuschedule_b200 import tracegen
    pop = make_population(2, seed=2)
    pop["arrive_tick"] = [0, 5]
    for seed in range(6):
        assert not block_starts(seed, 1, 200, LMAX)[1:].any()
        recs, rows = tracegen.bootstrap_packed(pop, seed, 1, 200, 3, 2, block_len=LMAX)
        s0 = (words(seed, 1, 0)[0] * 2) >> 64
        assert rows.tolist() == [(s0 + j) % 2 for j in range(200)]
        assert recs["arrive_tick"].tolist() == [5 * j * 3 // 2 for j in range(200)]


def test_block_crosses_the_end_of_the_population():
    """K = 7, one block: rows run s_0, s_0 + 1, ... round the population; a wrapped row takes an iid gap, every other
    row the gap that preceded it"""
    from gpuschedule_b200 import tracegen
    pop = make_population(7, seed=4)
    pop["arrive_tick"] = [0, 1, 3, 7, 15, 31, 63]                 # D = 1, 2, 4, 8, 16, 32: a gap names its index
    D = np.diff(pop["arrive_tick"].astype(np.int64))
    seed, stream, n = 12, 5, 30
    assert not block_starts(seed, stream, n, LMAX)[1:].any()
    recs, rows = tracegen.bootstrap_packed(pop, seed, stream, n, 1, 1, block_len=LMAX)
    s0 = (words(seed, stream, 0)[0] * 7) >> 64
    assert rows.tolist() == [(s0 + j) % 7 for j in range(n)]
    g = np.diff(recs["arrive_tick"].astype(np.int64))
    for j in range(1, n):
        if rows[j] == 0:
            assert g[j - 1] == D[(words(seed, stream, j)[1] * 6) >> 64]
        else:
            assert g[j - 1] == D[rows[j] - 1]
    assert (rows == 0).sum() >= 4                                    # the block wrapped several times


def test_zero_jobs_one_job_zero_scale_zero_gaps():
    from gpuschedule_b200 import tracegen
    pop = make_population(50, seed=5)
    recs, rows = tracegen.bootstrap_packed(pop, 1, 2, 0, block_len=8)
    assert len(recs) == 0 and len(rows) == 0
    recs, rows = tracegen.bootstrap_packed(pop, 1, 2, 1, block_len=8)
    assert rows.tolist() == [(words(1, 2, 0)[0] * 50) >> 64] and recs["arrive_tick"].tolist() == [0]
    recs, _ = tracegen.bootstrap_packed(pop, 1, 2, 500, 0, 1, block_len=8)
    assert (recs["arrive_tick"] == 0).all()
    flat = make_population(50, seed=5, zero_gaps=True)
    recs, rows = tracegen.bootstrap_packed(flat, 1, 2, 500, 1, 1, block_len=8)
    assert (recs["arrive_tick"] == 0).all()
    assert rows.tolist() == tracegen.bootstrap_packed(pop, 1, 2, 500, 1, 1, block_len=8)[1].tolist()


def test_block_len_argument_checks():
    from gpuschedule_b200 import tracegen
    pop = make_population(10, seed=6)
    for bad in (0, -1, 2 ** 32, 1.5, 2.0, True, "4", None):
        with pytest.raises(ValueError):
            tracegen.bootstrap_packed(pop, 1, 2, 10, block_len=bad)
    for good in (1, np.int64(7), np.uint32(LMAX), LMAX):
        tracegen.bootstrap_packed(pop, 1, 2, 10, block_len=good)


# ---------------------------------------------------------------- L = 1 is today's iid bootstrap
def test_block_len_one_is_the_iid_bootstrap(iid_emu):
    from gpuschedule_b200 import tracegen
    from gpuschedule_b200.capi import JOBIN_DTYPE
    rng = np.random.default_rng(17)
    checked = 0
    for k in (1, 2, 3, 64, 1000, 5000):
        pop = make_population(k, seed=k)
        for n in (0, 1, 255, 256, 257, 3000):
            for num, den in ((1, 1), (0, 1), (7, 3), (1, 2)):
                seed, stream = (int(x) for x in rng.integers(0, 1 << 64, size=2, dtype=np.uint64))
                got, rows = tracegen.bootstrap_packed(pop, seed, stream, n, num, den, block_len=1)
                want, want_rows = iid_reference(pop, seed, stream, n, num, den)
                assert got.tobytes() == want.tobytes() and np.array_equal(rows, want_rows), (k, n, num, den)
                assert got.tobytes() == tracegen.bootstrap_packed(pop, seed, stream, n, num, den)[0].tobytes()
                out = np.zeros(max(n, 1), dtype=JOBIN_DTYPE)
                spans, last = C.c_longlong(0), C.c_longlong(0)
                assert iid_emu.emu_boot_trace(pop.ctypes.data, k, seed, stream, n, num, den, 16, out.ctypes.data,
                                              C.byref(spans), C.byref(last)) == 0
                assert out[:n].tobytes() == got.tobytes()
                checked += 1
    assert checked == 6 * 6 * 4


def test_bootstrap_table_block_len_one_is_unchanged():
    from gpuschedule_b200 import ingest, tracegen
    base = ingest.JobTraceReader(os.path.join(GOLDEN, "kat0", "trace.csv")).prepare_jobs().table(0.5)
    for n, num, den in ((0, 1, 1), (1, 1, 1), (257, 1, 2), (1000, 7, 3)):
        a = tracegen.bootstrap_table(base, 5, n, n, num, den)
        b = tracegen.bootstrap_table(base, 5, n, n, num, den, block_len=1)
        want, rows = iid_reference(base.packed(), 5, n, n, num, den)
        assert a.packed().tobytes() == b.packed().tobytes() == want.tobytes()
        assert a.label == b.label and a.num_gpu_text == b.num_gpu_text == [base.num_gpu_text[r] for r in rows.tolist()]
        assert np.array_equal(a.util_avg, b.util_avg) and np.array_equal(a.util_max, b.util_max)


def test_bootstrap_table_blocked_packs_to_the_mirror():
    from gpuschedule_b200 import ingest, tracegen
    base = ingest.JobTraceReader(os.path.join(GOLDEN, "kat0", "trace.csv")).prepare_jobs().table(0.5)
    for n, L in ((0, 4), (1, 4), (257, 16), (1000, 3)):
        t = tracegen.bootstrap_table(base, 5, n, n, 1, 2, block_len=L)
        want, rows = tracegen.bootstrap_packed(base.packed(), 5, n, n, 1, 2, block_len=L)
        assert t.n == n and t.packed().tobytes() == want.tobytes()
        assert t.num_gpu_text == [base.num_gpu_text[r] for r in rows.tolist()]
        assert np.array_equal(t.util_avg, base.util_avg[rows]) and np.array_equal(t.submit, t.arrive_tick)


# ---------------------------------------------------------------- host build of the blocked kernel path vs the mirror
KS = (1, 2, 7, 300, 5000)
LS = (1, 2, 3, 16, 1000, LMAX)
SCALES = ((1, 1), (0, 1), (7, 3), (1, 2))


@pytest.mark.parametrize("k", KS)
def test_host_build_traces_match_mirror(emu, k):
    from gpuschedule_b200 import tracegen
    from gpuschedule_b200.capi import JOBIN_DTYPE
    pop = make_population(k, seed=k)
    checked = 0
    for L in LS:
        for n in (0, 1, 255, 256, 257, 1000, 3 * k + 5):
            num, den = SCALES[(n + L) % len(SCALES)]
            seed, stream = (k * 7919 + n) & U64, (U64 - n) ^ L
            out = np.zeros(max(n, 1), dtype=JOBIN_DTYPE)
            rows = np.zeros(max(n, 1), dtype=np.int64)
            spans, last = C.c_longlong(0), C.c_longlong(0)
            rc = emu.emu_boot_block_trace(pop.ctypes.data, k, seed, stream, n, num, den, L, 16, out.ctypes.data, rows.ctypes.data,
                                          C.byref(spans), C.byref(last))
            assert rc == 0
            want, want_rows = tracegen.bootstrap_packed(pop, seed, stream, n, num, den, block_len=L)
            assert out[:n].tobytes() == want.tobytes(), (k, L, n, num, den)
            assert rows[:n].tolist() == want_rows.tolist()
            assert spans.value == int(np.minimum(want["gpus"] // want["gpu_per_task"], 16).sum())
            assert last.value == (int(want["arrive_tick"][-1]) if n else 0)
            checked += 1
    assert checked == len(LS) * 7


def test_host_build_refuses_like_the_mirror(emu):
    from gpuschedule_b200 import tracegen
    from gpuschedule_b200.capi import JOBIN_DTYPE
    pop = make_population(100, seed=9)
    pop["arrive_tick"][50:] += 10 ** 6
    out, rows = np.zeros(2200, dtype=JOBIN_DTYPE), np.zeros(2200, dtype=np.int64)
    spans, last = C.c_longlong(0), C.c_longlong(0)
    assert emu.emu_boot_block_trace(pop.ctypes.data, 100, 1, 2, 2200, 1, 1, 16, 16, out.ctypes.data, rows.ctypes.data,
                                    C.byref(spans), C.byref(last)) == -1
    with pytest.raises(ValueError):
        tracegen.bootstrap_packed(pop, 1, 2, 2200, 1, 1, block_len=16)


# ---------------------------------------------------------------- structural properties
@pytest.mark.parametrize("k,L", [(300, 16), (5000, 1000), (7, 3), (2, 2)])
def test_blocks_continue_rows_and_gaps(k, L):
    from gpuschedule_b200 import tracegen
    pop = make_population(k, seed=k + 11)
    D = np.diff(pop["arrive_tick"].astype(np.int64))
    n = 20000
    recs, rows = tracegen.bootstrap_packed(pop, 8, 9, n, 1, 1, block_len=L)
    st = block_starts(8, 9, n, L)
    g = np.diff(recs["arrive_tick"].astype(np.int64))
    cont = np.flatnonzero(~st)
    assert len(cont) > n // 2 - n // L
    assert np.array_equal(rows[cont], (rows[cont - 1] + 1) % k)
    keep = cont[rows[cont] != 0]                                      # not wrapped: the row's own preceding gap
    assert np.array_equal(g[keep - 1], D[rows[keep] - 1])


def test_largest_block_length_has_one_block():
    from gpuschedule_b200 import tracegen
    pop = make_population(5000, seed=12)
    n = 10 ** 5
    assert not block_starts(1, 2, n, LMAX)[1:].any()
    recs, rows = tracegen.bootstrap_packed(pop, 1, 2, n, 1, 1, block_len=LMAX)
    assert np.array_equal(rows, (rows[0] + np.arange(n)) % 5000)


def test_block_start_rate():
    """over 10^6 seeded jobs at L = 16 the share of block starts is within 5 binomial standard deviations (0.39 % of
    p here) of p = ceil(2^64 / 16) / 2^64"""
    p = -(-(1 << 64) // 16) / 2.0 ** 64
    n = 10 ** 6
    count = int(block_starts(2024, 7, n + 1, 16)[1:].sum())
    sd = (n * p * (1 - p)) ** 0.5
    assert abs(count - n * p) <= 5 * sd, (count, n * p, sd)


def test_common_random_numbers_across_loads_and_block_lengths():
    from gpuschedule_b200 import tracegen
    pop = make_population(500, seed=8)
    a, ra = tracegen.bootstrap_packed(pop, 1, 2, 1000, 1, 1, block_len=16)
    b, rb = tracegen.bootstrap_packed(pop, 1, 2, 1000, 1, 2, block_len=16)
    assert np.array_equal(ra, rb) and np.array_equal(a["arrive_tick"] // 2, b["arrive_tick"])
    s16, s256 = block_starts(1, 2, 1000, 16), block_starts(1, 2, 1000, 256)
    assert not (s256 & ~s16).any()                  # floor(w2 L / 2^64) == 0 for L = 256 implies it for L = 16
    _, r256 = tracegen.bootstrap_packed(pop, 1, 2, 1000, 1, 1, block_len=256)
    both = np.flatnonzero(s256)
    assert np.array_equal(ra[both], r256[both])     # a job that starts a block under both starts at the same row


# ---------------------------------------------------------------- the sweep: argument errors before any engine, output columns
def test_block_len_argument_errors_before_any_engine(monkeypatch, tmp_path):
    from gpuschedule_b200 import capi, sweep

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(capi, "Engine", no_engine)
    monkeypatch.setattr(capi, "HorusEngine", no_engine)
    monkeypatch.setattr(sweep, "_plain_setup", no_engine)
    trace = os.path.join(GOLDEN, "kat0", "trace.csv")
    fifo = sweep.make_flags(trace_file=trace)
    for bad in (0, -1, 2 ** 32, 1.5, True):
        with pytest.raises(ValueError):
            sweep.summarize_bootstrap([fifo], 2, block_len=bad)
    out = str(tmp_path / "s.csv")
    for argv in (["--trace", trace, "--summary", out, "--block-len", "4"],
                 ["--trace", trace, "--block-len", "4"],
                 ["--trace", trace, "--bootstrap", "4", "--summary", out, "--block-len", "0"],
                 ["--trace", trace, "--bootstrap", "4", "--summary", out, "--block-len", "-1"],
                 ["--trace", trace, "--bootstrap", "4", "--summary", out, "--block-len", str(2 ** 32)],
                 ["--trace", trace, "--bootstrap", "4", "--summary", out, "--block-len", "1.5"]):
        with pytest.raises(SystemExit) as e:
            sweep.main(argv)
        assert e.value.code == 2, argv
    assert not os.path.exists(out)


def fake_outputs(nconf, nloads, R, B, C_, E, seed=0):
    from gpuschedule_b200 import capi
    rng = np.random.default_rng(seed)
    recs = np.zeros((nconf, nloads, R), dtype=capi.SUMMARY_DTYPE)
    recs["rows"] = rng.integers(100, 1000, size=recs.shape)
    recs["makespan"] = recs["rows"]
    recs["busy_gpus_sum"] = rng.integers(0, 1 << 30, size=recs.shape)
    recs["pending_rows"] = rng.integers(1, 50, size=recs.shape)
    recs["avg_pending_sum"] = rng.uniform(0, 1e5, size=recs.shape)
    recs["finished"] = rng.integers(1, 100, size=recs.shape)
    for f in ("wait_sum", "turnaround_sum", "jct_sum"):
        recs[f] = rng.integers(0, 1 << 20, size=recs.shape)
    bins = np.zeros((nconf, nloads, R, B), dtype=capi.TBIN_DTYPE)
    bins["rows"] = rng.integers(0, 20, size=bins.shape)
    bins["busy_gpus_sum"] = bins["rows"] * rng.integers(0, 100, size=bins.shape)
    bins["pending_rows"] = np.minimum(bins["rows"], 3)
    cls = np.zeros((nconf, nloads, R, C_), dtype=capi.JCLASS_DTYPE)
    cls["jobs"] = rng.integers(0, 30, size=cls.shape)
    for m in ("wait", "turnaround", "jct"):                           # every job of a class has the value v
        v = rng.integers(0, 1000, size=cls.shape)
        cls[m + "_sum"] = cls["jobs"] * v
        cls[m + "_sq_lo"] = cls["jobs"] * v * v
        cls[m + "_q"] = v[..., None]
    hist = np.zeros((nconf, nloads, R, C_, 3, E + 1), dtype=np.uint32)
    hist[..., -1] = cls["jobs"][..., None]
    return recs, bins, cls, hist


def read_rows(path):
    with open(path, newline="") as f:
        return list(csv.reader(f))


def test_writers_add_the_block_len_column_after_load(tmp_path):
    from gpuschedule_b200 import sweep
    trace = os.path.join(GOLDEN, "kat0", "trace.csv")
    sets = [sweep.make_flags(trace_file=trace, schedule=s) for s in ("fifo", "sjf")]
    loads = [1.0, 1.25]
    recs, bins, cls, hist = fake_outputs(2, 2, 3, 4, 2, 3)
    bounds, edges = (4,), (10, 100, 1000)
    writers = {
        "runs": lambda p, **k: sweep.write_bootstrap_csv(p, sets, loads, recs, **k),
        "ci": lambda p, **k: sweep.write_bootstrap_ci_csv(p, sets, loads, recs, **k),
        "timeline": lambda p, **k: sweep.write_timeline_ci_csv(p, sets, loads, bins, 500, **k),
        "jobdist": lambda p, **k: sweep.write_jobdist_ci_csv(p, sets, loads, cls, hist, bounds, edges, **k),
        "cdf": lambda p, **k: sweep.write_jobdist_cdf_ci_csv(p, sets, loads, cls, hist, bounds, edges, **k),
    }
    heads = {"runs": ["replica", "load", "trace"], "ci": sweep.SUMMARY_KEYS + ["load", "replicas"],
             "timeline": sweep.SUMMARY_KEYS + ["load", "bin"], "jobdist": sweep.SUMMARY_KEYS + ["load", "class"],
             "cdf": sweep.SUMMARY_KEYS + ["load", "class"]}
    for name, write in writers.items():
        plain, default, blocked = (str(tmp_path / f"{name}_{t}.csv") for t in ("plain", "default", "blocked"))
        write(plain)
        write(default, block_len=None)
        write(blocked, block_len=32)
        with open(plain, "rb") as a, open(default, "rb") as b:
            assert a.read() == b.read(), name
        p, q = read_rows(plain), read_rows(blocked)
        assert p[0][:len(heads[name])] == heads[name], name       # the columns as they were
        at = p[0].index("load") + 1
        assert q[0] == p[0][:at] + ["block_len"] + p[0][at:], name
        assert len(p) == len(q) > 1
        for x, y in zip(p[1:], q[1:]):
            assert y == x[:at] + ["32"] + x[at:], name

"""Mixed bootstrap replicas (gs_boot_mixes / gs_boot_traces_mixed, gpuschedule_b200/csrc/gs_boot.cuh) on a box without
a GPU.

tracegen.alias_table is checked against the construction written out with Python integers and against the library's
host builder; tracegen.bootstrap_packed(..., weights=w) against the definition with Python integers; equal weights
must give the unweighted replicas byte for byte; the mixed paths of gs_boot.cuh, compiled with g++ in the kernel's
chunked structure (tests/emu/boot_mix_emu.cpp), must make byte-identical traces; and the sweep's --mix argument checks
and output columns are checked on the host."""
import csv
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, REPO

U64 = (1 << 64) - 1
WMAX = 2 ** 32 - 1
LMAX = 2 ** 32 - 1


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("boot_mix_emu") / "libboot_mix_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "boot_mix_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.emu_boot_alias_build.restype = C.c_ulonglong
    lib.emu_boot_alias_build.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]
    lib.emu_boot_mix_trace.restype = C.c_int
    lib.emu_boot_mix_trace.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_ulonglong, C.c_ulonglong, C.c_longlong, C.c_int, C.c_int,
                                       C.c_uint, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_longlong),
                                       C.POINTER(C.c_longlong)]
    return lib


def make_population(k, seed):
    """k records under the load rules: arrivals non-decreasing from 0, gaps of distinct sizes so a wrong gap shows"""
    from gpuschedule_b200.capi import JOBIN_DTYPE
    rng = np.random.default_rng(seed)
    p = np.zeros(k, dtype=JOBIN_DTYPE)
    gaps = rng.choice([0, 0, 1, 2, 7, 30, 411], size=k)
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


def alias_reference(w):
    """the alias construction of include/gsched.h with plain Python lists and ints"""
    K, T = len(w), sum(w)
    q = [x * K for x in w]
    U, A = [None] * K, [None] * K
    S = [i for i in range(K) if q[i] < T]
    G = [i for i in range(K) if q[i] >= T]
    while S and G:
        s, g = S.pop(0), G[0]
        U[s], A[s] = q[s], g
        q[g] -= T - q[s]
        if q[g] < T:
            S.append(G.pop(0))
    assert not S
    for i in G:
        U[i], A[i] = T, i
    return U, A


def reconstruct(U, A, T):
    """U_m + sum over {i != m : A_i = m} of (T - U_i) for every row m"""
    K = len(U)
    out = [U[m] for m in range(K)]
    for i in range(K):
        if A[i] != i:
            out[A[i]] += T - U[i]
    return out


def definition(pop, seed, stream, n, num, den, L, w):
    """the mixed (block) bootstrap written out with Python integers: (arrivals, rows)"""
    K = len(pop)
    U, A = alias_reference(w)
    T = sum(w)
    D = [int(pop["arrive_tick"][i + 1]) - int(pop["arrive_tick"][i]) for i in range(K - 1)]
    S, b, arrivals, rows = 0, 0, [], []
    for j in range(n):
        x = words(seed, stream, j)
        start = j == 0 or (x[2] * L) >> 64 == 0
        if start:
            b = j
            c = (x[0] * K) >> 64
            s = c if (x[3] * T) >> 64 < U[c] else A[c]
        r = (s + (j - b)) % K
        if j > 0 and K > 1:
            S += D[(x[1] * (K - 1)) >> 64] if (start or r == 0) else D[r - 1]
        arrivals.append(S * num // den)
        rows.append(r)
    return arrivals, rows


WEIGHT_CASES = {
    "one row": [7],
    "one row zero-free max": [WMAX],
    "zeros and one": [0, 0, 0, 1, 0],
    "one non-zero of many": [0] * 40 + [3] + [0] * 59,
    "equal": [5] * 13,
    "all max": [WMAX] * 9,
    "max and ones": [WMAX, 1, 1, WMAX, 0, 1],
    "ascending": list(range(1, 30)),
    "two classes": [1] * 20 + [4] * 5 + [0] * 3,
}


# ---------------------------------------------------------------- the alias table
@pytest.mark.parametrize("name", sorted(WEIGHT_CASES))
def test_alias_table_matches_the_construction(emu, name):
    from gpuschedule_b200 import tracegen
    w = WEIGHT_CASES[name]
    U, A = tracegen.alias_table(w)
    want_U, want_A = alias_reference(w)
    assert U.tolist() == want_U and A.tolist() == want_A
    assert reconstruct(want_U, want_A, sum(w)) == [x * len(w) for x in w]
    K = len(w)
    cU, cA = np.zeros(K, dtype=np.uint64), np.zeros(K, dtype=np.int64)
    arr = np.asarray(w, dtype=np.uint32)
    assert emu.emu_boot_alias_build(arr.ctypes.data, K, cU.ctypes.data, cA.ctypes.data) == sum(w)
    assert cU.tolist() == want_U and cA.tolist() == want_A


def test_alias_table_random_weights(emu):
    from gpuschedule_b200 import tracegen
    rng = np.random.default_rng(3)
    for trial in range(60):
        K = int(rng.integers(1, 400))
        hi = int(rng.choice([2, 10, 1000, WMAX]))
        w = rng.integers(0, hi, size=K, endpoint=True).astype(np.uint64)
        w[rng.random(K) < rng.random()] = 0
        if not w.any():
            w[int(rng.integers(K))] = 1
        w = [int(x) for x in w]
        U, A = tracegen.alias_table(w)
        want_U, want_A = alias_reference(w)
        assert U.tolist() == want_U and A.tolist() == want_A
        T = sum(w)
        assert reconstruct(want_U, want_A, T) == [x * K for x in w]
        assert all(0 <= u <= T for u in want_U) and all(0 <= a < K for a in want_A)
        assert all(A_i == i for i, (U_i, A_i) in enumerate(zip(want_U, want_A)) if U_i == T)
        cU, cA = np.zeros(K, dtype=np.uint64), np.zeros(K, dtype=np.int64)
        arr = np.asarray(w, dtype=np.uint32)
        assert emu.emu_boot_alias_build(arr.ctypes.data, K, cU.ctypes.data, cA.ctypes.data) == T
        assert cU.tolist() == want_U and cA.tolist() == want_A


def test_alias_table_and_weight_argument_checks(emu):
    from gpuschedule_b200 import tracegen
    for bad in ([], [0], [0, 0, 0], [-1, 2], [2 ** 32], [1.5, 2], "12", [[1, 2]]):
        with pytest.raises(ValueError):
            tracegen.alias_table(bad)
    pop = make_population(10, seed=1)
    for bad in ([1] * 9, [1] * 11, [0] * 10, [2 ** 32] + [1] * 9):
        with pytest.raises(ValueError):
            tracegen.bootstrap_packed(pop, 1, 2, 10, weights=bad)
    z = np.zeros(4, dtype=np.uint32)
    assert emu.emu_boot_alias_build(z.ctypes.data, 4, np.zeros(4, np.uint64).ctypes.data, np.zeros(4, np.int64).ctypes.data) == 0


def test_class_weights():
    from gpuschedule_b200 import tracegen
    gpus = np.array([1, 4, 5, 16, 17, 64, 65, 512])
    w = tracegen.class_weights(gpus, (5, 17, 65), (1, 2, 3, 4))
    assert w.dtype == np.uint32 and w.tolist() == [1, 1, 2, 2, 3, 3, 4, 4]
    assert tracegen.class_weights(gpus, (), (WMAX,)).tolist() == [WMAX] * 8
    for bounds, mults in (((5, 5), (1, 1, 1)), ((5,), (1,)), ((5,), (1, 2, 3)), ((5,), (1, -1)), ((5,), (1, 2 ** 32))):
        with pytest.raises(ValueError):
            tracegen.class_weights(gpus, bounds, mults)


# ---------------------------------------------------------------- the mirror against the definition
@pytest.mark.parametrize("k,n,num,den,L", [(1, 300, 1, 1, 1), (2, 600, 1, 1, 1), (7, 300, 7, 3, 1), (37, 700, 1, 1, 16),
                                           (37, 300, 1, 1, 1), (5, 0, 1, 1, 4), (5, 1, 1, 1, 1), (50, 400, 0, 1, 8),
                                           (60, 500, 1, 2, LMAX)])
def test_mirror_matches_definition(k, n, num, den, L):
    from gpuschedule_b200 import tracegen
    pop = make_population(k, seed=k + 1)
    rng = np.random.default_rng(k * 31 + n)
    mixes = [[1] * k, [int(x) for x in rng.integers(0, 5, size=k)], [WMAX] + [1] * (k - 1), [0] * (k - 1) + [3]]
    for w in mixes:
        if not any(w):
            w[0] = 1
        for seed, stream in ((99, 4), (0, U64), (U64, 0)):
            recs, rows = tracegen.bootstrap_packed(pop, seed, stream, n, num, den, block_len=L, weights=w)
            arr, want_rows = definition(pop, seed, stream, n, num, den, L, w)
            assert rows.tolist() == want_rows
            assert recs["arrive_tick"].tolist() == arr
            for f in ("gpus", "gpu_per_task", "mem_bytes", "duration"):
                assert recs[f].tolist() == pop[f][want_rows].tolist()
            assert (recs["ps_count"] == 0).all()


@pytest.mark.parametrize("L", [1, 16])
def test_equal_weights_are_the_unweighted_bootstrap(L):
    from gpuschedule_b200 import tracegen
    for k in (1, 2, 64, 1000):
        pop = make_population(k, seed=k)
        for value in (1, 2, 7, WMAX):
            for n, num, den in ((0, 1, 1), (1, 1, 1), (257, 7, 3), (3000, 1, 2)):
                a = tracegen.bootstrap_packed(pop, 5, n + k, n, num, den, block_len=L)
                b = tracegen.bootstrap_packed(pop, 5, n + k, n, num, den, block_len=L, weights=[value] * k)
                assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1])


def test_zero_weight_rows_are_never_drawn_at_block_len_one():
    from gpuschedule_b200 import tracegen
    pop = make_population(300, seed=4)
    w = np.zeros(300, dtype=np.uint32)
    keep = np.arange(0, 300, 7)
    w[keep] = np.arange(1, len(keep) + 1)
    _, rows = tracegen.bootstrap_packed(pop, 1, 2, 50000, weights=w)
    assert np.isin(rows, keep).all()
    counts = np.bincount(rows, minlength=300)[keep]
    p = w[keep] / w.sum()
    sd = np.sqrt(50000 * p * (1 - p))
    assert (np.abs(counts - 50000 * p) <= 5 * sd + 1).all()     # row m is drawn with probability w_m / T
    w1 = np.zeros(300, dtype=np.uint32)
    w1[123] = 9
    _, rows = tracegen.bootstrap_packed(pop, 1, 2, 2000, weights=w1)
    assert (rows == 123).all()


def test_blocked_replicas_pick_only_block_starts_from_the_mix():
    """L > 1: block starts are weighted picks, every other job continues its block through the base trace in order (so
    rows of weight 0 appear inside blocks), and the blocks and gaps are those of the unweighted replica"""
    from gpuschedule_b200 import tracegen
    k, n, L = 400, 20000, 16
    pop = make_population(k, seed=8)
    w = np.zeros(k, dtype=np.uint32)
    w[::10] = 1
    recs, rows = tracegen.bootstrap_packed(pop, 3, 4, n, block_len=L, weights=w)
    ctr = np.zeros((n, 4), dtype=np.uint64)
    ctr[:, 0] = np.arange(1, n + 1, dtype=np.uint64)
    x = tracegen.philox4x64(3, 4, ctr)
    start = tracegen.mulhi64(x[:, 2], np.uint64(L)) == 0
    start[0] = True
    assert (w[rows[start]] > 0).all()
    cont = np.flatnonzero(~start)
    assert np.array_equal(rows[cont], (rows[cont - 1] + 1) % k)
    assert (w[rows] == 0).any()
    _, plain = tracegen.bootstrap_packed(pop, 3, 4, n, block_len=L)
    assert np.array_equal(start, np.r_[True, (plain[1:] != (plain[:-1] + 1) % k) | start[1:]])


def test_bootstrap_table_with_weights():
    from gpuschedule_b200 import ingest, tracegen
    base = ingest.JobTraceReader(os.path.join(GOLDEN, "kat0", "trace.csv")).prepare_jobs().table(0.5)
    w = tracegen.class_weights(base.gpus, (2, 8), (0, 1, 5))
    for n, L in ((0, 1), (1, 1), (257, 1), (1000, 3)):
        t = tracegen.bootstrap_table(base, 5, n, n, 1, 2, block_len=L, weights=w)
        want, rows = tracegen.bootstrap_packed(base.packed(), 5, n, n, 1, 2, block_len=L, weights=w)
        assert t.n == n and t.packed().tobytes() == want.tobytes()
        assert t.num_gpu_text == [base.num_gpu_text[r] for r in rows.tolist()]
    a = tracegen.bootstrap_table(base, 5, 9, 300)
    b = tracegen.bootstrap_table(base, 5, 9, 300, weights=[3] * base.n)
    assert a.packed().tobytes() == b.packed().tobytes()


# ---------------------------------------------------------------- host build of the mixed kernel paths vs the mirror
KS = (1, 2, 7, 300, 5000)
LS = (1, 2, 16, 1000, LMAX)
SCALES = ((1, 1), (0, 1), (7, 3), (1, 2))


def mixes_for(k, rng):
    ws = [None, np.full(k, 3, dtype=np.uint32), rng.integers(0, 6, size=k).astype(np.uint32)]
    skew = np.zeros(k, dtype=np.uint32)
    skew[::3] = WMAX
    ws.append(skew)
    for w in ws[1:]:
        if not w.any():
            w[0] = 1
    return ws


@pytest.mark.parametrize("k", KS)
def test_host_build_traces_match_mirror(emu, k):
    from gpuschedule_b200 import tracegen
    from gpuschedule_b200.capi import JOBIN_DTYPE
    pop = make_population(k, seed=k)
    rng = np.random.default_rng(k)
    checked = 0
    for wi, w in enumerate(mixes_for(k, rng)):
        for L in LS:
            for blocked in ((0, 1) if L == 1 else (1,)):
                for n in (0, 1, 255, 256, 257, 1000, 3 * k + 5):
                    num, den = SCALES[(n + L + wi) % len(SCALES)]
                    seed, stream = (k * 7919 + n + wi) & U64, (U64 - n) ^ L
                    out = np.zeros(max(n, 1), dtype=JOBIN_DTYPE)
                    rows = np.zeros(max(n, 1), dtype=np.int64)
                    spans, last = C.c_longlong(0), C.c_longlong(0)
                    rc = emu.emu_boot_mix_trace(pop.ctypes.data, k, None if w is None else w.ctypes.data, seed, stream, n, num, den, L,
                                                blocked, 16, out.ctypes.data, rows.ctypes.data, C.byref(spans), C.byref(last))
                    assert rc == 0
                    want, want_rows = tracegen.bootstrap_packed(pop, seed, stream, n, num, den, block_len=L, weights=w)
                    assert out[:n].tobytes() == want.tobytes(), (k, wi, L, blocked, n, num, den)
                    assert rows[:n].tolist() == want_rows.tolist()
                    assert spans.value == int(np.minimum(want["gpus"] // want["gpu_per_task"], 16).sum())
                    assert last.value == (int(want["arrive_tick"][-1]) if n else 0)
                    checked += 1
    assert checked == 4 * (len(LS) + 1) * 7


def test_host_build_refuses_like_the_mirror(emu):
    from gpuschedule_b200 import tracegen
    from gpuschedule_b200.capi import JOBIN_DTYPE
    pop = make_population(100, seed=9)
    pop["arrive_tick"][50:] += 10 ** 6
    out, rows = np.zeros(2200, dtype=JOBIN_DTYPE), np.zeros(2200, dtype=np.int64)
    spans, last = C.c_longlong(0), C.c_longlong(0)
    w = np.ones(100, dtype=np.uint32)
    assert emu.emu_boot_mix_trace(pop.ctypes.data, 100, w.ctypes.data, 1, 2, 2200, 1, 1, 1, 0, 16, out.ctypes.data, rows.ctypes.data,
                                  C.byref(spans), C.byref(last)) == -1
    with pytest.raises(ValueError):
        tracegen.bootstrap_packed(pop, 1, 2, 2200, 1, 1, weights=w)
    z = np.zeros(100, dtype=np.uint32)
    assert emu.emu_boot_mix_trace(pop.ctypes.data, 100, z.ctypes.data, 1, 2, 10, 1, 1, 1, 0, 16, out.ctypes.data, rows.ctypes.data,
                                  C.byref(spans), C.byref(last)) == -1


def test_common_random_numbers_across_mixes():
    """the gaps (w1) and the block starts (w2) do not depend on the mix"""
    from gpuschedule_b200 import tracegen
    pop = make_population(500, seed=8)
    pop["arrive_tick"] = np.arange(500) * 3                           # one gap size: arrivals are j * 3 whatever the rows
    a, _ = tracegen.bootstrap_packed(pop, 1, 2, 1000, weights=np.arange(500) % 4)
    b, _ = tracegen.bootstrap_packed(pop, 1, 2, 1000, weights=(np.arange(500) % 3 == 0).astype(np.uint32))
    assert np.array_equal(a["arrive_tick"], b["arrive_tick"])


# ---------------------------------------------------------------- the sweep: argument errors before any engine, output columns
def test_mix_argument_errors_before_any_engine(monkeypatch, tmp_path):
    from gpuschedule_b200 import capi, ingest, sweep

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(capi, "Engine", no_engine)
    monkeypatch.setattr(capi, "HorusEngine", no_engine)
    trace = os.path.join(GOLDEN, "kat0", "trace.csv")
    fifo = sweep.make_flags(trace_file=trace)
    for bad in (((5,), []), ((5,), [(1,)]), ((5,), [(1, 2, 3)]), ((5, 5), [(1, 1, 1)]), ((0,), [(1, 1)]), ((5,), [(1, -1)]),
                ((5,), [(1, 2 ** 32)]), None.__class__, 3):
        with pytest.raises(ValueError):
            sweep.summarize_bootstrap([fifo], 2, mix=bad)
    # a mix whose weights are all 0 on the trace: ValueError after the trace is read, before any engine
    gpus = ingest.JobTraceReader(trace).prepare_jobs().table(0.5).gpus
    top = int(gpus.max()) + 1
    with pytest.raises(ValueError, match="weight 0"):
        sweep.summarize_bootstrap([fifo], 2, mix=((top,), [(1, 1), (0, 1)]))

    def no_trace(*a, **k):
        raise AssertionError("a trace was read")
    monkeypatch.setattr(sweep, "_plain_setup", no_trace)
    out = str(tmp_path / "s.csv")
    base = ["--trace", trace, "--summary", out]
    for argv in (base + ["--mix", "1:1"],                                                     # no --bootstrap
                 base + ["--mix", "1:1", "--mix-classes", "4"],
                 base + ["--mix-classes", "4"],
                 base + ["--bootstrap", "4", "--mix", "1:1"],                                   # no --mix-classes
                 base + ["--bootstrap", "4", "--mix-classes", "4"],                             # no --mix
                 base + ["--bootstrap", "4", "--mix", "1:1:1", "--mix-classes", "4"],           # wrong counts
                 base + ["--bootstrap", "4", "--mix", "1", "--mix-classes", "4"],
                 base + ["--bootstrap", "4", "--mix", "1:1", "2", "--mix-classes", "4"],
                 base + ["--bootstrap", "4", "--mix", "1:-1", "--mix-classes", "4"],            # malformed
                 base + ["--bootstrap", "4", "--mix", "1:x", "--mix-classes", "4"],
                 base + ["--bootstrap", "4", "--mix", "1::1", "--mix-classes", "4", "8"],
                 base + ["--bootstrap", "4", "--mix", "1:1.5", "--mix-classes", "4"],
                 base + ["--bootstrap", "4", "--mix", "1:+1", "--mix-classes", "4"],
                 base + ["--bootstrap", "4", "--mix", "1:1:", "--mix-classes", "4", "8"],
                 base + ["--bootstrap", "4", "--mix", f"1:{2 ** 32}", "--mix-classes", "4"],   # above 2^32 - 1
                 base + ["--bootstrap", "4", "--mix", "1:1", "--mix-classes", "0"],            # bad bounds
                 base + ["--bootstrap", "4", "--mix", "1:1:1", "--mix-classes", "8", "4"],
                 base + ["--bootstrap", "4", "--mix", "1:1", "--mix-classes", "x"]):
        with pytest.raises(SystemExit) as e:
            sweep.main(argv)
        assert e.value.code == 2, argv
    assert not os.path.exists(out)


def fake_outputs(nconf, nloads, nmix, R, B, C_, E, seed=0):
    from gpuschedule_b200 import capi
    rng = np.random.default_rng(seed)
    lead = (nconf, nloads, nmix, R)
    recs = np.zeros(lead, dtype=capi.SUMMARY_DTYPE)
    recs["rows"] = rng.integers(100, 1000, size=recs.shape)
    recs["makespan"] = recs["rows"]
    recs["busy_gpus_sum"] = rng.integers(0, 1 << 30, size=recs.shape)
    recs["pending_rows"] = rng.integers(1, 50, size=recs.shape)
    recs["avg_pending_sum"] = rng.uniform(0, 1e5, size=recs.shape)
    recs["finished"] = rng.integers(1, 100, size=recs.shape)
    for f in ("wait_sum", "turnaround_sum", "jct_sum"):
        recs[f] = rng.integers(0, 1 << 20, size=recs.shape)
    bins = np.zeros(lead + (B,), dtype=capi.TBIN_DTYPE)
    bins["rows"] = rng.integers(0, 20, size=bins.shape)
    bins["busy_gpus_sum"] = bins["rows"] * rng.integers(0, 100, size=bins.shape)
    bins["pending_rows"] = np.minimum(bins["rows"], 3)
    cls = np.zeros(lead + (C_,), dtype=capi.JCLASS_DTYPE)
    cls["jobs"] = rng.integers(0, 30, size=cls.shape)
    for m in ("wait", "turnaround", "jct"):
        v = rng.integers(0, 1000, size=cls.shape)
        cls[m + "_sum"] = cls["jobs"] * v
        cls[m + "_sq_lo"] = cls["jobs"] * v * v
        cls[m + "_q"] = v[..., None]
    hist = np.zeros(lead + (C_, 3, E + 1), dtype=np.uint32)
    hist[..., -1] = cls["jobs"][..., None]
    prec = np.zeros((1,) + lead[1:] + (C_,), dtype=capi.JPAIR_DTYPE)
    prec["jobs"] = rng.integers(0, 30, size=prec.shape)
    phist = np.zeros((1,) + lead[1:] + (C_, 3, E + 1), dtype=np.uint32)
    phist[..., -1] = prec["jobs"][..., None]
    return recs, bins, cls, hist, prec, phist


def read_rows(path):
    with open(path, newline="") as f:
        return list(csv.reader(f))


@pytest.mark.parametrize("block_len", [None, 32])
def test_writers_add_the_mix_column(tmp_path, block_len):
    """with mixes every bootstrap file gets a mix column right after load (after block_len when present), and its lines
    are those of the (load, mix) pairs in that order; the mix-free files are those of one mix without the column"""
    from gpuschedule_b200 import sweep
    trace = os.path.join(GOLDEN, "kat0", "trace.csv")
    sets = [sweep.make_flags(trace_file=trace, schedule=s) for s in ("fifo", "sjf")]
    loads, specs = [1.0, 1.25], ["1:1", "0:3"]
    recs, bins, cls, hist, prec, phist = fake_outputs(2, 2, 2, 3, 4, 2, 3)
    bounds, edges = (4,), (-10, 0, 100)
    pairs = [(0, 1)]
    writers = {
        "runs": lambda p, r, b, c, h, pr, ph, **k: sweep.write_bootstrap_csv(p, sets, loads, r, **k),
        "ci": lambda p, r, b, c, h, pr, ph, **k: sweep.write_bootstrap_ci_csv(p, sets, loads, r, **k),
        "timeline": lambda p, r, b, c, h, pr, ph, **k: sweep.write_timeline_ci_csv(p, sets, loads, b, 500, **k),
        "jobdist": lambda p, r, b, c, h, pr, ph, **k: sweep.write_jobdist_ci_csv(p, sets, loads, c, h, bounds, edges, **k),
        "cdf": lambda p, r, b, c, h, pr, ph, **k: sweep.write_jobdist_cdf_ci_csv(p, sets, loads, c, h, bounds, edges, **k),
        "paired": lambda p, r, b, c, h, pr, ph, **k: sweep.write_paired_ci_csv(p, sets, pairs, loads, pr, ph, bounds, edges, **k),
        "paired_cdf": lambda p, r, b, c, h, pr, ph, **k: sweep.write_paired_cdf_csv(p, sets, pairs, pr, ph, bounds, edges, loads=loads, **k),
        "paired_summary": lambda p, r, b, c, h, pr, ph, **k: sweep.write_paired_summary_csv(p, sets, pairs, r, loads=loads, **k),
    }
    for name, write in writers.items():
        mixed = str(tmp_path / f"{name}_mixed.csv")
        write(mixed, recs, bins, cls, hist, prec, phist, block_len=block_len, mix=specs)
        q = read_rows(mixed)
        per_mix = []
        for m in range(2):                                               # one mix alone, without the column
            path = str(tmp_path / f"{name}_{m}.csv")
            pick = lambda a: a[:, :, m]
            write(path, pick(recs), pick(bins), pick(cls), pick(hist), pick(prec), pick(phist), block_len=block_len)
            per_mix.append(read_rows(path))
        default = str(tmp_path / f"{name}_default.csv")
        write(default, recs[:, :, 0], bins[:, :, 0], cls[:, :, 0], hist[:, :, 0], prec[:, :, 0], phist[:, :, 0], block_len=block_len, mix=None)
        with open(default, "rb") as a, open(str(tmp_path / f"{name}_0.csv"), "rb") as b:
            assert a.read() == b.read(), name
        head = per_mix[0][0]
        at = head.index("block_len" if block_len is not None else "load") + 1
        assert q[0] == head[:at] + ["mix"] + head[at:], name
        load_at = head.index("load")
        # the mix-free lines, tagged with their mix, in (config, load, mix) order
        want = []
        body = [p[1:] for p in per_mix]
        assert len(body[0]) == len(body[1])
        keyed = [(m, i, row) for m in range(2) for i, row in enumerate(body[m])]
        per_load = len(body[0]) // (len(sets if name in ("runs", "ci", "timeline", "jobdist", "cdf") else pairs) * len(loads))
        keyed.sort(key=lambda t: (t[1] // per_load, t[0], t[1]))
        for m, _, row in keyed:
            want.append(row[:at] + [specs[m]] + row[at:])
        assert q[1:] == want, name
        assert all(r[load_at] in ("1.0", "1.25") for r in q[1:])

"""Profiled bootstrap replicas (gs_boot_profiles / gs_boot_traces_profiled, gpuschedule_b200/csrc/gs_boot.cuh) on a box
without a GPU.

The host conversion and the arrival rule are checked against a restatement with Python ints and Fractions, both in
tracegen and in the library's own __host__ __device__ functions compiled with g++ (tests/emu/boot_profile_emu.cpp,
which also runs the kernel's chunked structure); the properties of the definition (monotone, exact segment starts,
the one-segment and periodic-identity cases, the map from the 1/1 replica) are checked on random profiles; the
arrival bound at 2^31 - 2 and 2^31 - 1; and the sweep's SPEC parsing, argument errors and output columns."""
import ctypes as C
import math
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from conftest import GOLDEN, REPO
from test_boot_mix_cpu import make_population, read_rows

U64 = (1 << 64) - 1
I31 = 2 ** 31 - 1


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("boot_profile_emu") / "libboot_profile_emu.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared", "-x", "c++",
                    "-I", os.path.join(REPO, "include"), "-I", os.path.join(REPO, "gpuschedule_b200", "csrc"),
                    "-o", out, os.path.join(REPO, "tests", "emu", "boot_profile_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.emu_boot_profile_invalid.restype = C.c_int
    lib.emu_boot_profile_invalid.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.emu_boot_profile_base.restype = C.c_longlong
    lib.emu_boot_profile_base.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.emu_boot_profile_arrive.restype = None
    lib.emu_boot_profile_arrive.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p]
    lib.emu_boot_profile_bound.restype = C.c_longlong
    lib.emu_boot_profile_bound.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_longlong]
    lib.emu_boot_profile_trace.restype = C.c_int
    lib.emu_boot_profile_trace.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_ulonglong, C.c_ulonglong,
                                           C.c_longlong, C.c_int, C.c_int, C.c_uint, C.c_int, C.c_int, C.c_void_p,
                                           C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    return lib


def seg_array(segs):
    from gpuschedule_b200.capi import BOOT_SEG_DTYPE
    a = np.zeros(len(segs), dtype=BOOT_SEG_DTYPE)
    for i, (t, num, den) in enumerate(segs):
        a[i] = (t, num, den, 0)
    return a


def ref_base(segs, P):
    """the conversion with Fractions: s_(k+1) = s_k + ceil((t_(k+1) - t_k) / (num_k / den_k))"""
    s = [0]
    ends = [t for t, _, _ in segs[1:]] + ([P] if P else [])
    for k, end in enumerate(ends):
        s.append(s[-1] + math.ceil(Fraction(end - segs[k][0]) / Fraction(segs[k][1], segs[k][2])))
    return s[:len(segs)], (s[-1] if P else 0)


def ref_arrive(S, segs, P):
    """the arrival rule with Fractions and Python ints"""
    s, B = ref_base(segs, P)
    q = 0
    if P:
        q, S = divmod(S, B)
    k = max(i for i in range(len(s)) if s[i] <= S)
    return q * P + segs[k][0] + math.floor((S - s[k]) * Fraction(segs[k][1], segs[k][2]))


SCALE_CHOICES = [(1, 1), (1, 65535), (65535, 1), (1, 2), (3, 1), (7, 3), (I31, 1), (1, I31), (I31, I31), (I31, I31 - 1), (65535, 65534)]


def random_profile(rng, periodic, m=None):
    m = int(rng.integers(1, 65)) if m is None else m
    span = int(rng.choice([m, 10 * m, 10 ** 5, 10 ** 7, I31 - 2]))
    t = sorted(set([0] + [int(x) for x in rng.integers(1, max(span, 2), size=m - 1)]))
    while len(t) < m:
        t.append(t[-1] + 1)
    segs = []
    for ti in t:
        if rng.random() < 0.5:
            num, den = SCALE_CHOICES[int(rng.integers(len(SCALE_CHOICES)))]
        else:
            num, den = int(rng.integers(1, 65536)), int(rng.integers(1, 65536))
        segs.append((ti, num, den))
    P = 0
    if periodic and t[-1] < I31 - 1:
        P = int(rng.integers(t[-1] + 1, min(I31 - 1, t[-1] + 1 + 10 ** int(rng.integers(0, 10)))))
    return segs, P


def probes(segs, P, rng, top):
    """base times around every segment start (and period boundary), plus random ones, all in [0, top]"""
    s, B = ref_base(segs, P)
    xs = {0, top}
    for q in ((0, 1, 5) if P else (0,)):
        for sk in s + ([B] if P else []):
            for d in (-2, -1, 0, 1, 2):
                x = q * B + sk + d
                if 0 <= x <= top:
                    xs.add(x)
    xs |= {int(x) for x in rng.integers(0, top + 1, size=40)}
    return sorted(xs)


def arrive_top(segs, P):
    """the largest base time whose arrival stays below 2^31 - 1 (the region the bound admits), by bisection"""
    lo, hi = 0, 1
    while ref_arrive(hi, segs, P) < I31:
        lo, hi = hi, hi * 2
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if ref_arrive(mid, segs, P) < I31 else (lo, mid)
    return lo


# ---------------------------------------------------------------- the conversion and the arrival rule
@pytest.mark.parametrize("periodic", [False, True])
def test_conversion_and_arrival_rule_match_the_restatement(emu, periodic):
    from gpuschedule_b200 import tracegen
    rng = np.random.default_rng(11 + periodic)
    for trial in range(120):
        segs, P = random_profile(rng, periodic, m=(1, 2, 64)[trial % 3] if trial < 9 else None)
        s, B = ref_base(segs, P)
        assert tracegen.profile_base(segs, P) == (s, B)
        a = seg_array(segs)
        assert emu.emu_boot_profile_invalid(a.ctypes.data, len(segs), P) == 0
        cs = np.zeros(len(segs), dtype=np.int64)
        assert emu.emu_boot_profile_base(a.ctypes.data, len(segs), P, cs.ctypes.data) == B
        assert cs.tolist() == s
        top = arrive_top(segs, P)
        xs = probes(segs, P, rng, top)
        want = [ref_arrive(x, segs, P) for x in xs]
        assert [tracegen.profile_arrive(x, segs, P) for x in xs] == want
        X = np.array(xs, dtype=np.int64)
        assert tracegen.profile_arrive(X, segs, P).tolist() == want
        out = np.zeros(len(xs), dtype=np.int64)
        emu.emu_boot_profile_arrive(a.ctypes.data, len(segs), P, X.ctypes.data, len(xs), out.ctypes.data)
        assert out.tolist() == want
        # (S - s_k) * num_k stays below 2^62 wherever the bound admits S
        for x in xs:
            xq = x % B if P else x
            k = max(i for i in range(len(s)) if s[i] <= xq)
            assert (xq - s[k]) * segs[k][1] < 2 ** 62


@pytest.mark.parametrize("periodic", [False, True])
def test_properties_of_the_definition(periodic):
    from gpuschedule_b200 import tracegen
    rng = np.random.default_rng(5 + periodic)
    for trial in range(80):
        segs, P = random_profile(rng, periodic, m=int(rng.integers(1, 9)))
        s, B = ref_base(segs, P)
        xs = probes(segs, P, rng, arrive_top(segs, P))
        a = [tracegen.profile_arrive(x, segs, P) for x in xs]
        assert all(y >= x for x, y in zip(a, a[1:]))                               # monotone
        for q in ((0, 1, 3) if P else (0,)):
            for k, (t, _, _) in enumerate(segs):                                   # exact segment starts, every period
                x = q * B + s[k]
                if tracegen.profile_arrive(x, segs, P) >= I31:
                    continue
                assert tracegen.profile_arrive(x, segs, P) == q * P + t
                if x > 0:
                    assert tracegen.profile_arrive(x - 1, segs, P) < q * P + t     # the first base time that reaches t_k


def test_one_segment_is_the_gap_scale_and_periodic_one_is_the_identity():
    from gpuschedule_b200 import tracegen
    S = np.array([0, 1, 2, 99, 10 ** 6, 10 ** 9, 2 ** 31 - 2], dtype=np.int64)
    for num, den in ((1, 1), (1, 2), (7, 3), (65535, 65534), (1, 65535)):
        assert tracegen.profile_arrive(S, [(0, num, den)]).tolist() == (S * num // den).tolist()
    for P in (1, 2, 1440, I31 - 2):
        assert tracegen.profile_arrive(S, [(0, 1, 1)], P).tolist() == S.tolist()


def test_profile_rules(emu):
    from gpuschedule_b200 import tracegen
    bad = [([], 0), ([(1, 1, 1)], 0), ([(0, 1, 1), (0, 1, 1)], 0), ([(0, 1, 1), (5, 1, 1), (4, 1, 1)], 0),
           ([(0, 1, 1), (I31, 1, 1)], 0), ([(0, 0, 1)], 0), ([(0, 1, 0)], 0), ([(0, -1, 1)], 0), ([(0, 1, 1)], -1),
           ([(0, 1, 1), (10, 1, 1)], 10), ([(0, 1, 1), (10, 1, 1)], 5), ([(0, 1, 1)] + [(k, 1, 1) for k in range(1, 65)], 0)]
    for segs, P in bad:
        with pytest.raises(ValueError):
            tracegen.check_profile(segs, P)
        a = seg_array(segs) if segs else seg_array([(0, 1, 1)])
        assert emu.emu_boot_profile_invalid(a.ctypes.data, len(segs), P) == 1, (segs, P)
    for segs, P in (([(0, 1, 1)], 0), ([(0, I31, I31), (I31 - 2, 1, 1)], I31 - 1 - 0 if False else 0),
                    ([(0, 1, 1), (I31 - 2, 1, 1)], 0), ([(k, 1, 1) for k in range(64)], 64)):
        tracegen.check_profile(segs, P)
        assert emu.emu_boot_profile_invalid(seg_array(segs).ctypes.data, len(segs), P) == 0


# ---------------------------------------------------------------- the bound, exactly
@pytest.mark.parametrize("periodic", [False, True])
def test_arrival_bound_at_the_limit(emu, periodic):
    """a population whose largest gap is 2: the worst-case base time is 2 (n - 1).  For each target, find a profile
    and n with arrive(2 (n - 1)) exactly 2^31 - 2 (accepted) or 2^31 - 1 (refused), and check the bound in the mirror
    and in the library's host code"""
    from gpuschedule_b200 import tracegen
    from gpuschedule_b200.capi import JOBIN_DTYPE
    pop = np.zeros(3, dtype=JOBIN_DTYPE)
    pop["arrive_tick"] = [0, 2, 4]
    pop["gpus"] = pop["gpu_per_task"] = 1
    pop["duration"] = 1.0
    P = 7000 if periodic else 0
    for target in (I31 - 1, I31):                              # 2^31 - 2 and 2^31 - 1
        for d in range(4000, 4010):                           # the 1/2 segment's length sets the parity of the base time
            segs = [(0, 1, 1), (1000, 1, 2), (1000 + d, 1, 1)]
            lo, hi = 0, 1 << 40                               # the least base time arriving at target or later
            while hi - lo > 1:
                mid = (lo + hi) // 2
                lo, hi = (lo, mid) if ref_arrive(mid, segs, P) >= target else (mid, hi)
            if ref_arrive(hi, segs, P) == target and hi % 2 == 0:
                break
        else:
            raise AssertionError("no profile reaches the target at an even base time")
        n = hi // 2 + 1
        assert n < 2 ** 31 - 64
        a = seg_array(segs)
        assert tracegen.profile_bound(n, 2, segs, P) == target
        assert emu.emu_boot_profile_bound(a.ctypes.data, 3, P, n, 2) == target
        assert tracegen.profile_bound(n - 1, 2, segs, P) < target
        if target == I31:
            with pytest.raises(ValueError, match="2\\^31 - 1"):
                tracegen.bootstrap_packed(pop, 1, 2, n, profile=(segs, P))
            out = np.zeros(1, dtype=JOBIN_DTYPE)
            spans, last = C.c_longlong(0), C.c_longlong(0)
            assert emu.emu_boot_profile_trace(pop.ctypes.data, 3, None, a.ctypes.data, 3, P, 1, 2, n, 1, 1, 1, 0, 1, out.ctypes.data,
                                              C.byref(spans), C.byref(last)) == -1
    with pytest.raises(ValueError):                           # a profiled replica keeps the gap scale 1 / 1
        tracegen.bootstrap_packed(pop, 1, 2, 10, 1, 2, profile=([(0, 1, 1)], P))


# ---------------------------------------------------------------- host build of the kernel paths vs the mirror
PROFILES = [None, ([(0, 1, 1)], 0), ([(0, 1, 2)], 0), ([(0, 1, 1), (300, 1, 3), (900, 1, 1)], 0),
            ([(0, 5, 3), (100, 3, 5), (700, 1, 1)], 1440), ([(k * 37, 1 + k % 5, 1 + k % 3) for k in range(64)], 64 * 37 + 1)]


@pytest.mark.parametrize("k", [1, 7, 300, 3000])
def test_host_build_traces_match_mirror(emu, k):
    from gpuschedule_b200 import tracegen
    from gpuschedule_b200.capi import JOBIN_DTYPE
    pop = make_population(k, seed=k)
    rng = np.random.default_rng(k)
    w = rng.integers(0, 4, size=k).astype(np.uint32)
    w[0] = 1
    checked = 0
    for pi, prof in enumerate(PROFILES):
        for weights in (None, w):
            for L, blocked in ((1, 0), (1, 1), (16, 1)):
                for n in (0, 1, 257, 1000):
                    seed, stream = (k * 7919 + n + pi) & U64, (U64 - n) ^ L
                    num, den = (1, 1) if prof is not None else ((1, 1), (7, 3))[n % 2]
                    out = np.zeros(max(n, 1), dtype=JOBIN_DTYPE)
                    spans, last = C.c_longlong(0), C.c_longlong(0)
                    a = seg_array(prof[0]) if prof is not None else None
                    rc = emu.emu_boot_profile_trace(pop.ctypes.data, k, None if weights is None else weights.ctypes.data,
                                                    None if a is None else a.ctypes.data, 0 if prof is None else len(prof[0]),
                                                    0 if prof is None else prof[1], seed, stream, n, num, den, L, blocked, 16,
                                                    out.ctypes.data, C.byref(spans), C.byref(last))
                    assert rc == 0
                    want, _ = tracegen.bootstrap_packed(pop, seed, stream, n, num, den, block_len=L, weights=weights, profile=prof)
                    assert out[:n].tobytes() == want.tobytes(), (k, pi, L, blocked, n)
                    assert spans.value == int(np.minimum(want["gpus"] // want["gpu_per_task"], 16).sum())
                    assert last.value == (int(want["arrive_tick"][-1]) if n else 0)
                    checked += 1
    assert checked == len(PROFILES) * 2 * 3 * 4


@pytest.mark.parametrize("L", [1, 16])
def test_profiled_replica_is_the_map_of_the_one_to_one_replica(L):
    """same (seed, stream): every field but the arrivals is the 1/1 replica's, and the arrivals are arrive_p of its
    arrivals; one segment {0, num, den} is the replica at gap scale num / den byte for byte, periodic {0, 1, 1} the
    1/1 replica"""
    from gpuschedule_b200 import tracegen
    pop = make_population(500, seed=3)
    w = (np.arange(500) % 3).astype(np.uint32)
    rng = np.random.default_rng(L)
    for weights in (None, w):
        base, rows = tracegen.bootstrap_packed(pop, 9, 4, 5000, block_len=L, weights=weights)
        for trial in range(6):
            segs, P = random_profile(rng, trial % 2 == 1, m=int(rng.integers(1, 12)))
            segs = [(t % 10 ** 6 if i else 0, num, den) for i, (t, num, den) in enumerate(segs)]
            segs = sorted(dict((t, (t, n_, d)) for t, n_, d in segs).values())
            P = P if not P else max(segs[-1][0] + 1, P % (2 * 10 ** 6))
            try:
                got, grows = tracegen.bootstrap_packed(pop, 9, 4, 5000, block_len=L, weights=weights, profile=(segs, P))
            except ValueError:
                continue
            assert np.array_equal(grows, rows)
            for f in ("gpus", "gpu_per_task", "ps_count", "mem_bytes", "duration"):
                assert np.array_equal(got[f], base[f])
            assert got["arrive_tick"].tolist() == [ref_arrive(int(x), segs, P) for x in base["arrive_tick"]]
        for num, den in ((1, 2), (7, 3), (3, 1)):
            a, _ = tracegen.bootstrap_packed(pop, 9, 4, 5000, num, den, block_len=L, weights=weights)
            b, _ = tracegen.bootstrap_packed(pop, 9, 4, 5000, block_len=L, weights=weights, profile=([(0, num, den)], 0))
            assert a.tobytes() == b.tobytes()
        c, _ = tracegen.bootstrap_packed(pop, 9, 4, 5000, block_len=L, weights=weights, profile=([(0, 1, 1)], 1440))
        assert c.tobytes() == base.tobytes()


# ---------------------------------------------------------------- the sweep: SPECs, argument errors, columns
def test_parse_profile_spec_and_segments():
    from gpuschedule_b200 import sweep
    assert sweep.parse_profile_spec("0:1,20000:3,22000:1") == (((0, 1.0), (20000, 3.0), (22000, 1.0)), 0)
    assert sweep.parse_profile_spec("0:0.6,480:1.4,1200:0.6@1440") == (((0, 0.6), (480, 1.4), (1200, 0.6)), 1440)
    assert sweep.parse_profile_spec("0:2") == (((0, 2.0),), 0)
    for bad in ("", "1:1", "0:1,0:2", "0:1,5:1,3:1", "0:0", "0:-1", "0:inf", "0:nan", "0:x", "0", "0:1,", "0:1@", "0:1@-5",
                "0:1,100:1@100", "0:1,100:1@50", "-1:1", "0:1@x", "0:1@1.5", f"0:1,{2 ** 31 - 1}:1", f"0:1@{2 ** 31 - 1}",
                ",".join(f"{k}:1" for k in range(65))):
        with pytest.raises(ValueError):
            sweep.parse_profile_spec(bad)
    segs, P = sweep.profile_segments(((0, 1.0), (100, 3.0)), 0, 0.5)
    assert segs == [(0, *sweep.load_gap_scale(0.5)), (100, *sweep.load_gap_scale(1.5))] and P == 0
    for factor in (1e-12, 1e12, 1e-320):
        with pytest.raises(ValueError):
            sweep.profile_segments(((0, factor),), 0, 1.0)


def test_profile_argument_errors_before_any_engine(monkeypatch, tmp_path):
    from gpuschedule_b200 import capi, sweep

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(capi, "Engine", no_engine)
    monkeypatch.setattr(capi, "HorusEngine", no_engine)
    trace = os.path.join(GOLDEN, "kat0", "trace.csv")
    fifo = sweep.make_flags(trace_file=trace)
    for bad in ([], [((), 0)], [(((1, 1.0),), 0)], [(((0, 0.0),), 0)], [(((0, 1.0), (5, 1.0)), 5)], 3, [(((0, 1e-12),), 0)]):
        with pytest.raises(ValueError):
            sweep.summarize_bootstrap([fifo], 2, profile=bad)
    with pytest.raises(ValueError, match="2\\^31 - 1"):           # after the trace is read, before any engine
        sweep.summarize_bootstrap([fifo], 2, n=2 ** 31 - 65, profile=[(((0, 1.0),), 0)])

    def no_trace(*a, **k):
        raise AssertionError("a trace was read")
    monkeypatch.setattr(sweep, "_plain_setup", no_trace)
    out = str(tmp_path / "s.csv")
    base = ["--trace", trace, "--summary", out]
    for argv in (base + ["--load-profile", "0:1"],                                   # no --bootstrap
                 base + ["--bootstrap", "4", "--load-profile"],
                 base + ["--bootstrap", "4", "--load-profile", "1:1"],
                 base + ["--bootstrap", "4", "--load-profile", "0:1,0:2"],
                 base + ["--bootstrap", "4", "--load-profile", "0:0"],
                 base + ["--bootstrap", "4", "--load-profile", "0:1", "0:x"],
                 base + ["--bootstrap", "4", "--load-profile", "0:1,10:2@10"],
                 base + ["--bootstrap", "4", "--load-profile", "0:1@-1"],
                 base + ["--bootstrap", "4", "--load-profile", "0:1e-12"],
                 base + ["--bootstrap", "4", "--load", "0.4", "--load-profile", "0:1,10:1e-9"]):   # L x F too small
        with pytest.raises(SystemExit) as e:
            sweep.main(argv)
        assert e.value.code == 2, argv
    assert not os.path.exists(out)


@pytest.mark.parametrize("mix", [None, ["1:1", "0:3"]])
def test_writers_add_the_profile_column(tmp_path, mix):
    """with profiles every bootstrap file gets a profile column after mix (after load / block_len without mixes), and
    its lines are in (load, mix, profile) order; without profiles every file is unchanged"""
    from test_boot_mix_cpu import fake_outputs
    from gpuschedule_b200 import sweep
    trace = os.path.join(GOLDEN, "kat0", "trace.csv")
    sets = [sweep.make_flags(trace_file=trace, schedule=s) for s in ("fifo", "sjf")]
    loads, specs = [1.0, 1.25], ["0:1", "0:1,100:3@500", "0:2"]
    nm = 1 if mix is None else 2
    # replicas of shape (configs, loads, mixes * profiles, R): reshape to the profile axis
    recs, bins, cls, hist, prec, phist = fake_outputs(2, 2, nm * 3, 3, 4, 2, 3)
    shape = lambda a: a.reshape(a.shape[:2] + ((nm, 3) if mix is not None else (3,)) + a.shape[3:])
    bounds, edges = (4,), (-10, 0, 100)
    pairs = [(0, 1)]
    writers = {
        "runs": lambda p, r, b, c, h, pr, ph, **k: sweep.write_bootstrap_csv(p, sets, loads, r, **k),
        "ci": lambda p, r, b, c, h, pr, ph, **k: sweep.write_bootstrap_ci_csv(p, sets, loads, r, **k),
        "timeline": lambda p, r, b, c, h, pr, ph, **k: sweep.write_timeline_ci_csv(p, sets, loads, b, 500, **k),
        "jobdist": lambda p, r, b, c, h, pr, ph, **k: sweep.write_jobdist_ci_csv(p, sets, loads, c, h, bounds, edges, **k),
        "paired_summary": lambda p, r, b, c, h, pr, ph, **k: sweep.write_paired_summary_csv(p, sets, pairs, r, loads=loads, **k),
    }
    arrays = [shape(x) for x in (recs, bins, cls, hist, prec, phist)]
    for name, write in writers.items():
        path = str(tmp_path / f"{name}.csv")
        write(path, *arrays, block_len=None, mix=mix, profile=specs)
        q = read_rows(path)
        head = q[0]
        at = head.index("mix") + 1 if mix is not None else head.index("load") + 1
        assert head[at] == "profile", name
        for p in range(3):                                     # one profile alone, without the column
            one = str(tmp_path / f"{name}_{p}.csv")
            write(one, *[a[:, :, :, p] if mix is not None else a[:, :, p] for a in arrays], block_len=None, mix=mix)
            rows = read_rows(one)
            assert rows[0] == head[:at] + head[at + 1:]
            mine = [r[:at] + r[at + 1:] for r in q[1:] if r[at] == specs[p]]
            assert mine == rows[1:], (name, p)
        keys = [tuple(r[head.index("load"):at + 1]) for r in q[1:]]
        order = [(float(k[0]),) + ((mix.index(k[1]),) if mix is not None else ()) + (specs.index(k[-1]),) for k in keys]
        per_conf = len(order) // (len(pairs) if name == "paired_summary" else len(sets))
        for c in range(len(order) // per_conf):
            chunk = order[c * per_conf:(c + 1) * per_conf]
            assert chunk == sorted(chunk), name

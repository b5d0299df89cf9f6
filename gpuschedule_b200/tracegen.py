"""Synthetic trace generator in the live-path CSV schema.

The reference never committed a trace (its .gitignore excludes data/*.csv), so
every workload in this repo is generated here, deterministically, from a seed.
Schema = the columns the live ingest consumes
(/root/reference/core/jobs/job_generator.py:181-193 and
 /root/reference/core/jobs/jobs_manager.py:233-238):

  type, normalized_time, minutes, gpu_per_container, gpu_utilization_avg,
  gpu_utilization_max, memory_max, memory_avg, used_gpus

plus three optional columns used only by the network-cost model
(/root/reference/core/network/network_service.py:3-39):
  model_name, iterations, ps_count

Distributions follow SURVEY.md section 8(d):
  inter-arrival ~ Exponential(mean 1/rate ticks), cumsum -> floor -> x10000
  used_gpus in {1,2,4,8,16,32} w.p. {.35,.20,.20,.15,.07,.03}
  minutes = clip(LogNormal(4,1), 2, 4000) rounded to 3 dp
  util_avg ~ U(5,90); util_max = min(100, avg + U(1,30))  (3 dp)
  memory_max = randint(512, 16384) MiB as integer bytes; memory_avg a fraction
"""
from __future__ import annotations

import collections
import operator

import numpy as np

# Iteration-count sample of the reference's distribution-driven generator
# (/root/reference/core/jobs/job_generator.py:24-31) -- values only, used as a
# sampling population for the optional `iterations` column.
_ITER_POP = np.array(
    [1, 1, 1, 1, 1, 1, 109, 126, 133, 138, 141, 143, 144, 147, 157, 168, 175,
     192, 193, 198, 235, 237, 242, 253, 258, 272, 272, 274, 288, 326, 326,
     362, 386, 391, 410, 438, 447, 468, 473, 513, 513, 521, 521, 525, 581,
     606, 607, 775, 775, 789, 822, 864, 864, 892, 903, 949, 1011, 1085, 1360,
     1501, 2178, 2239, 2275, 3304, 3469, 4861], dtype=np.int64)

GPU_CHOICES = np.array([1, 2, 4, 8, 16, 32], dtype=np.int64)
GPU_PROBS = np.array([.35, .20, .20, .15, .07, .03])

BASE_SEED = 20260921


def synth_columns(n_jobs: int, seed: int = 1, rate: float = 0.5,
                  gpu_choices=GPU_CHOICES, gpu_probs=GPU_PROBS,
                  gpu_per_container: int = 1, with_network: bool = False,
                  max_mem_mib: int = 16384):
    """Return a dict of column -> numpy array for an `n_jobs` trace."""
    from .model_factory import model_sizes
    rng = np.random.default_rng(BASE_SEED + int(seed))
    gaps = rng.exponential(1.0 / rate, size=n_jobs)
    arrive = np.floor(np.cumsum(gaps)).astype(np.int64)
    arrive -= arrive[0]
    cols = {}
    cols["type"] = np.array(["noninteractive"] * n_jobs, dtype=object)
    cols["normalized_time"] = arrive * 10000
    cols["minutes"] = np.round(
        np.clip(rng.lognormal(4.0, 1.0, size=n_jobs), 2.0, 4000.0), 3)
    cols["gpu_per_container"] = np.full(n_jobs, int(gpu_per_container), dtype=np.int64)
    avg = np.round(rng.uniform(5.0, 90.0, size=n_jobs), 3)
    mx = np.round(np.minimum(100.0, avg + rng.uniform(1.0, 30.0, size=n_jobs)), 3)
    cols["gpu_utilization_avg"] = avg
    cols["gpu_utilization_max"] = np.maximum(mx, avg)
    mem_mib = rng.integers(512, max_mem_mib, size=n_jobs, endpoint=True)
    cols["memory_max"] = mem_mib.astype(np.int64) * (1 << 20)
    cols["memory_avg"] = np.floor(
        cols["memory_max"] * rng.uniform(0.3, 0.9, size=n_jobs)).astype(np.int64)
    g = rng.choice(np.asarray(gpu_choices), size=n_jobs, p=np.asarray(gpu_probs))
    g = np.maximum(g // gpu_per_container, 1) * gpu_per_container
    cols["used_gpus"] = g.astype(np.int64)
    cols["model"] = np.array(["V100"] * n_jobs, dtype=object)
    if with_network:
        names = np.array(sorted(model_sizes.keys()), dtype=object)
        cols["model_name"] = names[rng.integers(0, len(names), size=n_jobs)]
        cols["iterations"] = _ITER_POP[rng.integers(0, len(_ITER_POP), size=n_jobs)]
        cols["ps_count"] = (cols["used_gpus"] // cols["gpu_per_container"]).astype(np.int64)
    return cols


# ---- bootstrap replicas: the host mirror of gs_boot_traces (gpuschedule_b200/csrc/gs_boot.cuh), bit for bit
_PHILOX_M = (np.uint64(0xD2E7470EE14C6C93), np.uint64(0xCA5A826395121157))
_PHILOX_W = (np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBB67AE8584CAA73B))
_LO32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def mulhi64(a, b):
    """high 64 bits of the 128-bit products a * b (uint64 arrays, broadcast)"""
    a, b = np.asarray(a, dtype=np.uint64), np.asarray(b, dtype=np.uint64)
    a_lo, a_hi, b_lo, b_hi = a & _LO32, a >> _S32, b & _LO32, b >> _S32
    lh, hl = a_lo * b_hi, a_hi * b_lo
    mid = ((a_lo * b_lo) >> _S32) + (lh & _LO32) + (hl & _LO32)
    return a_hi * b_hi + (lh >> _S32) + (hl >> _S32) + (mid >> _S32)


def philox4x64(seed, stream, counters):
    """Philox4x64-10 blocks with key (seed, stream) at `counters` (uint64, shape (..., 4)); returns the four words of
    each block, shape (..., 4).  numpy.random.Philox(key=[seed, stream], counter=c).random_raw(4) is the block at c + 1."""
    c = np.array(counters, dtype=np.uint64)
    if c.shape[-1:] != (4,):
        raise ValueError("counters must have shape (..., 4)")
    c0, c1, c2, c3 = (c[..., i] for i in range(4))
    k0, k1 = np.array(seed, dtype=np.uint64), np.array(stream, dtype=np.uint64)
    with np.errstate(over="ignore"):
        for r in range(10):
            if r:
                k0, k1 = k0 + _PHILOX_W[0], k1 + _PHILOX_W[1]
            hi0, lo0 = mulhi64(_PHILOX_M[0], c0), _PHILOX_M[0] * c0
            hi1, lo1 = mulhi64(_PHILOX_M[1], c2), _PHILOX_M[1] * c2
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return np.stack([c0, c1, c2, c3], axis=-1)


def check_block_len(block_len):
    """the mean block length L of a blocked bootstrap as an int in 1..2^32 - 1, or ValueError"""
    if isinstance(block_len, (bool, np.bool_)):
        raise ValueError("block_len must be an integer in 1..2^32 - 1")
    try:
        L = operator.index(block_len)
    except TypeError:
        raise ValueError("block_len must be an integer in 1..2^32 - 1") from None
    if not 1 <= L <= 2 ** 32 - 1:
        raise ValueError("block_len must be an integer in 1..2^32 - 1")
    return L


def alias_table(weights):
    """The exact integer alias table (Walker / Vose) of per-row weights w (uint32, at least one non-zero), as
    gs_boot_mixes builds it on the host (include/gsched.h): with T = sum w_i and q_i = w_i * K, FIFO worklists
    S = {i : q_i < T} and G = {i : q_i >= T} in ascending row order; while both are non-empty, the front s of S gets
    U_s = q_s, A_s = g (the front of G), q_g -= T - q_s, and g moves to the back of S once q_g < T; every row left in G
    gets U_i = T, A_i = i.  A job with unweighted row c and u = floor(w3 * T / 2^64) takes row c if u < U_c, else A_c.
    Returns (U, A) as uint64 / int64 arrays of K entries."""
    w = check_weights(weights)
    K, T = len(w), sum(w)
    q = [x * K for x in w]
    U, A = [0] * K, [0] * K
    S = collections.deque(i for i in range(K) if q[i] < T)
    G = collections.deque(i for i in range(K) if q[i] >= T)
    while S and G:
        s, g = S.popleft(), G[0]
        U[s], A[s] = q[s], g
        q[g] -= T - q[s]
        if q[g] < T:
            S.append(G.popleft())
    for i in G:
        U[i], A[i] = T, i
    return np.array(U, dtype=np.uint64), np.array(A, dtype=np.int64)


def check_weights(weights, k=None):
    """per-row weights as a list of Python ints in 0..2^32 - 1 with a non-zero sum (and k entries), or ValueError"""
    w = np.asarray(weights)
    if w.ndim != 1 or not len(w) or (w.dtype.kind not in "iu" and not (w.dtype == object and all(isinstance(x, int) for x in w.tolist()))):
        raise ValueError("weights: expected a non-empty 1-d sequence of integers")
    w = [int(x) for x in w.tolist()]
    if any(not 0 <= x <= 2 ** 32 - 1 for x in w):
        raise ValueError("weights: every weight must be in 0..2^32 - 1")
    if k is not None and len(w) != k:
        raise ValueError(f"weights: expected one weight per population row ({k}), got {len(w)}")
    if sum(w) < 1:
        raise ValueError("weights: the weights sum to 0")
    return w


def class_weights(gpus, bounds, multipliers):
    """per-row weights of a job mix given by size class: row i gets multipliers[c], where c, its class, is the number of
    `bounds` <= gpus[i] (the rule of gs_set_jobdist).  Returns uint32 weights, one per row."""
    b = [int(x) for x in bounds]
    if any(x <= y for y, x in zip(b, b[1:])):
        raise ValueError("class_weights: the class bounds must be strictly increasing")
    m = [int(x) for x in multipliers]
    if len(m) != len(b) + 1:
        raise ValueError(f"class_weights: expected {len(b) + 1} multipliers (one per class), got {len(m)}")
    if any(not 0 <= x <= 2 ** 32 - 1 for x in m):
        raise ValueError("class_weights: every multiplier must be in 0..2^32 - 1")
    cls = np.searchsorted(np.asarray(b, dtype=np.int64), np.asarray(gpus, dtype=np.int64), side="right")
    return np.asarray(m, dtype=np.uint32)[cls]


MAX_SEGMENTS = 64


def check_profile(segments, period=0):
    """a load profile (segments, period) as (starts, gap_nums, gap_dens, period), lists of Python ints, or ValueError.
    segments: BOOT_SEG_DTYPE records or (start, gap_num, gap_den) triples, 1..MAX_SEGMENTS of them; the rules of
    gs_boot_profiles (include/gsched.h): the first start 0, starts strictly increasing and below 2^31 - 1, every
    gap_num and gap_den in 1..2^31 - 1, and a period 0 (aperiodic) or above the last start and below 2^31 - 1"""
    a = np.asarray(segments)
    try:
        if a.dtype.names:
            t, num, den = (a[f].tolist() for f in ("start", "gap_num", "gap_den"))
        else:
            if a.ndim != 2 or a.shape[1] != 3 or a.dtype.kind not in "iu" and not (a.dtype == object and all(
                    isinstance(x, (int, np.integer)) and not isinstance(x, bool) for x in a.ravel().tolist())):
                raise ValueError
            t, num, den = ([int(x) for x in a[:, i].tolist()] for i in range(3))
        P = operator.index(period)
    except (TypeError, ValueError, IndexError):
        raise ValueError("profile: expected (segments, period): (start, gap_num, gap_den) integer triples and an integer") from None
    if not 1 <= len(t) <= MAX_SEGMENTS:
        raise ValueError(f"profile: needs 1..{MAX_SEGMENTS} segments, got {len(t)}")
    if t[0] != 0:
        raise ValueError("profile: the first segment must start at tick 0")
    if any(b <= a for a, b in zip(t, t[1:])) or t[-1] >= 2 ** 31 - 1:
        raise ValueError("profile: segment starts must be strictly increasing and below 2^31 - 1")
    if any(not 1 <= x <= 2 ** 31 - 1 for x in num + den):
        raise ValueError("profile: every gap scale needs gap_num and gap_den in 1..2^31 - 1")
    if P < 0 or P >= 2 ** 31 - 1 or 0 < P <= t[-1]:
        raise ValueError("profile: the period must be 0, or above the last start and below 2^31 - 1")
    return t, num, den, P


def profile_base(segments, period=0):
    """the exact host conversion of gs_boot_profiles: base-time starts s_0 = 0,
    s_(k+1) = s_k + ceil((t_(k+1) - t_k) * den_k / num_k), and B = s_m with t_m := P (0 when P = 0).  Returns (s, B)
    as Python ints"""
    t, num, den, P = check_profile(segments, period)
    s, ends = [0], t[1:] + ([P] if P else [])
    for k, end in enumerate(ends):
        s.append(s[-1] + -(-(end - t[k]) * den[k] // num[k]))
    return s[:len(t)], (s[-1] if P else 0)


def profile_arrive(S, segments, period=0):
    """arrival ticks of base times S >= 0 under a profile: a(S) = t_k + floor((S - s_k) * num_k / den_k) with k the
    last segment with s_k <= S, and (S div B) * P + a(S mod B) when P > 0.  S: an int (Python-int result, exact) or
    an int64 array (int64 result; the caller keeps the products below 2^63, as gs_boot_traces_profiled's bound does)"""
    t, num, den, P = check_profile(segments, period)
    s, B = profile_base(segments, period)
    if isinstance(S, (int, np.integer)):
        S = int(S)
        q, S = divmod(S, B) if P else (0, S)
        k = max(i for i in range(len(s)) if s[i] <= S)
        return q * P + t[k] + (S - s[k]) * num[k] // den[k]
    S = np.asarray(S, dtype=np.int64)
    q = np.zeros_like(S)
    if P:
        q, S = np.divmod(S, np.int64(B))
    k = np.searchsorted(np.asarray(s, dtype=np.int64), S, side="right") - 1
    T, sk, nk, dk = (np.asarray(x, dtype=np.int64)[k] for x in (t, s, num, den))
    return q * np.int64(P) + T + (S - sk) * nk // dk


def profile_bound(n, max_gap, segments, period=0):
    """the largest arrival tick any profiled replica of n jobs can reach, arrive((n - 1) * max_gap), exactly"""
    return profile_arrive((int(n) - 1) * int(max_gap), segments, period) if int(n) > 1 else 0


def bootstrap_packed(population, seed, stream, n, gap_num=1, gap_den=1, block_len=1, weights=None, profile=None):
    """Replica (seed, stream) of `n` jobs drawn from `population` (JOBIN_DTYPE records of one trace in admission order):
    job j resamples a row and an inter-arrival gap of the population with the Philox4x64-10 block at counter
    (j + 1, 0, 0, 0), and its arrival is floor(gap sum * gap_num / gap_den) (include/gsched.h, gs_boot_traces).
    block_len=L > 1 resamples blocks of consecutive rows of mean length L instead, each row with the gap that preceded
    it in the population (gs_boot_traces_blocked); L = 1 is the iid bootstrap.  weights (one uint32 per population
    row) draws row i with probability w_i / sum(w) through alias_table, at block starts only when blocked
    (gs_boot_traces_mixed); None is the unweighted bootstrap.  profile=(segments, period) takes the arrivals from a load
    profile, profile_arrive of the gap sums (gs_boot_traces_profiled; gap_num / gap_den must be 1 / 1), and leaves
    every other draw as it is.  Returns (JOBIN_DTYPE records, source rows)."""
    from .capi import JOBIN_DTYPE
    pop = np.ascontiguousarray(population, dtype=JOBIN_DTYPE)
    k, n, gap_num, gap_den = len(pop), int(n), int(gap_num), int(gap_den)
    if k < 1 or not 0 <= n < 2 ** 31 - 64 or gap_num < 0 or gap_den < 1:
        raise ValueError("bootstrap_packed: needs a population of at least one record, 0 <= n < 2^31 - 64, gap_num >= 0, gap_den >= 1")
    L = check_block_len(block_len)
    if weights is not None:
        weights = check_weights(weights, k)
        U, A = alias_table(weights)
    gaps = np.diff(pop["arrive_tick"].astype(np.int64))
    max_gap = int(gaps.max()) if len(gaps) else 0
    if profile is not None:
        if (gap_num, gap_den) != (1, 1):
            raise ValueError("bootstrap_packed: a profiled replica needs gap_num / gap_den = 1 / 1")
        if profile_bound(n, max_gap, *profile) >= 2 ** 31 - 1:
            raise ValueError("bootstrap_packed: the last arrival tick can reach 2^31 - 1 under the profile")
    elif n > 1 and (n - 1) * max_gap * gap_num // gap_den >= 2 ** 31 - 1:
        raise ValueError("bootstrap_packed: the last arrival tick can reach 2^31 - 1")
    ctr = np.zeros((n, 4), dtype=np.uint64)
    ctr[:, 0] = np.arange(1, n + 1, dtype=np.uint64)
    w = philox4x64(seed, stream, ctr)
    rows = mulhi64(w[:, 0], np.uint64(k)).astype(np.int64)
    if weights is not None:                                        # the alias pick: keep column c iff u < U_c
        u = mulhi64(w[:, 3], np.uint64(sum(weights)))
        rows = np.where(u < U[rows], rows, A[rows])
    j = np.arange(n, dtype=np.int64)
    start = mulhi64(w[:, 2], np.uint64(L)) == 0                   # block starts; always for L = 1
    start[:1] = True
    b = np.maximum.accumulate(np.where(start, j, 0)) if n else j  # last block start <= j
    rows = (rows[b] + (j - b)) % k
    g = np.zeros(n, dtype=np.int64)
    if k > 1 and n > 1:
        gi = mulhi64(w[1:, 1], np.uint64(k - 1)).astype(np.int64)
        g[1:] = gaps[np.where(start[1:] | (rows[1:] == 0), gi, rows[1:] - 1)]
    out = np.zeros(n, dtype=JOBIN_DTYPE)
    if profile is not None:
        out["arrive_tick"] = profile_arrive(np.cumsum(g), *profile)
    else:
        out["arrive_tick"] = np.cumsum(g) * gap_num // gap_den   # below 2^62 by the bound checked above
    src = pop[rows]
    for f in ("gpus", "gpu_per_task", "mem_bytes", "duration"):
        out[f] = src[f]
    return out, rows


def bootstrap_table(base_table, seed, stream, n, gap_num=1, gap_den=1, block_len=1, weights=None, profile=None):
    """bootstrap_packed of a JobTable as a JobTable of its own (labels 0..n-1, the source rows' num_gpu_text and
    utilisation columns, submit = arrive), so that a generated replica can go through the ordinary upload path and
    the ordinary log writers."""
    from .ingest import JobTable
    recs, rows = bootstrap_packed(base_table.packed(), seed, stream, n, gap_num, gap_den, block_len, weights, profile)
    pick = lambda a: None if a is None else np.ascontiguousarray(np.asarray(a)[rows])
    t = JobTable(
        n=len(recs), label=[str(i) for i in range(len(recs))],
        num_gpu_text=None if base_table.num_gpu_text is None else [base_table.num_gpu_text[r] for r in rows.tolist()],
        arrive_tick=recs["arrive_tick"].copy(), submit=recs["arrive_tick"].copy(), gpus=recs["gpus"].copy(),
        gpu_per_task=recs["gpu_per_task"].copy(), duration=recs["duration"].copy(), mem_bytes=recs["mem_bytes"].copy(),
        util_avg=pick(base_table.util_avg), util_max=pick(base_table.util_max))
    if "mem_avg_mib" in base_table.extra:
        t.extra["mem_avg_mib"] = pick(base_table.extra["mem_avg_mib"])
    return t


def synth_frame(n_jobs: int, **kw):
    import pandas as pd
    return pd.DataFrame(synth_columns(n_jobs, **kw))


def write_trace(path: str, n_jobs: int, **kw) -> str:
    synth_frame(n_jobs, **kw).to_csv(path, index=False)
    return path


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser(description="write a synthetic live-schema trace CSV")
    ap.add_argument("out")
    ap.add_argument("--jobs", type=int, default=1000)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--rate", type=float, default=0.5)
    ap.add_argument("--network", action="store_true")
    a = ap.parse_args()
    write_trace(a.out, a.jobs, seed=a.seed, rate=a.rate, with_network=a.network)

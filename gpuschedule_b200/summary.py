"""Derived numbers of run summaries (capi.SUMMARY_DTYPE records from gs_summarize / gs_horus_summarize): the few
values the reference's notebooks compute from a run's cluster.csv and job.csv.  Post-processing only, like
log_manager: every number follows from the record and the cluster shape.

    gpu_share          busy_gpus_sum / (rows * M * G)                      mean num_busy_gpus over the GPUs
    mem_mean           mean of the avg_gpu_memory_allocated column
    pending_mean       avg_pending_sum / pending_rows                      mean of avg_pending_time where it is non-zero
    wait_mean, turnaround_mean, jct_mean                                   means over the lines of job.csv
    util_mean          util_sum / rows (horus engine; NaN otherwise)       mean of avg_gpu_utilization, NaN as 0

`spread` takes many records of one configuration (bootstrap replicas, sweep.summarize_bootstrap) and gives, for the
makespan and each derived number, the mean, the sample standard deviation and a nearest-rank percentile interval.

Timelines (capi.TBIN_DTYPE bins from Engine.timeline / HorusEngine.timeline): `timeline_derived` gives the same kind
of numbers per bin -- the curves the notebooks plot against `delta` -- and `timeline_spread` their spread per bin over
the replicas that have rows in that bin (what groupby("delta").mean() averages over).

Job statistics by job size (capi.JCLASS_DTYPE records and CDF counts from Engine.jobdist / HorusEngine.jobdist):
`jobdist_derived` gives per class the job count, the mean, sample std (pandas' .std()) and five quantiles of wait,
turnaround and jct, and their CDF at every edge -- job_analysis.ipynb's breakdown by used_gpus and
scheduler_analysis.ipynb's mean / median / std -- and `jobdist_spread` their spread per class over the replicas that
have jobs in that class.

Job statistics by a chosen key with bounded slowdown (capi.SDCLASS_DTYPE records and CDF counts from
Engine.slowdown / HorusEngine.slowdown): `slowdown_derived` gives per class jobdist's numbers, the mean key and the
mean, sample std, minimum and five quantiles of the bounded slowdown (in units of slowdown: the record's fixed point
over 1024), and the four CDFs; `slowdown_spread` their spread per class over the replicas that have jobs in it.

Interference of the utilisation-aware engine (capi.IFCLASS_DTYPE records from HorusEngine.interference):
`interference_derived` gives per class scheduler_analysis.ipynb's "Degrade_Only" line (mean, median and sample std of
the jct of the jobs co-location slowed, actual > original) and its "normal" line (the same of actual_duration over
every finished job, in ticks), the share of jobs degraded, their mean excess, the GPU time they lost, the share
preempted more than once, and jobdist's numbers of the degraded and the clean jobs; `interference_spread` their spread
per class over runs (seeded repeats) that have jobs in it.

Time-weighted occupancy (capi.OCC_DTYPE records and histograms from Engine.occupancy / HorusEngine.occupancy):
`occupancy_derived` gives the time-weighted GPU share, the shares of time saturated and with jobs waiting, the GPU
time left idle while jobs waited, mean running and queued jobs, busy-GPU points over all time and over waiting time,
and the queue-length CDF; `occupancy_spread` their spread over replicas.

Paired comparisons (capi.JPAIR_DTYPE records and CDF counts from Engine.compare / HorusEngine.compare): `pair_derived`
gives per class and quantity the per-job differences d = x_b - x_a of two configurations on the same trace -- their
mean, sample std, shares below / at / above zero, ten order statistics and CDF --, `pair_spread` their spread over
replicas, and `paired_spread` the replica-level differences b - a of the makespan and every derived number.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

QUANTILES = (50, 90, 95, 99, 100)


def u128(lo, hi):
    """an exact Python int from the two 64-bit halves of a 128-bit field"""
    return (int(hi) << 64) | int(lo)


def _div(a, b):
    return a / b if b else math.nan


def derived(rec, n_nodes, gpus_per_node, gpu_mem_cap_mib):
    """dict of the derived numbers of one record (cluster: M nodes of G GPUs, gpu_mem_cap_mib MiB each)"""
    rows = int(rec["rows"])
    k = int(rec["finished"])
    mem = u128(rec["mem_busy_lo"], rec["mem_busy_hi"])
    return dict(
        gpu_share=_div(int(rec["busy_gpus_sum"]), rows * n_nodes * gpus_per_node),
        mem_mean=_div(mem / 1048576.0 / (n_nodes * gpus_per_node * gpu_mem_cap_mib), rows),
        pending_mean=_div(float(rec["avg_pending_sum"]), int(rec["pending_rows"])),
        wait_mean=_div(int(rec["wait_sum"]), k),
        turnaround_mean=_div(int(rec["turnaround_sum"]), k),
        jct_mean=_div(int(rec["jct_sum"]), k),
        util_mean=_div(float(rec["util_sum"]), rows),
    )


SPREAD_METRICS = ("makespan", "gpu_share", "mem_mean", "pending_mean", "wait_mean", "turnaround_mean", "jct_mean", "util_mean")
SPREAD_STATS = ("mean", "std", "lo", "hi")


def nearest_rank(q, k):
    """index of the element at fraction q (a Fraction, or a number taken by its decimal text) of k > 0 sorted values:
    ceil(q * k) - 1, at least 0 -- gs_summary's rule, where q is given in per mille"""
    q = q if isinstance(q, Fraction) else Fraction(str(q))
    return max(-((-q.numerator * k) // q.denominator) - 1, 0)


def spread(records, n_nodes, gpus_per_node, gpu_mem_cap_mib, level=0.95):
    """Spread across replicas (e.g. bootstrap replicas of one configuration) of the makespan and of every derived
    number: {metric: {mean, std (sample, ddof 1), lo, hi}}, where [lo, hi] is the nearest-rank interval holding the
    central `level` of the replicas' values.  A metric that is NaN for any replica is NaN throughout; std is NaN for
    fewer than two replicas."""
    level = Fraction(str(level))
    if not 0 < level <= 1:
        raise ValueError("level must be in (0, 1]")
    cols = {m: [] for m in SPREAD_METRICS}
    for rec in records:
        d = derived(rec, n_nodes, gpus_per_node, gpu_mem_cap_mib)
        cols["makespan"].append(float(rec["makespan"]))
        for m in SPREAD_METRICS[1:]:
            cols[m].append(d[m])
    return {m: _spread_of(np.asarray(vals, dtype=np.float64), level) for m, vals in cols.items()}


def _spread_of(v, level):
    """mean, sample std and nearest-rank interval of the values v (level: a Fraction); NaN throughout if any is NaN"""
    k = len(v)
    if k == 0 or np.isnan(v).any():
        return dict.fromkeys(SPREAD_STATS, math.nan)
    s = np.sort(v)
    return dict(mean=float(v.mean()), std=float(v.std(ddof=1)) if k > 1 else math.nan,
                lo=float(s[nearest_rank((1 - level) / 2, k)]), hi=float(s[nearest_rank((1 + level) / 2, k)]))


def spread_columns():
    """names of the flat columns of a spread, in the order `spread_flat` returns them"""
    return [f"{m}_{s}" for m in SPREAD_METRICS for s in SPREAD_STATS]


def spread_flat(sp):
    return [sp[m][s] for m in SPREAD_METRICS for s in SPREAD_STATS]


def columns():
    """names of the flat columns `flat` returns, in order"""
    names = ["n", "rows", "done", "status", "makespan", "busy_gpus_sum", "running_sum", "queued_sum", "busy_gpus_max",
             "running_max", "queued_max", "pend_max_max", "pend_sum_sum", "mem_busy_sum", "pending_rows", "avg_pending_sum",
             "util_sum", "finished", "wait_sum", "turnaround_sum", "jct_sum", "preempt_sum", "gpu_ticks_sum"]
    for col in ("wait", "turnaround", "jct"):
        names += [f"{col}_p{q}" for q in QUANTILES]
    return names + ["gpu_share", "mem_mean", "pending_mean", "wait_mean", "turnaround_mean", "jct_mean", "util_mean"]


def flat(rec, n_nodes, gpus_per_node, gpu_mem_cap_mib):
    """one record as a list of Python values in the order of `columns()` (128-bit fields as exact ints)"""
    vals = []
    for name in columns()[:23]:
        if name == "pend_sum_sum":
            vals.append(u128(rec["pend_sum_lo"], rec["pend_sum_hi"]))
        elif name == "mem_busy_sum":
            vals.append(u128(rec["mem_busy_lo"], rec["mem_busy_hi"]))
        elif name in ("avg_pending_sum", "util_sum"):
            vals.append(float(rec[name]))
        else:
            vals.append(int(rec[name]))
    for col in ("wait_q", "turnaround_q", "jct_q"):
        vals += [int(v) for v in rec[col]]
    d = derived(rec, n_nodes, gpus_per_node, gpu_mem_cap_mib)
    return vals + [d[k] for k in ("gpu_share", "mem_mean", "pending_mean", "wait_mean", "turnaround_mean", "jct_mean", "util_mean")]


# ---------------------------------------------------------------- timelines
TIMELINE_METRICS = ("gpu_share", "running_mean", "queued_mean", "mem_mean", "pending_mean_all", "pending_mean_nz", "pend_max",
                    "util_mean", "finished_last")


def _u128_float(lo, hi):
    """float64 of 128-bit fields, elementwise (exactly rounded, as float(u128(lo, hi)))"""
    lo, hi = np.asarray(lo, dtype=np.uint64), np.asarray(hi, dtype=np.uint64)
    out = lo.astype(np.float64)
    for idx in zip(*np.nonzero(hi)):
        out[idx] = float(u128(lo[idx], hi[idx]))
    return out


def timeline_derived(bins, n_nodes, gpus_per_node, gpu_mem_cap_mib):
    """Per-bin numbers of TBIN_DTYPE bins (any shape; every array has that shape).  NaN where a bin has no rows:
        delta_min, delta_max   the bin's smallest / largest `delta` (its tick range)
        rows                   its rows (int)
        gpu_share              busy_gpus_sum / (rows * M * G)
        running_mean, queued_mean   mean num_running_jobs / num_queuing_jobs
        mem_mean               mean avg_gpu_memory_allocated
        pending_mean_all       avg_pending_sum / rows: mean avg_pending_time over all rows (the time plots' curve)
        pending_mean_nz        avg_pending_sum / pending_rows: over the rows where it is non-zero (the bar charts')
        pend_max               max max_pending_time
        util_mean              util_sum / rows (horus engine; NaN otherwise)
        finished_last          jobs finished by the bin's last row"""
    bins = np.asarray(bins)
    rows = bins["rows"].astype(np.int64)
    empty = rows == 0
    r = np.where(empty, np.nan, rows.astype(np.float64))
    mg = n_nodes * gpus_per_node
    with np.errstate(invalid="ignore", divide="ignore"):
        pr = bins["pending_rows"].astype(np.float64)
        mem = _u128_float(bins["mem_busy_lo"], bins["mem_busy_hi"])
        out = dict(
            delta_min=np.where(empty, np.nan, bins["delta_min"].astype(np.float64)),
            delta_max=np.where(empty, np.nan, bins["delta_max"].astype(np.float64)),
            rows=rows,
            gpu_share=bins["busy_gpus_sum"].astype(np.float64) / (r * mg),
            running_mean=bins["running_sum"].astype(np.float64) / r,
            queued_mean=bins["queued_sum"].astype(np.float64) / r,
            mem_mean=mem / 1048576.0 / (mg * gpu_mem_cap_mib) / r,
            pending_mean_all=bins["avg_pending_sum"] / r,
            pending_mean_nz=np.where(pr > 0, bins["avg_pending_sum"] / np.where(pr > 0, pr, 1.0), np.nan),   # (empty bins have none)
            pend_max=np.where(empty, np.nan, bins["pend_max_max"].astype(np.float64)),
            util_mean=bins["util_sum"] / r,
            finished_last=np.where(empty, np.nan, bins["finished_last"].astype(np.float64)),
        )
    return out


def timeline_spread(bins, n_nodes, gpus_per_node, gpu_mem_cap_mib, level=0.95):
    """Spread per bin across replicas: `bins` has shape (replicas, B).  For every bin, over the replicas that have rows
    in it: {"replicas": int array (B,), metric: {mean, std, lo, hi: float arrays (B,)}} for every TIMELINE_METRICS
    entry, with spread's rules (sample std, nearest-rank interval holding the central `level`; NaN throughout where a
    value is NaN for any of those replicas or none has rows)."""
    level = Fraction(str(level))
    if not 0 < level <= 1:
        raise ValueError("level must be in (0, 1]")
    bins = np.asarray(bins)
    if bins.ndim != 2:
        raise ValueError("timeline_spread: bins must have shape (replicas, bins)")
    d = timeline_derived(bins, n_nodes, gpus_per_node, gpu_mem_cap_mib)
    reach = d["rows"] > 0
    nb = bins.shape[1]
    out = {"replicas": reach.sum(axis=0).astype(np.int64)}
    for m in TIMELINE_METRICS:
        cols = [_spread_of(d[m][reach[:, b], b], level) for b in range(nb)]
        out[m] = {s: np.array([c[s] for c in cols], dtype=np.float64) for s in SPREAD_STATS}
    return out


def timeline_columns():
    """names of the flat per-bin columns `timeline_flat` returns, in order"""
    return ["delta_min", "delta_max", "rows"] + list(TIMELINE_METRICS)


def timeline_flat(d, b):
    """bin b of a timeline_derived dict as a list of Python values (ints for counts, NaN kept)"""
    vals = []
    for name in timeline_columns():
        v = d[name][b]
        vals.append(int(v) if name == "rows" or (name in ("delta_min", "delta_max", "pend_max", "finished_last") and not np.isnan(v))
                    else float(v))
    return vals


def timeline_spread_columns():
    return [f"{m}_{s}" for m in TIMELINE_METRICS for s in SPREAD_STATS]


def timeline_spread_flat(sp, b):
    return [float(sp[m][s][b]) for m in TIMELINE_METRICS for s in SPREAD_STATS]


# ---------------------------------------------------------------- job statistics by job size
JOBDIST_QUANTITIES = ("wait", "turnaround", "jct")
JOBDIST_STATS = ("mean", "std") + tuple(f"p{q}" for q in QUANTILES)
JOBDIST_METRICS = tuple(f"{m}_{s}" for m in JOBDIST_QUANTITIES for s in JOBDIST_STATS)


def _jclass_numbers(rec):
    """the JOBDIST_METRICS of one JCLASS_DTYPE record as a dict of floats (NaN for an empty class; std NaN below two
    jobs).  The sample variance (n * sumsq - sum^2) / (n * (n - 1)) is exact in Python ints and rounded once."""
    n = int(rec["jobs"])
    out = {}
    for m in JOBDIST_QUANTITIES:
        s, sq = int(rec[m + "_sum"]), u128(rec[m + "_sq_lo"], rec[m + "_sq_hi"])
        out[m + "_mean"] = s / n if n else math.nan
        out[m + "_std"] = math.sqrt(float(Fraction(n * sq - s * s, n * (n - 1)))) if n > 1 else math.nan
        for q, v in zip(QUANTILES, rec[m + "_q"].tolist()):
            out[f"{m}_p{q}"] = float(v) if n else math.nan
    return out


def jobdist_derived(classes, hist, edges):
    """Per class of one replica: `classes` JCLASS_DTYPE (C,), `hist` CDF counts (C, 3, E + 1), `edges` the E edges.
    Returns {"jobs": int array (C,), metric: float array (C,) for every JOBDIST_METRICS entry,
    "<quantity>_cdf": float array (C, E) = #(value <= edge) / jobs}; NaN for an empty class."""
    classes, hist = np.asarray(classes), np.asarray(hist, dtype=np.int64)
    if classes.ndim != 1 or hist.shape != (len(classes), 3, len(edges) + 1):
        raise ValueError("jobdist_derived: expected classes (C,) and hist (C, 3, len(edges) + 1)")
    jobs = classes["jobs"].astype(np.int64)
    out = {"jobs": jobs}
    nums = [_jclass_numbers(rec) for rec in classes]
    for name in JOBDIST_METRICS:
        out[name] = np.array([d[name] for d in nums], dtype=np.float64)
    cum = np.cumsum(hist, axis=2)[:, :, :len(edges)]
    with np.errstate(invalid="ignore", divide="ignore"):
        for i, m in enumerate(JOBDIST_QUANTITIES):
            out[m + "_cdf"] = np.where(jobs[:, None] > 0, cum[:, i, :] / np.where(jobs > 0, jobs, 1)[:, None], np.nan)
    return out


def jobdist_spread(classes, hist, edges, level=0.95):
    """Spread per class across replicas: `classes` (replicas, C), `hist` (replicas, C, 3, E + 1).  For every class,
    over the replicas that have at least one job in it: {"replicas": int array (C,), metric: {mean, std, lo, hi: float
    arrays (C,)} for every JOBDIST_METRICS entry, "<quantity>_cdf": {mean, std, lo, hi: float arrays (C, E)}}, with
    spread's rules (sample std, nearest-rank interval holding the central `level`, NaN where a value is NaN for any
    of those replicas or no replica has jobs in the class)."""
    level = Fraction(str(level))
    if not 0 < level <= 1:
        raise ValueError("level must be in (0, 1]")
    classes, hist = np.asarray(classes), np.asarray(hist)
    if classes.ndim != 2 or hist.shape != classes.shape + (3, len(edges) + 1):
        raise ValueError("jobdist_spread: expected classes (replicas, C) and hist (replicas, C, 3, len(edges) + 1)")
    per = [jobdist_derived(classes[r], hist[r], edges) for r in range(classes.shape[0])]
    nc, ne = classes.shape[1], len(edges)
    reach = classes["jobs"] > 0
    out = {"replicas": reach.sum(axis=0).astype(np.int64)}
    for name in JOBDIST_METRICS:
        cols = [_spread_of(np.array([d[name][c] for r, d in enumerate(per) if reach[r, c]], dtype=np.float64), level) for c in range(nc)]
        out[name] = {s: np.array([col[s] for col in cols], dtype=np.float64) for s in SPREAD_STATS}
    for m in JOBDIST_QUANTITIES:
        st = {s: np.full((nc, ne), math.nan) for s in SPREAD_STATS}
        cdf = np.stack([d[m + "_cdf"] for d in per]) if per else np.zeros((0, nc, ne))
        for c in range(nc):
            sub = cdf[reach[:, c], c, :]
            for e in range(ne):
                sp = _spread_of(sub[:, e], level)
                for s in SPREAD_STATS:
                    st[s][c, e] = sp[s]
        out[m + "_cdf"] = st
    return out


def jobdist_columns():
    """names of the flat per-class columns `jobdist_flat` returns, in order"""
    return ["jobs"] + list(JOBDIST_METRICS)


def jobdist_flat(d, c):
    """class c of a jobdist_derived dict as a list of Python values"""
    return [int(d["jobs"][c])] + [float(d[name][c]) for name in JOBDIST_METRICS]


def jobdist_spread_columns():
    return [f"{name}_{s}" for name in JOBDIST_METRICS for s in SPREAD_STATS]


def jobdist_spread_flat(sp, c):
    return [float(sp[name][s][c]) for name in JOBDIST_METRICS for s in SPREAD_STATS]


# ---------------------------------------------------------------- job statistics by key with bounded slowdown
SLOWDOWN_ONE = 1024                                       # fixed-point units of sd per unit of slowdown
SLOWDOWN_QUANTITIES = JOBDIST_QUANTITIES + ("sd",)
SLOWDOWN_METRICS = ("key_mean", "sd_mean", "sd_std") + tuple(f"sd_p{q}" for q in QUANTILES) + ("sd_min",) + JOBDIST_METRICS
SLOWDOWN_COUNTS = ("jobs", "sd_clamped")


def _sdclass_numbers(rec):
    """the SLOWDOWN_METRICS of one SDCLASS_DTYPE record as a dict of floats (NaN for an empty class; std NaN below two
    jobs).  The slowdown numbers are in units of slowdown; mean and sample variance are exact in Python ints and
    rounded once (the division by 1024 is exact)."""
    n = int(rec["jc"]["jobs"])
    out = _jclass_numbers(rec["jc"])
    s, sq = int(rec["sd_sum"]), u128(rec["sd_sq_lo"], rec["sd_sq_hi"])
    out["key_mean"] = u128(rec["key_sum_lo"], rec["key_sum_hi"]) / n if n else math.nan
    out["sd_mean"] = s / (n * SLOWDOWN_ONE) if n else math.nan
    out["sd_std"] = math.sqrt(float(Fraction(n * sq - s * s, n * (n - 1)))) / SLOWDOWN_ONE if n > 1 else math.nan
    for q, v in zip(QUANTILES, rec["sd_q"].tolist()):
        out[f"sd_p{q}"] = v / SLOWDOWN_ONE if n else math.nan
    out["sd_min"] = int(rec["sd_min"]) / SLOWDOWN_ONE if n else math.nan
    return out


def _sd_rows(hist, ne, nsd):
    """the (C, 4, ...) CDF count rows of a (C, 3 * (ne + 1) + nsd + 1) slowdown histogram: three of ne + 1, one of nsd + 1"""
    nb = ne + 1
    return [hist[:, m * nb:(m + 1) * nb] for m in range(3)] + [hist[:, 3 * nb:3 * nb + nsd + 1]]


def slowdown_derived(recs, hist, edges, sd_edges):
    """Per class of one replica: `recs` SDCLASS_DTYPE (C,), `hist` CDF counts (C, 3 * (E + 1) + Esd + 1), `edges` the E
    edges of wait / turnaround / jct, `sd_edges` the Esd edges of sd (units of 1/1024).  Returns {"jobs", "sd_clamped":
    int arrays (C,), metric: float array (C,) for every SLOWDOWN_METRICS entry, "<quantity>_cdf": float array (C, E)
    (C, Esd for sd) = #(value <= edge) / jobs}; NaN for an empty class."""
    recs, hist = np.asarray(recs), np.asarray(hist, dtype=np.int64)
    ne, nsd = len(edges), len(sd_edges)
    if recs.ndim != 1 or hist.shape != (len(recs), 3 * (ne + 1) + nsd + 1):
        raise ValueError("slowdown_derived: expected recs (C,) and hist (C, 3 * (len(edges) + 1) + len(sd_edges) + 1)")
    jobs = recs["jc"]["jobs"].astype(np.int64)
    out = {"jobs": jobs, "sd_clamped": recs["sd_clamped"].astype(np.int64)}
    nums = [_sdclass_numbers(rec) for rec in recs]
    for name in SLOWDOWN_METRICS:
        out[name] = np.array([d[name] for d in nums], dtype=np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        for m, rows, n_e in zip(SLOWDOWN_QUANTITIES, _sd_rows(hist, ne, nsd), (ne, ne, ne, nsd)):
            cum = np.cumsum(rows, axis=1)[:, :n_e]
            out[m + "_cdf"] = np.where(jobs[:, None] > 0, cum / np.where(jobs > 0, jobs, 1)[:, None], np.nan)
    return out


def slowdown_spread(recs, hist, edges, sd_edges, level=0.95):
    """Spread per class across replicas: `recs` (replicas, C), `hist` (replicas, C, 3 * (E + 1) + Esd + 1).  For every
    class, over the replicas that have at least one job in it: {"replicas": int array (C,), metric: {mean, std, lo, hi:
    float arrays (C,)} for every SLOWDOWN_METRICS entry, "<quantity>_cdf": {mean, std, lo, hi: float arrays (C, E)
    (C, Esd for sd)}}, with spread's rules (sample std, nearest-rank interval holding the central `level`, NaN where a
    value is NaN for any of those replicas or no replica has jobs in the class)."""
    level = Fraction(str(level))
    if not 0 < level <= 1:
        raise ValueError("level must be in (0, 1]")
    recs, hist = np.asarray(recs), np.asarray(hist)
    if recs.ndim != 2 or hist.shape != recs.shape + (3 * (len(edges) + 1) + len(sd_edges) + 1,):
        raise ValueError("slowdown_spread: expected recs (replicas, C) and hist (replicas, C, 3 * (len(edges) + 1) + len(sd_edges) + 1)")
    per = [slowdown_derived(recs[r], hist[r], edges, sd_edges) for r in range(recs.shape[0])]
    nc = recs.shape[1]
    reach = recs["jc"]["jobs"] > 0
    out = {"replicas": reach.sum(axis=0).astype(np.int64)}
    for name in SLOWDOWN_METRICS:
        cols = [_spread_of(np.array([d[name][c] for r, d in enumerate(per) if reach[r, c]], dtype=np.float64), level) for c in range(nc)]
        out[name] = {s: np.array([col[s] for col in cols], dtype=np.float64) for s in SPREAD_STATS}
    for m, ne in zip(SLOWDOWN_QUANTITIES, (len(edges),) * 3 + (len(sd_edges),)):
        st = {s: np.full((nc, ne), math.nan) for s in SPREAD_STATS}
        cdf = np.stack([d[m + "_cdf"] for d in per]) if per else np.zeros((0, nc, ne))
        for c in range(nc):
            sub = cdf[reach[:, c], c, :]
            for e in range(ne):
                sp = _spread_of(sub[:, e], level)
                for s in SPREAD_STATS:
                    st[s][c, e] = sp[s]
        out[m + "_cdf"] = st
    return out


def slowdown_columns():
    """names of the flat per-class columns `slowdown_flat` returns, in order"""
    return list(SLOWDOWN_COUNTS) + list(SLOWDOWN_METRICS)


def slowdown_flat(d, c):
    """class c of a slowdown_derived dict as a list of Python values"""
    return [int(d[k][c]) for k in SLOWDOWN_COUNTS] + [float(d[name][c]) for name in SLOWDOWN_METRICS]


def slowdown_spread_columns():
    return [f"{name}_{s}" for name in SLOWDOWN_METRICS for s in SPREAD_STATS]


def slowdown_spread_flat(sp, c):
    return [float(sp[name][s][c]) for name in SLOWDOWN_METRICS for s in SPREAD_STATS]


# ---------------------------------------------------------------- job statistics by arrival time
ARRIVAL_COUNTS = ("arrived", "jobs", "unfinished", "sd_clamped")
ARRIVAL_METRICS = SLOWDOWN_METRICS                        # key_mean: the mean arrival tick of the bin's finished jobs
ARRIVAL_SPREAD_METRICS = ("arrived", "jobs", "unfinished") + ARRIVAL_METRICS


def _i128(lo, hi):
    v = u128(lo, hi)
    return v - (1 << 128) if v >> 127 else v


def arrivals_derived(recs):
    """Per arrival bin of one replica: `recs` ABIN_DTYPE (B,).  Returns {"arrived", "jobs", "unfinished" (arrived -
    jobs), "sd_clamped": int arrays (B,), metric: float array (B,) for every ARRIVAL_METRICS entry}, the numbers of
    slowdown_derived over each bin's finished jobs, with key_mean the mean arrival tick; NaN for a bin without
    finished jobs."""
    recs = np.asarray(recs)
    if recs.ndim != 1:
        raise ValueError("arrivals_derived: expected recs (B,)")
    s = recs["s"]
    jobs = s["jc"]["jobs"].astype(np.int64)
    arrived = recs["arrived"].astype(np.int64)
    out = {"arrived": arrived, "jobs": jobs, "unfinished": arrived - jobs, "sd_clamped": s["sd_clamped"].astype(np.int64)}
    nums = [_sdclass_numbers(rec) for rec in s]
    for d, rec, n in zip(nums, s, jobs.tolist()):
        d["key_mean"] = _i128(rec["key_sum_lo"], rec["key_sum_hi"]) / n if n else math.nan
    for name in ARRIVAL_METRICS:
        out[name] = np.array([d[name] for d in nums], dtype=np.float64)
    return out


def arrivals_spread(recs, level=0.95):
    """Spread per bin across replicas: `recs` ABIN_DTYPE (replicas, B).  For every bin, over the replicas with at least
    one finished job in it: {"replicas": int array (B,), metric: {mean, std, lo, hi: float arrays (B,)} for every
    ARRIVAL_SPREAD_METRICS entry}, with spread's rules (sample std, nearest-rank interval holding the central `level`,
    NaN where no replica has finished jobs in the bin)."""
    level = Fraction(str(level))
    if not 0 < level <= 1:
        raise ValueError("level must be in (0, 1]")
    recs = np.asarray(recs)
    if recs.ndim != 2:
        raise ValueError("arrivals_spread: expected recs (replicas, B)")
    per = [arrivals_derived(recs[r]) for r in range(recs.shape[0])]
    nb = recs.shape[1]
    reach = recs["s"]["jc"]["jobs"] > 0
    out = {"replicas": reach.sum(axis=0).astype(np.int64)}
    for name in ARRIVAL_SPREAD_METRICS:
        cols = [_spread_of(np.array([d[name][b] for r, d in enumerate(per) if reach[r, b]], dtype=np.float64), level) for b in range(nb)]
        out[name] = {s: np.array([col[s] for col in cols], dtype=np.float64) for s in SPREAD_STATS}
    return out


def arrivals_columns():
    """names of the flat per-bin columns `arrivals_flat` returns, in order"""
    return list(ARRIVAL_COUNTS) + list(ARRIVAL_METRICS)


def arrivals_flat(d, b):
    """bin b of an arrivals_derived dict as a list of Python values"""
    return [int(d[k][b]) for k in ARRIVAL_COUNTS] + [float(d[name][b]) for name in ARRIVAL_METRICS]


def arrivals_spread_columns():
    return [f"{name}_{s}" for name in ARRIVAL_SPREAD_METRICS for s in SPREAD_STATS]


def arrivals_spread_flat(sp, b):
    return [float(sp[name][s][b]) for name in ARRIVAL_SPREAD_METRICS for s in SPREAD_STATS]


# ---------------------------------------------------------------- interference (utilisation-aware engine)
IF_ONE = 1024                                             # fixed-point units per tick
IF_COUNTS = ("jobs", "degraded", "preempted_jobs", "clamped")
IF_NOTEBOOK = ("degraded_jct_mean", "degraded_jct_median", "degraded_jct_std", "actual_mean", "actual_median", "actual_std")
IF_METRICS = (IF_NOTEBOOK + ("degraded_share", "excess_mean", "lost_gpu_time", "preempted_share")
              + tuple(f"{g}_{m}" for g in ("degraded", "clean") for m in JOBDIST_METRICS if f"{g}_{m}" not in IF_NOTEBOOK))


def _ifclass_numbers(rec):
    """the IF_COUNTS and IF_METRICS of one IFCLASS_DTYPE record (durations in ticks: the fixed point over 1024, an
    exact division; NaN where a group is empty; std NaN below two jobs).  Means and sample variances are exact in
    Python ints and rounded once."""
    kd, kc = int(rec["degraded"]["jobs"]), int(rec["clean"]["jobs"])
    n = kd + kc
    out = dict(jobs=n, degraded=kd, preempted_jobs=int(rec["preempted_jobs"]), clamped=int(rec["clamped"]))
    deg, cln = _jclass_numbers(rec["degraded"]), _jclass_numbers(rec["clean"])
    out["degraded_jct_mean"], out["degraded_jct_std"] = deg["jct_mean"], deg["jct_std"]
    out["degraded_jct_median"] = sum(int(v) for v in rec["degraded_jct_mid"]) / 2 if kd else math.nan
    s, sq = int(rec["actual_sum"]), u128(rec["actual_sq_lo"], rec["actual_sq_hi"])
    out["actual_mean"] = s / (n * IF_ONE) if n else math.nan
    out["actual_median"] = sum(int(v) for v in rec["actual_mid"]) / (2 * IF_ONE) if n else math.nan
    out["actual_std"] = math.sqrt(float(Fraction(n * sq - s * s, n * (n - 1)))) / IF_ONE if n > 1 else math.nan
    lost = u128(rec["lost_gpu_time_lo"], rec["lost_gpu_time_hi"])
    out["degraded_share"] = kd / n if n else math.nan
    out["excess_mean"] = int(rec["excess_sum"]) / (kd * IF_ONE) if kd else math.nan
    out["lost_gpu_time"] = lost / IF_ONE if n else math.nan
    out["preempted_share"] = int(rec["preempted_jobs"]) / n if n else math.nan
    for g, d in (("degraded", deg), ("clean", cln)):
        for m in JOBDIST_METRICS:
            out.setdefault(f"{g}_{m}", d[m])
    return out


def interference_derived(recs):
    """Per class of one replica: `recs` IFCLASS_DTYPE (C,).  Returns {count: int array (C,) for every IF_COUNTS entry,
    metric: float array (C,) for every IF_METRICS entry}.  degraded_jct_mean / _median / _std are the notebook's
    "Degrade_Only" jct.mean() / .median() / .std() and actual_mean / _median / _std its "normal" actual_duration ones
    (to within 2^-11 tick: the durations are kept in units of 2^-10)."""
    recs = np.asarray(recs)
    if recs.ndim != 1:
        raise ValueError("interference_derived: expected IFCLASS_DTYPE records (C,)")
    nums = [_ifclass_numbers(rec) for rec in recs]
    out = {k: np.array([d[k] for d in nums], dtype=np.int64) for k in IF_COUNTS}
    for name in IF_METRICS:
        out[name] = np.array([d[name] for d in nums], dtype=np.float64)
    return out


def interference_spread(recs, level=0.95):
    """Spread per class across runs (e.g. seeded repeats of one configuration): `recs` (runs, C).  For every class,
    over the runs that have at least one finished job in it: {"replicas": int array (C,), metric: {mean, std, lo, hi:
    float arrays (C,)} for every IF_METRICS entry}, with spread's rules (sample std, nearest-rank interval holding the
    central `level`, NaN where a value is NaN for any of those runs or no run has jobs in the class)."""
    level = Fraction(str(level))
    if not 0 < level <= 1:
        raise ValueError("level must be in (0, 1]")
    recs = np.asarray(recs)
    if recs.ndim != 2:
        raise ValueError("interference_spread: expected recs (runs, C)")
    per = [interference_derived(recs[r]) for r in range(recs.shape[0])]
    reach = (recs["degraded"]["jobs"] + recs["clean"]["jobs"]) > 0
    out = {"replicas": reach.sum(axis=0).astype(np.int64)}
    for name in IF_METRICS:
        cols = [_spread_of(np.array([d[name][c] for r, d in enumerate(per) if reach[r, c]], dtype=np.float64), level)
                for c in range(recs.shape[1])]
        out[name] = {s: np.array([col[s] for col in cols], dtype=np.float64) for s in SPREAD_STATS}
    return out


def interference_columns():
    """names of the flat per-class columns `interference_flat` returns, in order"""
    return list(IF_COUNTS) + list(IF_METRICS)


def interference_flat(d, c):
    """class c of an interference_derived dict as a list of Python values"""
    return [int(d[k][c]) for k in IF_COUNTS] + [float(d[name][c]) for name in IF_METRICS]


def interference_spread_columns():
    return [f"{name}_{s}" for name in IF_METRICS for s in SPREAD_STATS]


def interference_spread_flat(sp, c):
    return [float(sp[name][s][c]) for name in IF_METRICS for s in SPREAD_STATS]


# ---------------------------------------------------------------- time-weighted occupancy
OCC_METRICS = (("gpu_share", "saturated_share", "wait_share", "idle_wait_share", "idle_in_wait_share", "running_mean", "queued_mean")
               + tuple(f"busy_p{q}" for q in QUANTILES) + tuple(f"busy_wait_p{q}" for q in QUANTILES))


def _hist_point(hist, q):
    """the value at fraction q of the multiset that holds hist[b] copies of b (nearest rank); NaN when it is empty"""
    hist = [int(x) for x in hist]
    k = sum(hist)
    if k == 0:
        return math.nan
    r, acc = nearest_rank(q, k), 0
    for b, c in enumerate(hist):
        acc += c
        if acc > r:
            return float(b)
    raise AssertionError("unreachable")


def occupancy_derived(rec, busy_hist, queue_hist, edges):
    """Numbers of one replica's time-weighted occupancy: `rec` OCC_DTYPE, `busy_hist` (2, P) with P > total_gpus (the
    ticks with b busy GPUs over all time, then over the ticks with a queue), `queue_hist` (E + 1,), `edges` the E queue
    edges.  With T = ticks and G = total_gpus:
        gpu_share            busy_sum / (T G)                the time-weighted mean of num_busy_gpus over the GPUs
        saturated_share      H_all[G] / T                    share of time with every GPU busy
        wait_share           wait_ticks / T                  share of time with jobs queued
        idle_wait_share      idle_wait_sum / (T G)           GPU time left idle while jobs waited, over all GPU time
        idle_in_wait_share   idle_wait_sum / (wait_ticks G)  the same over the GPU time while jobs waited
        running_mean, queued_mean                            running_sum / T, queued_sum / T
        busy_p<q>, busy_wait_p<q>                            nearest-rank points of busy GPUs, each tick one value, over
                                                             all time / over the ticks with a queue
        queue_cdf            (E,)                            share of time with queue length <= each edge
    NaN where a denominator is 0."""
    T, G, W = int(rec["ticks"]), int(rec["total_gpus"]), int(rec["wait_ticks"])
    busy_hist, queue_hist = np.asarray(busy_hist), np.asarray(queue_hist)
    if busy_hist.ndim != 2 or busy_hist.shape[0] != 2 or busy_hist.shape[1] <= G or queue_hist.shape != (len(edges) + 1,):
        raise ValueError("occupancy_derived: expected busy_hist (2, > total_gpus) and queue_hist (len(edges) + 1,)")
    out = dict(
        gpu_share=_div(int(rec["busy_sum"]), T * G),
        saturated_share=_div(int(busy_hist[0, G]), T),
        wait_share=_div(W, T),
        idle_wait_share=_div(int(rec["idle_wait_sum"]), T * G),
        idle_in_wait_share=_div(int(rec["idle_wait_sum"]), W * G),
        running_mean=_div(int(rec["running_sum"]), T),
        queued_mean=_div(int(rec["queued_sum"]), T),
    )
    for q in QUANTILES:
        out[f"busy_p{q}"] = _hist_point(busy_hist[0, :G + 1], Fraction(q, 100))
        out[f"busy_wait_p{q}"] = _hist_point(busy_hist[1, :G + 1], Fraction(q, 100))
    cum = np.cumsum(queue_hist.astype(np.int64))[:len(edges)]
    out["queue_cdf"] = cum / T if T else np.full(len(edges), math.nan)
    return out


def occupancy_spread(recs, busy_hists, queue_hists, edges, level=0.95):
    """Spread across replicas (records (replicas,), busy_hists (replicas, 2, P), queue_hists (replicas, E + 1)) of every
    OCC_METRICS entry and of the queue CDF at each edge: {metric: {mean, std, lo, hi}, "queue_cdf": {mean, std, lo, hi:
    float arrays (E,)}}, with spread's rules (NaN throughout where a replica's value is NaN)."""
    level = Fraction(str(level))
    if not 0 < level <= 1:
        raise ValueError("level must be in (0, 1]")
    per = [occupancy_derived(recs[r], busy_hists[r], queue_hists[r], edges) for r in range(len(recs))]
    out = {m: _spread_of(np.array([d[m] for d in per], dtype=np.float64), level) for m in OCC_METRICS}
    cdf = np.stack([d["queue_cdf"] for d in per]) if per else np.zeros((0, len(edges)))
    cols = [_spread_of(cdf[:, e], level) for e in range(len(edges))]
    out["queue_cdf"] = {s: np.array([c[s] for c in cols], dtype=np.float64) for s in SPREAD_STATS}
    return out


def occupancy_columns():
    """names of the flat columns `occupancy_flat` returns, in order"""
    return ["rows", "ticks", "busy_sum", "running_sum", "queued_sum", "wait_ticks", "idle_wait_sum", "running_max", "queued_max",
            "total_gpus"] + list(OCC_METRICS)


def occupancy_flat(rec, d):
    """one OCC_DTYPE record and its occupancy_derived dict as a list of Python values"""
    return [int(rec[k]) for k in occupancy_columns()[:10]] + [float(d[m]) for m in OCC_METRICS]


def occupancy_spread_columns():
    return [f"{m}_{s}" for m in OCC_METRICS for s in SPREAD_STATS]


def occupancy_spread_flat(sp):
    return [float(sp[m][s]) for m in OCC_METRICS for s in SPREAD_STATS]


# ---------------------------------------------------------------- paired comparisons of two configurations
PAIR_POINTS =("p0", "p1", "p5", "p10", "p50_lo", "p50", "p90", "p95", "p99", "p100")
PAIR_STATS = ("d_mean", "d_std", "lt_share", "eq_share", "gt_share") + tuple(f"d_{p}" for p in PAIR_POINTS)
PAIR_METRICS = tuple(f"{m}_{s}" for m in JOBDIST_QUANTITIES for s in PAIR_STATS)
PAIR_COUNTS = ("jobs", "only_a", "only_b")


def _jpair_numbers(rec):
    """the PAIR_METRICS of one JPAIR_DTYPE record as a dict of floats (NaN without jobs; std NaN below two jobs).  The
    mean is the exact sum over the job count rounded once, the sample variance (n * sumsq - sum^2) / (n * (n - 1))
    exact in Python ints and rounded once.  Points: d_p100 .. d_p50 from q_hi, d_p50_lo .. d_p0 from q_lo."""
    n = int(rec["jobs"])
    out = {}
    for i, m in enumerate(JOBDIST_QUANTITIES):
        s, sq = int(rec["d_sum"][i]), u128(rec["d_sq_lo"][i], rec["d_sq_hi"][i])
        out[m + "_d_mean"] = s / n if n else math.nan
        out[m + "_d_std"] = math.sqrt(float(Fraction(n * sq - s * s, n * (n - 1)))) if n > 1 else math.nan
        for k in ("lt", "eq", "gt"):
            out[f"{m}_{k}_share"] = int(rec[k][i]) / n if n else math.nan
        hi, lo = rec["q_hi"][i].tolist(), rec["q_lo"][i].tolist()
        for p, v in zip(("p50", "p90", "p95", "p99", "p100"), hi):
            out[f"{m}_d_{p}"] = float(v) if n else math.nan
        for p, v in zip(("p50_lo", "p10", "p5", "p1", "p0"), lo):
            out[f"{m}_d_{p}"] = float(v) if n else math.nan
    return out


def pair_derived(recs, hist, edges):
    """Per class of one pair: `recs` JPAIR_DTYPE (C,), `hist` CDF counts of d (C, 3, E + 1), `edges` the E signed edges.
    Returns {"jobs", "only_a", "only_b": int arrays (C,), metric: float array (C,) for every PAIR_METRICS entry,
    "<quantity>_cdf": float array (C, E) = #(d <= edge) / jobs}; NaN for a class without jobs in both runs."""
    recs, hist = np.asarray(recs), np.asarray(hist, dtype=np.int64)
    if recs.ndim != 1 or hist.shape != (len(recs), 3, len(edges) + 1):
        raise ValueError("pair_derived: expected recs (C,) and hist (C, 3, len(edges) + 1)")
    out = {k: recs[k].astype(np.int64) for k in PAIR_COUNTS}
    nums = [_jpair_numbers(rec) for rec in recs]
    for name in PAIR_METRICS:
        out[name] = np.array([d[name] for d in nums], dtype=np.float64)
    jobs = out["jobs"]
    cum = np.cumsum(hist, axis=2)[:, :, :len(edges)]
    with np.errstate(invalid="ignore", divide="ignore"):
        for i, m in enumerate(JOBDIST_QUANTITIES):
            out[m + "_cdf"] = np.where(jobs[:, None] > 0, cum[:, i, :] / np.where(jobs > 0, jobs, 1)[:, None], np.nan)
    return out


def pair_spread(recs, hist, edges, level=0.95):
    """Spread per class across replicas of one pair of configurations: `recs` (replicas, C), `hist` (replicas, C, 3,
    E + 1).  For every class, over the replicas with jobs finished in both runs in it: {"replicas": int array (C,),
    name: {mean, std, lo, hi: float arrays (C,)} for the counts (PAIR_COUNTS) and every PAIR_METRICS entry,
    "<quantity>_cdf": {mean, std, lo, hi: float arrays (C, E)}}, with spread's rules."""
    level = Fraction(str(level))
    if not 0 < level <= 1:
        raise ValueError("level must be in (0, 1]")
    recs, hist = np.asarray(recs), np.asarray(hist)
    if recs.ndim != 2 or hist.shape != recs.shape + (3, len(edges) + 1):
        raise ValueError("pair_spread: expected recs (replicas, C) and hist (replicas, C, 3, len(edges) + 1)")
    per = [pair_derived(recs[r], hist[r], edges) for r in range(recs.shape[0])]
    nc, ne = recs.shape[1], len(edges)
    reach = recs["jobs"] > 0
    out = {"replicas": reach.sum(axis=0).astype(np.int64)}
    for name in PAIR_COUNTS + PAIR_METRICS:
        cols = [_spread_of(np.array([d[name][c] for r, d in enumerate(per) if reach[r, c]], dtype=np.float64), level) for c in range(nc)]
        out[name] = {s: np.array([col[s] for col in cols], dtype=np.float64) for s in SPREAD_STATS}
    for m in JOBDIST_QUANTITIES:
        st = {s: np.full((nc, ne), math.nan) for s in SPREAD_STATS}
        cdf = np.stack([d[m + "_cdf"] for d in per]) if per else np.zeros((0, nc, ne))
        for c in range(nc):
            for e in range(ne):
                sp = _spread_of(cdf[reach[:, c], c, e], level)
                for s in SPREAD_STATS:
                    st[s][c, e] = sp[s]
        out[m + "_cdf"] = st
    return out


def pair_columns():
    """names of the flat per-(class, quantity) columns `pair_flat` returns, in order"""
    return list(PAIR_COUNTS) + list(PAIR_STATS)


def pair_flat(d, c, m):
    """class c, quantity m of a pair_derived dict as a list of Python values"""
    return [int(d[k][c]) for k in PAIR_COUNTS] + [float(d[f"{m}_{s}"][c]) for s in PAIR_STATS]


def pair_spread_columns():
    return [f"{name}_{s}" for name in PAIR_COUNTS + PAIR_STATS for s in SPREAD_STATS]


def pair_spread_flat(sp, c, m):
    return [float(sp[name if name in PAIR_COUNTS else f"{m}_{name}"][s][c]) for name in PAIR_COUNTS + PAIR_STATS for s in SPREAD_STATS]


PAIRED_STATS = SPREAD_STATS + ("b_lt_a", "b_eq_a", "b_gt_a")


def paired_spread(records_a, records_b, cluster_a, cluster_b, level=0.95):
    """Replica-level differences of two configurations run on the same replicas (common random numbers): for every
    replica r, b - a of the makespan and of every derived number, each side derived with its own cluster
    ((n_nodes, gpus_per_node, gpu_mem_cap_mib)).  Returns {metric: {mean, std, lo, hi (spread's rules over the
    differences), b_lt_a, b_eq_a, b_gt_a (replicas where b < a, b == a, b > a; a NaN difference counts in none)}}
    for every SPREAD_METRICS entry."""
    level = Fraction(str(level))
    if not 0 < level <= 1:
        raise ValueError("level must be in (0, 1]")
    if len(records_a) != len(records_b):
        raise ValueError("paired_spread: the two configurations need the same replicas")
    diff = {m: [] for m in SPREAD_METRICS}
    for ra, rb in zip(records_a, records_b):
        da, db = derived(ra, *cluster_a), derived(rb, *cluster_b)
        diff["makespan"].append(float(int(rb["makespan"]) - int(ra["makespan"])))
        for m in SPREAD_METRICS[1:]:
            diff[m].append(db[m] - da[m])
    out = {}
    for m, vals in diff.items():
        v = np.asarray(vals, dtype=np.float64)
        sp = _spread_of(v, level)
        sp.update(b_lt_a=int((v < 0).sum()), b_eq_a=int((v == 0).sum()), b_gt_a=int((v > 0).sum()))
        out[m] = sp
    return out


def paired_columns():
    return [f"{m}_{s}" for m in SPREAD_METRICS for s in PAIRED_STATS]


def paired_flat(sp):
    return [sp[m][s] for m in SPREAD_METRICS for s in PAIRED_STATS]

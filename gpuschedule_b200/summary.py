"""Derived numbers of run summaries (capi.SUMMARY_DTYPE records from gs_summarize / gs_horus_summarize): the few
values the reference's notebooks compute from a run's cluster.csv and job.csv.  Post-processing only, like
log_manager: every number follows from the record and the cluster shape.

    gpu_share          busy_gpus_sum / (rows * M * G)                      mean num_busy_gpus over the GPUs
    mem_mean           mean of the avg_gpu_memory_allocated column
    pending_mean       avg_pending_sum / pending_rows                      mean of avg_pending_time where it is non-zero
    wait_mean, turnaround_mean, jct_mean                                   means over the lines of job.csv
    util_mean          util_sum / rows (horus engine; NaN otherwise)       mean of avg_gpu_utilization, NaN as 0
"""
from __future__ import annotations

import math

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

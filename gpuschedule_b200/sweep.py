"""Replica-batched sweeps: what the reference's execute.py runs as N sequential processes
(/root/reference/execute.py:47-55) becomes ONE engine handle with N replicas advanced by the same
kernel launches.  Every replica keeps its own flags, trace, policy and output directory, and
writes the same files a single run_sim.py invocation would."""
from __future__ import annotations

import argparse
import datetime
import math
import operator
import os
import types
from fractions import Fraction

import numpy as np

from . import capi, rngcol, summary, tracegen
from .infrastructure import Infrastructure
from .jobs import JobQueueManager, JobsManager
from .log_manager import LogManager
from .schedule import Scheduler

DEFAULTS = dict(trace_file="tf_job.csv", log_path="batched", scheme="yarn", schedule="fifo", pack=False,
                num_switch=1, num_node_p_switch=32, enable_network_costs=False, enable_migration=False,
                bandwidth=1250, internode_latency=0.015, gpu_memory_capacity=32, num_queue=1, num_buffer=5,
                num_gpu_p_node=8, num_cpu_p_node=128, mem_p_node=512, cluster_spec=None, device=0,
                queue_limit="3600,7200,18000", gittins_delta=3250.0, seed=-1)


def make_flags(**overrides):
    """A flags namespace with run_sim.py's defaults (run_sim.py:19-94) plus overrides."""
    unknown = set(overrides) - set(DEFAULTS)
    if unknown:
        raise ValueError(f"unknown flags: {sorted(unknown)}")
    return types.SimpleNamespace(**{**DEFAULTS, **overrides})


def _is_utilisation_aware(fl):
    return fl.scheme in Scheduler.UTILISATION_AWARE or fl.schedule in Scheduler.UTILISATION_AWARE


def _horus_setup(flag_sets, chunk, rows_cap):
    """per configuration: infrastructure, jobs, and the replica's own random stream (see run_batched_horus)"""
    sims = []
    for fl in flag_sets:
        infra = Infrastructure(fl)
        jm = JobsManager(fl, JobQueueManager(fl, fl.trace_file))
        rs = np.random.RandomState(fl.seed if getattr(fl, "seed", -1) >= 0 else None)
        raw = fl.schedule == "horus+"
        draw = (lambda k, rs=rs: rs.randint(0, 2 ** 32, size=k, dtype=np.uint32)) if raw else (lambda k, rs=rs: rs.standard_normal(k))
        sims.append(dict(fl=fl, infra=infra, jm=jm, raw=raw, draw=draw, stream=draw(chunk), rows_cap=rows_cap))
    return sims


def _horus_run(eng, sims, rows_cap):
    """configure, load and run every replica to the end; a replica that ran out of rows or of samples starts over
    with twice the rows / a longer stream while the others keep their results"""
    for i, sm in enumerate(sims):
        fl = sm["fl"]
        eng.config(i, sm["infra"].gs_cluster(), capi.make_horus_params(fl.scheme, fl.schedule, int(fl.num_buffer), int(fl.num_queue)))
        eng.load_trace(i, sm["jm"].table)
        (eng.load_words if sm["raw"] else eng.load_stream)(i, sm["stream"])
    cap = rows_cap
    while True:
        for sm in sims:
            sm["ran_cap"] = cap                           # the row window this launch really gives every replica
        try:
            eng.run(rows_cap=cap)
            return
        except capi.GsError as e:
            if e.code != capi.GS_ERR_CAPACITY:
                raise
            for i, sm in enumerate(sims):                 # finished replicas keep their results; the short ones start over
                st = eng.stats(i)
                if st.status != capi.GS_ERR_CAPACITY:
                    continue
                if st.ticks < sm["ran_cap"]:              # ran out of samples: continue this replica's stream
                    sm["stream"] = np.concatenate([sm["stream"], sm["draw"](len(sm["stream"]))])
                else:                                     # ran out of rows
                    sm["rows_cap"] = 2 * sm["ran_cap"]
                (eng.load_words if sm["raw"] else eng.load_stream)(i, sm["stream"])
            cap = max(sm["rows_cap"] for sm in sims)


def run_batched_horus(flag_sets, device=0, out_root="log", chunk=1 << 21, rows_cap=1 << 16):
    """The horus / horus+ / gandiva configurations of a sweep as replicas of ONE gs_horus launch.  Every replica
    owns a numpy RandomState (seeded with flags.seed when >= 0, fresh entropy otherwise -- the reference's repeats
    are unseeded) whose stream it consumes exactly like the single-run path does with numpy's global one, so a
    seeded replica writes the same bytes as `run_sim.py --seed s`.  Returns [(output_dir, stats)]."""
    sims = _horus_setup(flag_sets, chunk, rows_cap)
    results = []
    with capi.HorusEngine(device=device, nsims=len(sims)) as eng:
        _horus_run(eng, sims, rows_cap)
        for i, sm in enumerate(sims):
            fl, infra, jm = sm["fl"], sm["infra"], sm["jm"]
            rows, util, flags_arr, recs, order = eng.fetch(i)
            stats = eng.stats(i)
            stamp = datetime.datetime.now().strftime("%Y-%m-%d-%H-%M-%S-%f")
            out_dir = os.path.join(out_root, fl.log_path, f"{stamp}-r{i}")
            os.makedirs(out_dir, exist_ok=True)
            lm = LogManager(out_dir, fl)
            lm.init(infra)
            cl = infra.gs_cluster()
            m, g = cl.num_switch * cl.num_node_p_switch, cl.num_gpu_p_node
            lm.write_cluster_rows(rows, rngcol.sampled_utilization_text(util, flags_arr), m * g * cl.gpu_mem_cap_mib)
            lm.write_horus_job_rows(jm.table, recs, order)
            results.append((out_dir, stats))
    return results


def _plain_setup(flag_sets):
    """per configuration of the fifo / event-driven engine: (flags, infrastructure, jobs, policy)"""
    sims = []
    for fl in flag_sets:
        infra = Infrastructure(fl)
        jm = JobsManager(fl, JobQueueManager(fl, fl.trace_file))
        sched = Scheduler(infra, jm, None)
        sims.append((fl, infra, jm, sched.make_policy(jm.table)))
    return sims


def _plain_load(eng, sims):
    for i, (fl, infra, jm, pol) in enumerate(sims):
        eng.config(i, infra.gs_cluster(), pol)
        eng.load_trace(i, jm.table)


def run_batched(flag_sets, device=0, out_root="log"):
    """Run every configuration of `flag_sets` (list of flags namespaces) as one replica each.
    Returns [(output_dir, stats)] in the order of `flag_sets`; the utilisation-aware configurations go through
    run_batched_horus (their own engine handle), the others through one gs_run batch."""
    aware = [i for i, fl in enumerate(flag_sets) if _is_utilisation_aware(fl)]
    if aware:
        plain = [i for i in range(len(flag_sets)) if i not in set(aware)]
        out = [None] * len(flag_sets)
        for idx, res in zip(aware, run_batched_horus([flag_sets[i] for i in aware], device, out_root)):
            out[idx] = res
        if plain:
            for idx, res in zip(plain, run_batched([flag_sets[i] for i in plain], device, out_root)):
                out[idx] = res
        return out
    sims = _plain_setup(flag_sets)
    results = []
    with capi.Engine(device=device, nsims=len(sims)) as eng:
        _plain_load(eng, sims)
        rows_all = eng.run_all()
        for i, (fl, infra, jm, pol) in enumerate(sims):
            recs, order = eng.fetch_jobs(i)
            span_off, spans = eng.fetch_spans(i)
            stats = eng.stats(i)
            stamp = datetime.datetime.now().strftime("%Y-%m-%d-%H-%M-%S-%f")
            out_dir = os.path.join(out_root, fl.log_path, f"{stamp}-r{i}")
            os.makedirs(out_dir, exist_ok=True)
            lm = LogManager(out_dir, fl)
            lm.init(infra)
            cl = infra.gs_cluster()
            m, g = cl.num_switch * cl.num_node_p_switch, cl.num_gpu_p_node
            if getattr(fl, "seed", -1) >= 0:
                np.random.seed(fl.seed)
            util = rngcol.utilization_text(len(rows_all[i]), m, g, jm.table, recs, span_off, spans)
            lm.write_cluster_rows(rows_all[i], util, m * g * cl.gpu_mem_cap_mib)
            lm.write_job_rows(jm.table, recs, order)
            results.append((out_dir, stats))
    return results


def check_timeline(timeline):
    """(bin width W, bins B) of a timeline argument, or ValueError"""
    try:
        W, B = (int(x) for x in timeline)
    except (TypeError, ValueError):
        raise ValueError("timeline: expected (bin width, bins)") from None
    if not 1 <= W <= 2 ** 40:
        raise ValueError("timeline: the bin width must be in 1..2^40 ticks")
    if not 1 <= B <= capi.TIMELINE_MAX_BINS:
        raise ValueError(f"timeline: the bin count must be in 1..{capi.TIMELINE_MAX_BINS}")
    return W, B


DEFAULT_CDF_EDGES = tuple(2 ** i for i in range(31))


def check_jobdist(jobdist):
    """(class bounds, CDF edges) of a jobdist argument as tuples of ints, or ValueError"""
    try:
        bounds, edges = jobdist
        bounds, edges = [int(x) for x in bounds], [int(x) for x in edges]
    except (TypeError, ValueError):
        raise ValueError("jobdist: expected (class bounds, CDF edges), two sequences of ints") from None
    if len(bounds) > capi.JOBDIST_MAX_CLASSES - 1:
        raise ValueError(f"jobdist: at most {capi.JOBDIST_MAX_CLASSES - 1} class bounds")
    if any(b < 1 or b >= 2 ** 31 for b in bounds) or any(b <= a for a, b in zip(bounds, bounds[1:])):
        raise ValueError("jobdist: the class bounds must be >= 1, int32 and strictly increasing")
    if len(edges) > capi.JOBDIST_MAX_EDGES:
        raise ValueError(f"jobdist: at most {capi.JOBDIST_MAX_EDGES} CDF edges")
    if any(not -2 ** 31 <= e < 2 ** 31 for e in edges) or any(b <= a for a, b in zip(edges, edges[1:])):
        raise ValueError("jobdist: the CDF edges must be int32 and strictly increasing")
    return tuple(bounds), tuple(edges)


DEFAULT_SD_EDGES = tuple(1024 * 2 ** i for i in range(21))      # slowdown 1, 2, 4, ... 2^20 in units of 1/1024


def check_slowdown(slowdown):
    """(key, class bounds, tau, CDF edges, sd CDF edges) of a slowdown argument, the sequences as tuples of ints, or
    ValueError: key one of capi.JKEYS; at most 7 bounds, each >= 1, int64 and strictly increasing; tau >= 1 and int64;
    at most 255 edges and 255 sd edges (units of 1/1024), each list int32 and strictly increasing"""
    try:
        key, bounds, tau, edges, sd_edges = slowdown
        bounds, edges, sd_edges = ([int(x) for x in seq] for seq in (bounds, edges, sd_edges))
        tau = int(tau)
    except (TypeError, ValueError):
        raise ValueError("slowdown: expected (key, class bounds, tau, CDF edges, sd CDF edges)") from None
    if key not in capi.JKEYS:
        raise ValueError(f"slowdown: the key must be one of {', '.join(capi.JKEYS)}")
    if len(bounds) > capi.JOBDIST_MAX_CLASSES - 1:
        raise ValueError(f"slowdown: at most {capi.JOBDIST_MAX_CLASSES - 1} class bounds")
    if any(b < 1 or b >= 2 ** 63 for b in bounds) or any(b <= a for a, b in zip(bounds, bounds[1:])):
        raise ValueError("slowdown: the class bounds must be >= 1, int64 and strictly increasing")
    if not 1 <= tau < 2 ** 63:
        raise ValueError("slowdown: tau must be >= 1 and int64")
    for name, seq, cap in (("CDF edges", edges, capi.JOBDIST_MAX_EDGES), ("sd CDF edges", sd_edges, capi.SLOWDOWN_MAX_EDGES)):
        if len(seq) > cap:
            raise ValueError(f"slowdown: at most {cap} {name}")
        if any(not -2 ** 31 <= e < 2 ** 31 for e in seq) or any(b <= a for a, b in zip(seq, seq[1:])):
            raise ValueError(f"slowdown: the {name} must be int32 and strictly increasing")
    return key, tuple(bounds), tau, tuple(edges), tuple(sd_edges)


def _sd_row(sd):
    """uint32 CDF counts per (replica, class) of a checked slowdown setting"""
    return 3 * (len(sd[3]) + 1) + len(sd[4]) + 1


def check_arrivals(arrivals):
    """(bin width W, bins B, tau) of an arrivals argument, or ValueError: W >= 1 and int64, B in 1..1024, tau >= 1
    and int64"""
    try:
        W, B, tau = (int(x) for x in arrivals)
    except (TypeError, ValueError):
        raise ValueError("arrivals: expected (bin width, bins, tau)") from None
    if not 1 <= W < 2 ** 63:
        raise ValueError("arrivals: the bin width must be >= 1 and int64")
    if not 1 <= B <= capi.ARRIVALS_MAX_BINS:
        raise ValueError(f"arrivals: the bin count must be in 1..{capi.ARRIVALS_MAX_BINS}")
    if not 1 <= tau < 2 ** 63:
        raise ValueError("arrivals: tau must be >= 1 and int64")
    return W, B, tau


DEFAULT_QUEUE_EDGES = (0,) + tuple(2 ** i for i in range(31))      # queue length 0, 1, 2, 4, ... 2^30


def check_occupancy(edges):
    """the queue edges of an occupancy argument as a tuple of ints, or ValueError: at most 255, each >= 0, int32 and
    strictly increasing"""
    try:
        edges = tuple(int(x) for x in edges)
    except (TypeError, ValueError):
        raise ValueError("occupancy: expected a sequence of queue edges") from None
    if len(edges) > capi.OCC_MAX_EDGES:
        raise ValueError(f"occupancy: at most {capi.OCC_MAX_EDGES} queue edges")
    if any(not 0 <= e < 2 ** 31 for e in edges) or any(b <= a for a, b in zip(edges, edges[1:])):
        raise ValueError("occupancy: the queue edges must be >= 0, int32 and strictly increasing")
    return edges


def _occ_pitch(flag_sets):
    """busy histogram entries per row of a sweep's occupancy arrays: the largest M * G of its configurations, plus 1"""
    pitch = 1
    for fl in flag_sets:
        cl = Infrastructure(fl).gs_cluster()
        pitch = max(pitch, cl.num_switch * cl.num_node_p_switch * cl.num_gpu_p_node + 1)
    return pitch


def check_interference(bounds):
    """the class bounds of an interference argument as a tuple of ints, or ValueError (jobdist's rules)"""
    try:
        return check_jobdist((bounds, ()))[0]
    except ValueError as e:
        raise ValueError(f"interference: {str(e).split(': ', 1)[1]}") from None


DEFAULT_DIFF_EDGES = tuple(-2 ** i for i in range(30, -1, -1)) + (0,) + tuple(2 ** i for i in range(31))


def check_compare(compare, flag_sets):
    """(pairs as a tuple of (a, b) configuration indices, class bounds, signed CDF edges) of a compare argument, or
    ValueError: both configurations of a pair must share a trace file and an engine (both utilisation-aware or
    neither)"""
    try:
        pairs, bounds, edges = compare
        pairs = tuple((int(a), int(b)) for a, b in pairs)
    except (TypeError, ValueError):
        raise ValueError("compare: expected (pairs of configuration indices, class bounds, CDF edges)") from None
    try:
        bounds, edges = check_jobdist((bounds, edges))
    except ValueError as e:
        raise ValueError(f"compare: {e}") from None
    for a, b in pairs:
        if not (0 <= a < len(flag_sets) and 0 <= b < len(flag_sets)):
            raise ValueError(f"compare: pair ({a}, {b}) names a configuration that does not exist")
        fa, fb = flag_sets[a], flag_sets[b]
        if fa.trace_file != fb.trace_file:
            raise ValueError(f"compare: configurations {a} and {b} run on different trace files")
        if _is_utilisation_aware(fa) != _is_utilisation_aware(fb):
            raise ValueError(f"compare: {fa.schedule} and {fb.schedule} run on different engines (utilisation-aware and not); "
                             "such pairs are not supported")
    return pairs, bounds, edges


def _compare_in(eng, pairs, members, bounds, edges):
    """gs_compare of the pairs whose configurations are replicas `members` of the handle (in that order)"""
    pos = {c: i for i, c in enumerate(members)}
    return eng.compare([pos[a] for a, _ in pairs], [pos[b] for _, b in pairs], bounds, edges)


def summarize_batched(flag_sets, device=0, chunk=1 << 21, rows_cap=1 << 16, timeline=None, jobdist=None, compare=None, slowdown=None,
                      occupancy=None, interference=None, arrivals=None):
    """One run summary (capi.SUMMARY_DTYPE) per configuration of `flag_sets`, in order, computed on the device: the
    same configurations and random streams as run_batched, but no row or job record is read back and nothing is
    written.  The utilisation-aware configurations go through the gs_horus retry loop of run_batched_horus.
    timeline=(W, B): also bin every replica's rows on the device (gs_set_timeline) and return (summaries,
    TBIN_DTYPE bins of shape (len(flag_sets), B)).
    jobdist=(bounds, edges): also compute every replica's job statistics by job size on the device (gs_set_jobdist)
    and append (JCLASS_DTYPE records (len(flag_sets), C), CDF counts (len(flag_sets), C, 3, E + 1)) to the result.
    compare=(pairs, bounds, edges): also compare every pair (a, b) of configuration indices job by job on the device
    (gs_compare, after the runs) and append (JPAIR_DTYPE records (len(pairs), C), CDF counts of d (len(pairs), C, 3,
    E + 1)) as the last element; both configurations of a pair must share a trace file and an engine.
    slowdown=(key, bounds, tau, edges, sd_edges): also compute every replica's job statistics by key with bounded
    slowdown on the device (gs_set_slowdown) and append (SDCLASS_DTYPE records (len(flag_sets), C), CDF counts
    (len(flag_sets), C, 3 * (E + 1) + Esd + 1)) after the jobdist element (before the compare element).
    occupancy=queue edges: also compute every replica's time-weighted occupancy on the device (gs_set_occupancy) and
    append (OCC_DTYPE records (len(flag_sets),), busy histograms (len(flag_sets), 2, P), queue histograms
    (len(flag_sets), E + 1)) as the last element, P the largest M * G of the configurations plus 1.
    interference=class bounds: also compute the interference statistics of every utilisation-aware replica on the
    device (gs_horus_set_interference) and append IFCLASS_DTYPE records (len(flag_sets), C) as the last element (after
    the occupancy element); the rows of the other configurations are zero.
    arrivals=(W, B, tau): also compute every replica's job statistics by arrival time on the device (gs_set_arrivals)
    and append ABIN_DTYPE records (len(flag_sets), B) as the last element."""
    if arrivals is not None:
        arr = check_arrivals(arrivals)
        arr_recs = np.zeros((len(flag_sets), arr[1]), dtype=capi.ABIN_DTYPE)
    if interference is not None:
        if_bounds = check_interference(interference)
        if_recs = np.zeros((len(flag_sets), len(if_bounds) + 1), dtype=capi.IFCLASS_DTYPE)
    if occupancy is not None:
        occ_edges = check_occupancy(occupancy)
        occ_recs = np.zeros(len(flag_sets), dtype=capi.OCC_DTYPE)
        occ_busy = np.zeros((len(flag_sets), 2, _occ_pitch(flag_sets)), dtype=np.uint64)
        occ_q = np.zeros((len(flag_sets), len(occ_edges) + 1), dtype=np.uint64)
    if slowdown is not None:
        sd = check_slowdown(slowdown)
        sd_nc = len(sd[1]) + 1
        sd_recs = np.zeros((len(flag_sets), sd_nc), dtype=capi.SDCLASS_DTYPE)
        sd_hist = np.zeros((len(flag_sets), sd_nc, _sd_row(sd)), dtype=np.uint32)
    if compare is not None:
        pairs, cmp_bounds, cmp_edges = check_compare(compare, flag_sets)
        cmp_recs = np.zeros((len(pairs), len(cmp_bounds) + 1), dtype=capi.JPAIR_DTYPE)
        cmp_hist = np.zeros((len(pairs), len(cmp_bounds) + 1, 3, len(cmp_edges) + 1), dtype=np.uint32)
    if timeline is not None:
        W, B = check_timeline(timeline)
        bins = np.zeros((len(flag_sets), B), dtype=capi.TBIN_DTYPE)
    if jobdist is not None:
        jd_bounds, jd_edges = check_jobdist(jobdist)
        nc = len(jd_bounds) + 1
        jd_cls = np.zeros((len(flag_sets), nc), dtype=capi.JCLASS_DTYPE)
        jd_hist = np.zeros((len(flag_sets), nc, 3, len(jd_edges) + 1), dtype=np.uint32)
    out = np.zeros(len(flag_sets), dtype=capi.SUMMARY_DTYPE)
    aware = [i for i, fl in enumerate(flag_sets) if _is_utilisation_aware(fl)]
    plain = [i for i in range(len(flag_sets)) if i not in set(aware)]
    if aware:
        sims = _horus_setup([flag_sets[i] for i in aware], chunk, rows_cap)
        with capi.HorusEngine(device=device, nsims=len(sims)) as eng:
            _horus_run(eng, sims, rows_cap)
            if timeline is not None:
                eng.set_timeline(W, B)
            if jobdist is not None:
                eng.set_jobdist(jd_bounds, jd_edges)
            if slowdown is not None:
                eng.set_slowdown(*sd)
            if occupancy is not None:
                eng.set_occupancy(occ_edges)
            if interference is not None:
                eng.set_interference(if_bounds)
            if arrivals is not None:
                eng.set_arrivals(*arr)
            out[aware] = eng.summarize()
            if arrivals is not None:
                arr_recs[aware] = eng.arrivals()
            if interference is not None:
                if_recs[aware] = eng.interference()
            if occupancy is not None:
                occ_recs[aware], ob, occ_q[aware] = eng.occupancy()
                occ_busy[aware, :, :ob.shape[2]] = ob
            if timeline is not None:
                bins[aware] = eng.timeline()
            if jobdist is not None:
                jd_cls[aware], jd_hist[aware] = eng.jobdist()
            if slowdown is not None:
                sd_recs[aware], sd_hist[aware] = eng.slowdown()
            sel = [k for k, (a, _) in enumerate(pairs) if a in set(aware)] if compare is not None else []
            if sel:
                cmp_recs[sel], cmp_hist[sel] = _compare_in(eng, [pairs[k] for k in sel], aware, cmp_bounds, cmp_edges)
    if plain:
        sims = _plain_setup([flag_sets[i] for i in plain])
        with capi.Engine(device=device, nsims=len(sims)) as eng:
            _plain_load(eng, sims)
            if timeline is not None:
                eng.set_timeline(W, B)
            if jobdist is not None:
                eng.set_jobdist(jd_bounds, jd_edges)
            if slowdown is not None:
                eng.set_slowdown(*sd)
            if occupancy is not None:
                eng.set_occupancy(occ_edges)
            if arrivals is not None:
                eng.set_arrivals(*arr)
            out[plain] = eng.run_summarized()
            if arrivals is not None:
                arr_recs[plain] = eng.arrivals()
            if occupancy is not None:
                occ_recs[plain], ob, occ_q[plain] = eng.occupancy()
                occ_busy[plain, :, :ob.shape[2]] = ob
            if timeline is not None:
                bins[plain] = eng.timeline()
            if jobdist is not None:
                jd_cls[plain], jd_hist[plain] = eng.jobdist()
            if slowdown is not None:
                sd_recs[plain], sd_hist[plain] = eng.slowdown()
            sel = [k for k, (a, _) in enumerate(pairs) if a in set(plain)] if compare is not None else []
            if sel:
                cmp_recs[sel], cmp_hist[sel] = _compare_in(eng, [pairs[k] for k in sel], plain, cmp_bounds, cmp_edges)
    res = ((out,) + ((bins,) if timeline is not None else ()) + (((jd_cls, jd_hist),) if jobdist is not None else ())
           + (((sd_recs, sd_hist),) if slowdown is not None else ()) + (((cmp_recs, cmp_hist),) if compare is not None else ())
           + (((occ_recs, occ_busy, occ_q),) if occupancy is not None else ()) + ((if_recs,) if interference is not None else ())
           + ((arr_recs,) if arrivals is not None else ()))
    return res[0] if len(res) == 1 else res


def load_gap_scale(load):
    """offered load L as the gap scale 1/L of gs_boot_params: (gap_num, gap_den)"""
    f = Fraction(1.0 / float(load)).limit_denominator(65535)
    return f.numerator, f.denominator


def check_mix(mix):
    """(class bounds, [multipliers per mix]) of a mix argument as tuples of ints, or ValueError: bounds >= 1, int32 and
    strictly increasing; at least one mix, each with one multiplier in 0..2^32 - 1 per class (len(bounds) + 1)"""
    try:
        bounds, mults = mix
        bounds = tuple(int(b) for b in bounds)
        mults = [tuple(int(x) for x in m) for m in mults]
    except (TypeError, ValueError):
        raise ValueError("mix: expected (class bounds, [multipliers, ...]), sequences of ints") from None
    if any(b < 1 or b >= 2 ** 31 for b in bounds) or any(b <= a for a, b in zip(bounds, bounds[1:])):
        raise ValueError("mix: the class bounds must be >= 1, int32 and strictly increasing")
    if not mults:
        raise ValueError("mix: at least one mix")
    for m in mults:
        if len(m) != len(bounds) + 1:
            raise ValueError(f"mix: every mix needs {len(bounds) + 1} multipliers (one per class), got {len(m)}")
        if any(not 0 <= x <= 2 ** 32 - 1 for x in m):
            raise ValueError("mix: every multiplier must be in 0..2^32 - 1")
    return bounds, mults


def parse_mix_spec(spec, nclasses):
    """the multipliers of a --mix SPEC: nclasses non-negative integers joined by ':', each <= 2^32 - 1, or ValueError"""
    parts = str(spec).split(":")
    if not all(p.isascii() and p.isdigit() for p in parts):
        raise ValueError(f"--mix: {spec!r} is not non-negative integers joined by ':'")
    if len(parts) != nclasses:
        raise ValueError(f"--mix: {spec!r} has {len(parts)} weights, the {nclasses} classes of --mix-classes need {nclasses}")
    m = tuple(int(p) for p in parts)
    if any(x > 2 ** 32 - 1 for x in m):
        raise ValueError(f"--mix: {spec!r} has a weight above 2^32 - 1")
    return m


def check_profiles(profile):
    """[(points, period), ...] of a profile argument as a list of (((tick, factor), ...), period), or ValueError: at
    least one profile; each with 1..64 points whose ticks are ints starting at 0, strictly increasing and below
    2^31 - 1, whose load factors are positive and finite, and a period 0 (aperiodic) or above the last tick and below
    2^31 - 1"""
    try:
        out = []
        for points, period in profile:
            pts = tuple((operator.index(t), float(f)) for t, f in points)
            out.append((pts, operator.index(period)))
    except (TypeError, ValueError):
        raise ValueError("profile: expected [(points, period), ...] with points (tick, load factor) pairs") from None
    if not out:
        raise ValueError("profile: at least one profile")
    for pts, period in out:
        if not 1 <= len(pts) <= tracegen.MAX_SEGMENTS:
            raise ValueError(f"profile: every profile needs 1..{tracegen.MAX_SEGMENTS} points")
        ticks = [t for t, _ in pts]
        if ticks[0] != 0 or any(b <= a for a, b in zip(ticks, ticks[1:])) or ticks[-1] >= 2 ** 31 - 1:
            raise ValueError("profile: the ticks must start at 0, increase strictly and stay below 2^31 - 1")
        if not all(math.isfinite(f) and f > 0 for _, f in pts):
            raise ValueError("profile: every load factor must be positive and finite")
        if period < 0 or period >= 2 ** 31 - 1 or 0 < period <= ticks[-1]:
            raise ValueError("profile: the period must be 0, or above the last tick and below 2^31 - 1")
    return out


def profile_segments(points, period, load):
    """the gs_boot_profiles segments of a profile at offered load L: segment k starts at tick T_k with the gap scale
    load_gap_scale(L * F_k).  Returns (segments as (start, gap_num, gap_den) triples, period), or ValueError for a
    scale whose numerator is 0 or above 2^31 - 1"""
    segs = []
    for t, f in points:
        try:
            num, den = load_gap_scale(float(load) * f)
        except (OverflowError, ZeroDivisionError):
            num = 0
        if not 1 <= num <= 2 ** 31 - 1:
            raise ValueError(f"profile: the load {float(load) * f!r} (load {load} x factor {f}) cannot be expressed as a gap scale")
        segs.append((t, num, den))
    return segs, period


def parse_profile_spec(spec):
    """the (points, period) of a --load-profile SPEC T0:F0,T1:F1,...[@P]: integer ticks from 0, positive finite load
    factors, an optional period; or ValueError"""
    text = str(spec)
    body, at, per = text.partition("@")
    if at and not (per.isascii() and per.isdigit()):
        raise ValueError(f"--load-profile: {spec!r}: the period after '@' must be a non-negative integer")
    points = []
    for part in body.split(","):
        t, colon, f = part.partition(":")
        if not colon or not (t.isascii() and t.isdigit()):
            raise ValueError(f"--load-profile: {spec!r} is not TICK:FACTOR pairs joined by ','")
        try:
            fv = float(f)
        except ValueError:
            raise ValueError(f"--load-profile: {spec!r}: {f!r} is not a load factor") from None
        points.append((int(t), fv))
    try:
        return check_profiles([(points, int(per) if at else 0)])[0]
    except ValueError as e:
        raise ValueError(f"--load-profile: {spec!r}: {e}") from None


def _check_bootstrap_args(flag_sets, replicas, loads, n, block_len=1, mix=None, profile=None):
    if int(replicas) < 1:
        raise ValueError("bootstrap: replicas must be >= 1")
    if not len(loads) or not all(math.isfinite(float(L)) and float(L) > 0 for L in loads):
        raise ValueError("bootstrap: loads must be positive and finite")
    if any(load_gap_scale(L)[0] > 2 ** 31 - 1 for L in loads):
        raise ValueError("bootstrap: a load is too small to be expressed as a gap scale")
    if n is not None and not 0 <= int(n) < 2 ** 31 - 64:
        raise ValueError("bootstrap: n out of range")
    try:
        tracegen.check_block_len(block_len)
    except ValueError as e:
        raise ValueError(f"bootstrap: {e}") from None
    if mix is not None:
        check_mix(mix)
    if profile is not None:
        for points, period in check_profiles(profile):
            for L in loads:
                tracegen.check_profile(*profile_segments(points, period, L))
    aware = [fl.schedule for fl in flag_sets if _is_utilisation_aware(fl)]
    if aware:
        raise ValueError(f"bootstrap: the utilisation-aware engine ({', '.join(sorted(set(aware)))}) has no generated traces")


def summarize_bootstrap(flag_sets, replicas, loads=(1.0,), seed=0, n=None, device=0, timeline=None, jobdist=None, block_len=1,
                        compare=None, mix=None, slowdown=None, occupancy=None, profile=None, arrivals=None):
    """Bootstrap spread of a sweep: every configuration of `flag_sets` runs `replicas` traces drawn on the device from
    its base trace file (gs_boot_traces: jobs and inter-arrival gaps resampled with Philox4x64-10 under key
    (seed, replica index)), at every offered load L of `loads` (the base trace's gaps scaled by 1/L), each replica
    summarised on the device.  A replica has `n` jobs (default: as many as its base trace).  The same replica index
    draws the same jobs and gaps under every configuration and load (common random numbers), so configurations can be
    compared replica by replica.  Returns SUMMARY_DTYPE records of shape (len(flag_sets), len(loads), replicas).

    One engine handle per base trace file.  A gittins replica takes its index table from the base trace (the
    replica's own trace never reaches the host).  Utilisation-aware configurations are an argument error, as are
    replicas < 1 and non-positive loads; every argument is checked before a trace is read or an engine created.
    timeline=(W, B): also bin every replica's rows on the device and return (summaries, TBIN_DTYPE bins of shape
    (len(flag_sets), len(loads), replicas, B)).  jobdist=(bounds, edges): also append (JCLASS_DTYPE records
    (len(flag_sets), len(loads), replicas, C), CDF counts (len(flag_sets), len(loads), replicas, C, 3, E + 1)).
    block_len=L > 1 draws every replica as a stationary block bootstrap with mean block length L
    (gs_boot_traces_blocked): runs of consecutive jobs keep their order and the gaps between them, so a trace's bursts
    survive resampling; the same replica index is coupled across values of L.
    compare=(pairs, bounds, edges): also compare replica (a, L, r) with (b, L, r) job by job on the device for every pair
    (a, b) of configuration indices (both on one trace file) and append (JPAIR_DTYPE records (len(pairs), len(loads),
    replicas, C), CDF counts of d (len(pairs), len(loads), replicas, C, 3, E + 1)) as the last element.
    mix=(bounds, [multipliers, ...]): draw the replicas from other job mixes (gs_boot_traces_mixed): under mix m, a base
    trace row of size class c (the number of bounds <= its num_gpu) is drawn with weight multipliers[m][c] instead of
    uniformly; gaps and arrivals are drawn as without a mix, and the same replica index is coupled across mixes.
    Every returned array gains a mix axis right after the loads axis, (configurations, loads, mixes, replicas, ...),
    and compare pairs (a, L, mix, r) with (b, L, mix, r).  A mix whose weights sum to 0 on a base trace is a
    ValueError, raised before any engine is created.  A gittins replica still takes its index table from the base
    trace: the policy is not told about the shift.  With L > 1, only block starts are drawn from the mix.
    slowdown=(key, bounds, tau, edges, sd_edges): also append (SDCLASS_DTYPE records (..., C), CDF counts (..., C,
    3 * (E + 1) + Esd + 1)) with the replicas' leading axes, after the jobdist element (before the compare element).
    occupancy=queue edges: also append (OCC_DTYPE records (...), busy histograms (..., 2, P), queue histograms
    (..., E + 1)) with the replicas' leading axes as the last element, P as in summarize_batched.
    profile=[(points, period), ...]: give the replicas a time-varying offered load (gs_boot_traces_profiled).  points
    are (tick, load factor) pairs starting at tick 0; at load L, the segment from tick T_k on has the gap scale
    load_gap_scale(L * F_k), and a period P > 0 repeats the profile every P ticks.  Rows, gaps, block starts and mix
    picks are those of the unprofiled replica; only the arrivals move.  Every returned array gains a profile axis
    right after the mix axis (after the loads axis without mixes), and compare pairs (a, L[, mix], profile, r) with
    (b, L[, mix], profile, r).  A replica whose last arrival could reach 2^31 - 1 is a ValueError, raised after the
    traces are read and before any engine is created.
    arrivals=(W, B, tau): also append ABIN_DTYPE records (..., B) with the replicas' leading axes as the last element."""
    if arrivals is not None:
        arr = check_arrivals(arrivals)
    if occupancy is not None:
        occ_edges = check_occupancy(occupancy)
    _check_bootstrap_args(flag_sets, replicas, loads, n, block_len, mix, profile)
    if profile is not None:
        profile = check_profiles(profile)
    if slowdown is not None:
        sd = check_slowdown(slowdown)
        sd_nc, sd_row = len(sd[1]) + 1, _sd_row(sd)
    if mix is not None:
        mix_bounds, mix_mults = check_mix(mix)
    if compare is not None:
        pairs, cmp_bounds, cmp_edges = check_compare(compare, flag_sets)
    block_len = tracegen.check_block_len(block_len)
    if timeline is not None:
        W, B = check_timeline(timeline)
    if jobdist is not None:
        jd_bounds, jd_edges = check_jobdist(jobdist)
        nc, nb = len(jd_bounds) + 1, len(jd_edges) + 1
    R, loads = int(replicas), [float(L) for L in loads]
    M = 1 if mix is None else len(mix_mults)
    NP = 1 if profile is None else len(profile)
    lead = (len(loads),) + (() if mix is None else (M,)) + (() if profile is None else (NP,)) + (R,)   # one configuration's replicas
    per = len(loads) * M * NP * R
    profs = None if profile is None else [profile_segments(pts, period, L) for L in loads for pts, period in profile]
    out = np.zeros((len(flag_sets),) + lead, dtype=capi.SUMMARY_DTYPE)
    if timeline is not None:
        bins = np.zeros((len(flag_sets),) + lead + (B,), dtype=capi.TBIN_DTYPE)
    if jobdist is not None:
        jd_cls = np.zeros((len(flag_sets),) + lead + (nc,), dtype=capi.JCLASS_DTYPE)
        jd_hist = np.zeros((len(flag_sets),) + lead + (nc, 3, nb), dtype=np.uint32)
    if occupancy is not None:
        occ_pitch = _occ_pitch(flag_sets)
        occ_recs = np.zeros((len(flag_sets),) + lead, dtype=capi.OCC_DTYPE)
        occ_busy = np.zeros((len(flag_sets),) + lead + (2, occ_pitch), dtype=np.uint64)
        occ_q = np.zeros((len(flag_sets),) + lead + (len(occ_edges) + 1,), dtype=np.uint64)
    if slowdown is not None:
        sd_recs = np.zeros((len(flag_sets),) + lead + (sd_nc,), dtype=capi.SDCLASS_DTYPE)
        sd_hist = np.zeros((len(flag_sets),) + lead + (sd_nc, sd_row), dtype=np.uint32)
    if arrivals is not None:
        arr_recs = np.zeros((len(flag_sets),) + lead + (arr[1],), dtype=capi.ABIN_DTYPE)
    if compare is not None:
        cmp_nc, cmp_nb = len(cmp_bounds) + 1, len(cmp_edges) + 1
        cmp_recs = np.zeros((len(pairs),) + lead + (cmp_nc,), dtype=capi.JPAIR_DTYPE)
        cmp_hist = np.zeros((len(pairs),) + lead + (cmp_nc, 3, cmp_nb), dtype=np.uint32)
    by_trace = {}
    for c, fl in enumerate(flag_sets):
        by_trace.setdefault(fl.trace_file, []).append(c)
    groups = []                                           # every trace is read and every mix checked before any engine
    for configs in by_trace.values():
        sims = _plain_setup([flag_sets[c] for c in configs])
        base = sims[0][2].table
        weights = None
        if mix is not None:
            weights = np.stack([tracegen.class_weights(base.gpus, mix_bounds, m) for m in mix_mults])
            for m, w in enumerate(weights):
                if not w.any():
                    raise ValueError(f"bootstrap: mix {':'.join(map(str, mix_mults[m]))} gives every job of "
                                     f"{flag_sets[configs[0]].trace_file} weight 0")
        if profs is not None:
            jobs = base.n if n is None else int(n)
            gaps = np.diff(base.arrive_tick.astype(np.int64))
            max_gap = int(gaps.max()) if len(gaps) else 0
            for q, prof in enumerate(profs):
                if tracegen.profile_bound(jobs, max_gap, *prof) >= 2 ** 31 - 1:
                    pts, period = profile[q % NP]
                    raise ValueError(f"bootstrap: under the profile {pts}{f' @ {period}' if period else ''} at load {loads[q // NP]}, "
                                     f"a replica of {jobs} jobs of {flag_sets[configs[0]].trace_file} can arrive at 2^31 - 1 or later")
        groups.append((configs, sims, base, weights))
    for configs, sims, base, weights in groups:
        jobs = base.n if n is None else int(n)
        params = np.zeros(len(configs) * per, dtype=capi.BOOT_PARAMS_DTYPE)
        mix_of = np.zeros(len(params), dtype=np.int32)    # replica (config k, load l, mix m, profile q, r) is
        prof_of = np.zeros(len(params), dtype=np.int32)   # k * per + ((l * M + m) * NP + q) * R + r
        with capi.Engine(device=device, nsims=len(params)) as eng:
            i = 0
            for fl, infra, jm, pol in sims:
                for li, L in enumerate(loads):
                    num, den = load_gap_scale(L) if profile is None else (1, 1)
                    for m in range(M):
                        for q in range(NP):
                            for r in range(R):
                                eng.config(i, infra.gs_cluster(), pol)
                                params[i] = (seed, r, jobs, num, den)
                                mix_of[i] = m
                                prof_of[i] = li * NP + q
                                i += 1
            eng.boot_population(base)
            if weights is not None:
                eng.boot_mixes(weights)
            if profs is not None:
                eng.boot_profiles(profs)
            eng.boot_traces(params, block_len=None if block_len == 1 else block_len, mix=None if weights is None else mix_of,
                            profile=None if profs is None else prof_of)
            if timeline is not None:
                eng.set_timeline(W, B)
            if jobdist is not None:
                eng.set_jobdist(jd_bounds, jd_edges)
            if slowdown is not None:
                eng.set_slowdown(*sd)
            if occupancy is not None:
                eng.set_occupancy(occ_edges)
            if arrivals is not None:
                eng.set_arrivals(*arr)
            recs = eng.run_summarized()
            occ = eng.occupancy() if occupancy is not None else None
            ar = eng.arrivals() if arrivals is not None else None
            tl = eng.timeline() if timeline is not None else None
            jd = eng.jobdist() if jobdist is not None else None
            sdr = eng.slowdown() if slowdown is not None else None
            sel = [k for k, (a, _) in enumerate(pairs) if a in set(configs)] if compare is not None else []
            if sel:
                pos = {c: k for k, c in enumerate(configs)}
                span = np.arange(per)                             # replica (config k, load l[, mix m], r) is k * per + ...
                ia = np.concatenate([pos[pairs[k][0]] * per + span for k in sel])
                ib = np.concatenate([pos[pairs[k][1]] * per + span for k in sel])
                cr, ch = eng.compare(ia, ib, cmp_bounds, cmp_edges)
                cmp_recs[sel] = cr.reshape((len(sel),) + lead + (cmp_nc,))
                cmp_hist[sel] = ch.reshape((len(sel),) + lead + (cmp_nc, 3, cmp_nb))
        for k, c in enumerate(configs):
            part = slice(k * per, (k + 1) * per)
            out[c] = recs[part].reshape(lead)
            if tl is not None:
                bins[c] = tl[part].reshape(lead + (B,))
            if jd is not None:
                jd_cls[c] = jd[0][part].reshape(lead + (nc,))
                jd_hist[c] = jd[1][part].reshape(lead + (nc, 3, nb))
            if sdr is not None:
                sd_recs[c] = sdr[0][part].reshape(lead + (sd_nc,))
                sd_hist[c] = sdr[1][part].reshape(lead + (sd_nc, sd_row))
            if occ is not None:
                ob = occ[1][part]
                occ_recs[c] = occ[0][part].reshape(lead)
                occ_busy[c][..., :ob.shape[2]] = ob.reshape(lead + (2, ob.shape[2]))
                occ_q[c] = occ[2][part].reshape(lead + (len(occ_edges) + 1,))
            if ar is not None:
                arr_recs[c] = ar[part].reshape(lead + (arr[1],))
    res = ((out,) + ((bins,) if timeline is not None else ()) + (((jd_cls, jd_hist),) if jobdist is not None else ())
           + (((sd_recs, sd_hist),) if slowdown is not None else ()) + (((cmp_recs, cmp_hist),) if compare is not None else ())
           + (((occ_recs, occ_busy, occ_q),) if occupancy is not None else ()) + ((arr_recs,) if arrivals is not None else ()))
    return res[0] if len(res) == 1 else res


def _block_col(block_len):
    """the block_len column of the bootstrap files: none for iid replicas (block_len None)"""
    return [] if block_len is None else ["block_len"]


def _block_val(block_len):
    return [] if block_len is None else [block_len]


def _mix_col(mix, profile=None):
    """the mix and profile columns of the bootstrap files: none without job mixes (mix None) and load profiles
    (profile None)"""
    return ([] if mix is None else ["mix"]) + ([] if profile is None else ["profile"])


def _load_lines(loads, block_len, mix, per_load, profile=None):
    """[(values of the load, block_len, mix and profile columns, arrays)] of one configuration's (load[, mix][, profile])
    lines in line order: per_load holds one entry per load, with mixes (their SPEC texts) one per (load, mix), and with
    load profiles (their SPEC texts) one per (load[, mix], profile)"""
    lines = [([L] + _block_val(block_len), x) for L, x in zip(loads, per_load)]
    if mix is not None:
        lines = [(keys + [m], x) for keys, per_mix in lines for m, x in zip(mix, per_mix)]
    if profile is not None:
        lines = [(keys + [p], x) for keys, per_prof in lines for p, x in zip(profile, per_prof)]
    return lines


def write_bootstrap_csv(path, flag_sets, loads, records, block_len=None, mix=None, profile=None):
    """one line per (configuration, load[, mix], replica): replica, load, block_len (with a block length), mix (with
    job mixes: their SPEC texts), the configuration's flags, the summary columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["replica", "load"] + _block_col(block_len) + _mix_col(mix, profile) + SUMMARY_KEYS + summary.columns())
        for fl, per_load in zip(flag_sets, records):
            cl = Infrastructure(fl).gs_cluster()
            shape = (cl.num_switch * cl.num_node_p_switch, cl.num_gpu_p_node, cl.gpu_mem_cap_mib)
            for keys, recs in _load_lines(loads, block_len, mix, per_load, profile):
                for r, rec in enumerate(recs):
                    w.writerow([r] + keys + [fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed] + summary.flat(rec, *shape))


def write_bootstrap_ci_csv(path, flag_sets, loads, records, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration, load[, mix]): the flags, the load, block_len (with a block length), mix (with job
    mixes), the replica count and summary.spread's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["load"] + _block_col(block_len) + _mix_col(mix, profile) + ["replicas", "level"] + summary.spread_columns())
        for fl, per_load in zip(flag_sets, records):
            cl = Infrastructure(fl).gs_cluster()
            shape = (cl.num_switch * cl.num_node_p_switch, cl.num_gpu_p_node, cl.gpu_mem_cap_mib)
            for keys, recs in _load_lines(loads, block_len, mix, per_load, profile):
                w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed] + keys + [len(recs), level]
                           + summary.spread_flat(summary.spread(recs, *shape, level=level)))


SUMMARY_KEYS = ["trace", "scheme", "schedule", "num_buffer", "num_queue", "seed"]


def _bin_bounds(b, W, B):
    """first tick of bin b and the first tick after it ("inf" for the open-ended last bin)"""
    return [b * W, "inf" if b == B - 1 else (b + 1) * W]


def write_timeline_csv(path, flag_sets, bins, width):
    """one line per (configuration, bin): the flags, the bin, its tick range and summary.timeline_derived's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["bin", "bin_start", "bin_end"] + summary.timeline_columns())
        for fl, tb in zip(flag_sets, bins):
            cl = Infrastructure(fl).gs_cluster()
            d = summary.timeline_derived(tb, cl.num_switch * cl.num_node_p_switch, cl.num_gpu_p_node, cl.gpu_mem_cap_mib)
            for b in range(len(tb)):
                w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed, b]
                           + _bin_bounds(b, width, len(tb)) + summary.timeline_flat(d, b))


def write_timeline_ci_csv(path, flag_sets, loads, bins, width, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration, load[, mix], bin): the flags, the load, block_len (with a block length), mix (with
    job mixes), the bin, its tick range, the number of replicas with rows in it and summary.timeline_spread's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["load"] + _block_col(block_len) + _mix_col(mix, profile) + ["bin", "bin_start", "bin_end", "replicas", "level"] + summary.timeline_spread_columns())
        for fl, per_load in zip(flag_sets, bins):
            cl = Infrastructure(fl).gs_cluster()
            shape = (cl.num_switch * cl.num_node_p_switch, cl.num_gpu_p_node, cl.gpu_mem_cap_mib)
            for keys, tb in _load_lines(loads, block_len, mix, per_load, profile):
                sp = summary.timeline_spread(tb, *shape, level=level)
                for b in range(tb.shape[1]):
                    w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed] + keys + [b]
                               + _bin_bounds(b, width, tb.shape[1]) + [int(sp["replicas"][b]), level] + summary.timeline_spread_flat(sp, b))


def write_arrivals_csv(path, flag_sets, recs, arr):
    """one line per (configuration, arrival bin): the flags, the bin, its arrival-tick range, tau and
    summary.arrivals_derived's columns; arr = (W, B, tau)"""
    import csv
    W, _, tau = arr
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["bin", "bin_start", "bin_end", "tau"] + summary.arrivals_columns())
        for fl, rc in zip(flag_sets, recs):
            d = summary.arrivals_derived(rc)
            for b in range(len(rc)):
                w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed, b]
                           + _bin_bounds(b, W, len(rc)) + [tau] + summary.arrivals_flat(d, b))


def write_arrivals_ci_csv(path, flag_sets, loads, recs, arr, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration, load[, block_len][, mix][, profile], arrival bin): the flags, the load columns, the
    bin, its arrival-tick range, tau, the number of replicas with finished jobs in it and summary.arrivals_spread's
    columns"""
    import csv
    W, _, tau = arr
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["load"] + _block_col(block_len) + _mix_col(mix, profile) + ["bin", "bin_start", "bin_end", "tau", "replicas", "level"]
                   + summary.arrivals_spread_columns())
        for fl, per_load in zip(flag_sets, recs):
            for keys, rc in _load_lines(loads, block_len, mix, per_load, profile):
                sp = summary.arrivals_spread(rc, level=level)
                for b in range(rc.shape[1]):
                    w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed] + keys + [b]
                               + _bin_bounds(b, W, rc.shape[1]) + [tau, int(sp["replicas"][b]), level] + summary.arrivals_spread_flat(sp, b))


def _class_range(c, bounds):
    """smallest and largest num_gpu of class c ("inf" for the open-ended last class)"""
    return [bounds[c - 1] if c > 0 else 0, bounds[c] - 1 if c < len(bounds) else "inf"]


def write_jobdist_csv(path, flag_sets, classes, hist, bounds, edges):
    """one line per (configuration, class): the flags, the class, its num_gpu range and summary.jobdist_derived's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["class", "gpus_min", "gpus_max"] + summary.jobdist_columns())
        for fl, cl, hs in zip(flag_sets, classes, hist):
            d = summary.jobdist_derived(cl, hs, edges)
            for c in range(len(cl)):
                w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed, c] + _class_range(c, bounds)
                           + summary.jobdist_flat(d, c))


def write_jobdist_ci_csv(path, flag_sets, loads, classes, hist, bounds, edges, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration, load[, mix], class): the flags, the load, block_len (with a block length), mix
    (with job mixes), the class, its num_gpu range, the number of replicas with jobs in it and
    summary.jobdist_spread's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["load"] + _block_col(block_len) + _mix_col(mix, profile) + ["class", "gpus_min", "gpus_max", "replicas", "level"]
                   + summary.jobdist_spread_columns())
        for fl, per_cl, per_hs in zip(flag_sets, classes, hist):
            for (keys, cl), (_, hs) in zip(_load_lines(loads, block_len, mix, per_cl, profile), _load_lines(loads, block_len, mix, per_hs, profile)):
                sp = summary.jobdist_spread(cl, hs, edges, level=level)
                for c in range(cl.shape[1]):
                    w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed] + keys + [c]
                               + _class_range(c, bounds) + [int(sp["replicas"][c]), level] + summary.jobdist_spread_flat(sp, c))


def write_interference_csv(path, flag_sets, recs, bounds):
    """one line per (utilisation-aware configuration, class): the flags, the class, its num_gpu range and
    summary.interference_derived's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["class", "gpus_min", "gpus_max"] + summary.interference_columns())
        for fl, rc in zip(flag_sets, recs):
            if not _is_utilisation_aware(fl):
                continue
            d = summary.interference_derived(rc)
            for c in range(len(rc)):
                w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed, c] + _class_range(c, bounds)
                           + summary.interference_flat(d, c))


def write_interference_ci_csv(path, flag_sets, repeats, recs, bounds, level=0.95):
    """one line per (utilisation-aware configuration, class) over its `repeats` seeded repeats (flag_sets[i * repeats
    + rep]): the flags with the first repeat's seed, the repeat count, the class, its num_gpu range, the number of
    repeats with jobs in it and summary.interference_spread's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["repeats", "class", "gpus_min", "gpus_max", "replicas", "level"] + summary.interference_spread_columns())
        for i in range(0, len(flag_sets), repeats):
            fl = flag_sets[i]
            if not _is_utilisation_aware(fl):
                continue
            sp = summary.interference_spread(recs[i:i + repeats], level=level)
            for c in range(recs.shape[1]):
                w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed, repeats, c]
                           + _class_range(c, bounds) + [int(sp["replicas"][c]), level] + summary.interference_spread_flat(sp, c))


def write_jobdist_cdf_csv(path, flag_sets, classes, hist, bounds, edges):
    """one line per (configuration, class, quantity, edge): the flags, the class, its num_gpu range, the quantity,
    the edge, the class's jobs and the fraction of them with a value <= the edge"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["class", "gpus_min", "gpus_max", "quantity", "edge", "jobs", "cdf"])
        for fl, cl, hs in zip(flag_sets, classes, hist):
            d = summary.jobdist_derived(cl, hs, edges)
            for c in range(len(cl)):
                for m in summary.JOBDIST_QUANTITIES:
                    for e, edge in enumerate(edges):
                        w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed, c] + _class_range(c, bounds)
                                   + [m, edge, int(d["jobs"][c]), float(d[m + "_cdf"][c, e])])


def write_jobdist_cdf_ci_csv(path, flag_sets, loads, classes, hist, bounds, edges, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration, load[, mix], class, quantity, edge): the flags, the load, block_len (with a block
    length), mix (with job mixes), the class, its num_gpu range, the quantity, the edge, the number of replicas with jobs in the class and
    the spread of the CDF value"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["load"] + _block_col(block_len) + _mix_col(mix, profile) + ["class", "gpus_min", "gpus_max", "quantity", "edge", "replicas", "level"]
                   + [f"cdf_{s}" for s in summary.SPREAD_STATS])
        for fl, per_cl, per_hs in zip(flag_sets, classes, hist):
            for (keys, cl), (_, hs) in zip(_load_lines(loads, block_len, mix, per_cl, profile), _load_lines(loads, block_len, mix, per_hs, profile)):
                sp = summary.jobdist_spread(cl, hs, edges, level=level)
                for c in range(cl.shape[1]):
                    for m in summary.JOBDIST_QUANTITIES:
                        for e, edge in enumerate(edges):
                            w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed]
                                       + keys + [c] + _class_range(c, bounds) + [m, edge, int(sp["replicas"][c]), level]
                                       + [float(sp[m + "_cdf"][s][c, e]) for s in summary.SPREAD_STATS])


def _sd_keys(fl, sd, c, lk=()):
    """the flags, the load columns lk (bootstrap files), the key, the class, its key range and tau of a slowdown line"""
    key, bounds, tau = sd[0], sd[1], sd[2]
    return [fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed] + list(lk) + [key, c] + _class_range(c, bounds) + [tau]


def _sd_edges_of(sd):
    """per SLOWDOWN_QUANTITIES entry, the edges in the quantity's own unit (ticks; slowdown for sd)"""
    return [sd[3]] * 3 + [[e / summary.SLOWDOWN_ONE for e in sd[4]]]


def write_slowdown_csv(path, flag_sets, recs, hist, sd):
    """one line per (configuration, class): the flags, the key, the class, its key range, tau and
    summary.slowdown_derived's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["key", "class", "key_min", "key_max", "tau"] + summary.slowdown_columns())
        for fl, rc, hs in zip(flag_sets, recs, hist):
            d = summary.slowdown_derived(rc, hs, sd[3], sd[4])
            for c in range(len(rc)):
                w.writerow(_sd_keys(fl, sd, c) + summary.slowdown_flat(d, c))


def write_slowdown_ci_csv(path, flag_sets, loads, recs, hist, sd, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration, load[, block_len][, mix], class): the flags, the load, block_len (with a block
    length), mix (with job mixes), the key, the class, its key range, tau, the replicas with jobs in the class and
    summary.slowdown_spread's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["load"] + _block_col(block_len) + _mix_col(mix, profile) + ["key", "class", "key_min", "key_max", "tau"]
                   + ["replicas", "level"] + summary.slowdown_spread_columns())
        for fl, per_rc, per_hs in zip(flag_sets, recs, hist):
            for (keys, rc), (_, hs) in zip(_load_lines(loads, block_len, mix, per_rc, profile), _load_lines(loads, block_len, mix, per_hs, profile)):
                sp = summary.slowdown_spread(rc, hs, sd[3], sd[4], level=level)
                for c in range(rc.shape[1]):
                    w.writerow(_sd_keys(fl, sd, c, keys) + [int(sp["replicas"][c]), level] + summary.slowdown_spread_flat(sp, c))


def write_slowdown_cdf_csv(path, flag_sets, recs, hist, sd, loads=None, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration[, load[, block_len][, mix]], class, quantity, edge): the flags[, the load, block_len,
    mix], the key, the class, its key range, tau, the quantity (wait, turnaround, jct in ticks; sd in units of slowdown),
    the edge in that unit and the fraction of the class's jobs with a value <= the edge (with loads: the replicas with
    jobs in the class and the spread of that fraction)"""
    import csv
    boot = loads is not None
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + (["load"] + _block_col(block_len) + _mix_col(mix, profile) if boot else []) + ["key", "class", "key_min", "key_max", "tau"]
                   + ["quantity", "edge"] + (["replicas", "level"] + [f"cdf_{s}" for s in summary.SPREAD_STATS] if boot else ["jobs", "cdf"]))
        for fl, per_rc, per_hs in zip(flag_sets, recs, hist):
            lines = (zip(_load_lines(loads, block_len, mix, per_rc, profile), _load_lines(loads, block_len, mix, per_hs, profile)) if boot
                     else [(([], per_rc), ([], per_hs))])
            for (lk, rc), (_, hs) in lines:
                d = summary.slowdown_spread(rc, hs, sd[3], sd[4], level=level) if boot else summary.slowdown_derived(rc, hs, sd[3], sd[4])
                for c in range(rc.shape[-1]):
                    for m, edges in zip(summary.SLOWDOWN_QUANTITIES, _sd_edges_of(sd)):
                        for e, edge in enumerate(edges):
                            tail = ([int(d["replicas"][c]), level] + [float(d[m + "_cdf"][s][c, e]) for s in summary.SPREAD_STATS] if boot
                                    else [int(d["jobs"][c]), float(d[m + "_cdf"][c, e])])
                            w.writerow(_sd_keys(fl, sd, c, lk) + [m, edge] + tail)


def write_occupancy_csv(path, flag_sets, recs, busy, queue, edges):
    """one line per configuration: the flags, summary.occupancy_columns() (the record, then occupancy_derived's numbers)"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + summary.occupancy_columns())
        for fl, rc, bh, qh in zip(flag_sets, recs, busy, queue):
            w.writerow(_occ_keys(fl) + summary.occupancy_flat(rc, summary.occupancy_derived(rc, bh, qh, edges)))


def write_occupancy_ci_csv(path, flag_sets, loads, recs, busy, queue, edges, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration, load[, block_len][, mix]): the flags, the load columns, the replica count and
    summary.occupancy_spread's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["load"] + _block_col(block_len) + _mix_col(mix, profile) + ["replicas", "level"] + summary.occupancy_spread_columns())
        for fl, per_rc, per_bh, per_qh in zip(flag_sets, recs, busy, queue):
            lines = zip(_load_lines(loads, block_len, mix, per_rc, profile), _load_lines(loads, block_len, mix, per_bh, profile), _load_lines(loads, block_len, mix, per_qh, profile))
            for (keys, rc), (_, bh), (_, qh) in lines:
                sp = summary.occupancy_spread(rc, bh, qh, edges, level=level)
                w.writerow(_occ_keys(fl) + keys + [len(rc), level] + summary.occupancy_spread_flat(sp))


def _occ_keys(fl):
    return [fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed]


def _cdf_points(hist):
    """(ticks, share of ticks <= each bin) of a histogram; NaN shares when it is empty"""
    t = int(np.asarray(hist, dtype=np.uint64).sum())
    cum = np.cumsum(np.asarray(hist, dtype=np.uint64))
    return t, (cum / t if t else np.full(len(cum), np.nan))


def write_occupancy_cdf_csv(path, flag_sets, recs, busy, queue, edges, loads=None, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration[, load[, block_len][, mix]], quantity, point): quantity busy (every b = 0 .. M * G,
    all time), busy_wait (the same over the ticks with a queue) or queue (at every queue edge), the point and the
    share of time at or below it (with loads: the replicas and the spread of that share)"""
    import csv
    boot = loads is not None
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + (["load"] + _block_col(block_len) + _mix_col(mix, profile) if boot else []) + ["quantity", "point"]
                   + (["replicas", "level"] + [f"cdf_{s}" for s in summary.SPREAD_STATS] if boot else ["ticks", "cdf"]))
        for fl, per_rc, per_bh, per_qh in zip(flag_sets, recs, busy, queue):
            G = Infrastructure(fl).gs_cluster()
            G = G.num_switch * G.num_node_p_switch * G.num_gpu_p_node
            lines = (zip(_load_lines(loads, block_len, mix, per_rc, profile), _load_lines(loads, block_len, mix, per_bh, profile),
                         _load_lines(loads, block_len, mix, per_qh, profile)) if boot else [(([], per_rc), ([], per_bh), ([], per_qh))])
            for (lk, rc), (_, bh), (_, qh) in lines:
                if not boot:
                    rc, bh, qh = rc[None], bh[None], qh[None]
                rows = [("busy", b, bh[:, 0, :G + 1], b) for b in range(G + 1)] + [("busy_wait", b, bh[:, 1, :G + 1], b) for b in range(G + 1)]
                rows += [("queue", e, qh, i) for i, e in enumerate(edges)]
                cdfs = {}
                for m, point, h, i in rows:
                    if m not in cdfs:
                        cdfs[m] = [_cdf_points(x) for x in h]
                    vals = np.array([c[1][i] for c in cdfs[m]], dtype=np.float64)
                    if boot:
                        sp = summary._spread_of(vals, Fraction(str(level)))
                        w.writerow(_occ_keys(fl) + lk + [m, point, len(vals), level] + [float(sp[s]) for s in summary.SPREAD_STATS])
                    else:
                        w.writerow(_occ_keys(fl) + [m, point, cdfs[m][0][0], float(vals[0])])


def _pair_keys(fl, base):
    return [fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed, base.schedule]


def write_paired_csv(path, flag_sets, pairs, recs, hist, bounds, edges):
    """one line per (configuration b of a pair, class, quantity): b's flags, the base configuration's schedule, the
    class, its num_gpu range, the quantity and summary.pair_derived's columns for d = x_b - x_base"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["base_schedule", "class", "gpus_min", "gpus_max", "quantity"] + summary.pair_columns())
        for (a, b), rc, hs in zip(pairs, recs, hist):
            d = summary.pair_derived(rc, hs, edges)
            for c in range(len(rc)):
                for m in summary.JOBDIST_QUANTITIES:
                    w.writerow(_pair_keys(flag_sets[b], flag_sets[a]) + [c] + _class_range(c, bounds) + [m] + summary.pair_flat(d, c, m))


def write_paired_ci_csv(path, flag_sets, pairs, loads, recs, hist, bounds, edges, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration b of a pair, load[, mix], class, quantity): b's flags, the base schedule, the load,
    block_len (with a block length), mix (with job mixes), the class, its num_gpu range, the quantity, the replicas with jobs finished in
    both runs in the class and summary.pair_spread's columns"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["base_schedule", "load"] + _block_col(block_len) + _mix_col(mix, profile) + ["class", "gpus_min", "gpus_max", "quantity", "replicas", "level"]
                   + summary.pair_spread_columns())
        for (a, b), per_rc, per_hs in zip(pairs, recs, hist):
            for (keys, rc), (_, hs) in zip(_load_lines(loads, block_len, mix, per_rc, profile), _load_lines(loads, block_len, mix, per_hs, profile)):
                sp = summary.pair_spread(rc, hs, edges, level=level)
                for c in range(rc.shape[1]):
                    for m in summary.JOBDIST_QUANTITIES:
                        w.writerow(_pair_keys(flag_sets[b], flag_sets[a]) + keys + [c] + _class_range(c, bounds)
                                   + [m, int(sp["replicas"][c]), level] + summary.pair_spread_flat(sp, c, m))


def write_paired_cdf_csv(path, flag_sets, pairs, recs, hist, bounds, edges, loads=None, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration b of a pair[, load[, mix]], class, quantity, edge): b's flags, the base schedule[, the
    load, block_len, mix], the class, its num_gpu range, the quantity, the edge and the fraction of the jobs finished in both
    runs with d <= edge (with loads: the replicas with such jobs and the spread of that fraction)"""
    import csv
    boot = loads is not None
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["base_schedule"] + (["load"] + _block_col(block_len) + _mix_col(mix, profile) if boot else []) + ["class", "gpus_min", "gpus_max", "quantity", "edge"]
                   + (["replicas", "level"] + [f"cdf_{s}" for s in summary.SPREAD_STATS] if boot else ["jobs", "cdf"]))
        for (a, b), per_rc, per_hs in zip(pairs, recs, hist):
            keys = _pair_keys(flag_sets[b], flag_sets[a])
            lines = (zip(_load_lines(loads, block_len, mix, per_rc, profile), _load_lines(loads, block_len, mix, per_hs, profile)) if boot
                     else [(([], per_rc), ([], per_hs))])
            for (lk, rc), (_, hs) in lines:
                d = summary.pair_spread(rc, hs, edges, level=level) if boot else summary.pair_derived(rc, hs, edges)
                for c in range(rc.shape[-1]):
                    for m in summary.JOBDIST_QUANTITIES:
                        for e, edge in enumerate(edges):
                            tail = ([int(d["replicas"][c]), level] + [float(d[m + "_cdf"][s][c, e]) for s in summary.SPREAD_STATS] if boot
                                    else [int(d["jobs"][c]), float(d[m + "_cdf"][c, e])])
                            w.writerow(keys + lk + [c] + _class_range(c, bounds) + [m, edge] + tail)


def write_paired_summary_csv(path, flag_sets, pairs, records, loads=None, level=0.95, block_len=None, mix=None, profile=None):
    """one line per (configuration b of a pair[, load[, mix]]): b's flags, the base schedule[, the load, block_len, mix],
    the replicas and summary.paired_spread's columns: the replica-level differences b - base of the makespan and of
    every derived number (records: (configurations, loads[, mixes], replicas) with loads, else one record per
    configuration)"""
    import csv
    boot = loads is not None

    def shape(fl):
        cl = Infrastructure(fl).gs_cluster()
        return cl.num_switch * cl.num_node_p_switch, cl.num_gpu_p_node, cl.gpu_mem_cap_mib
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + ["base_schedule"] + (["load"] + _block_col(block_len) + _mix_col(mix, profile) if boot else []) + ["replicas", "level"]
                   + summary.paired_columns())
        for a, b in pairs:
            sa, sb = shape(flag_sets[a]), shape(flag_sets[b])
            per = (zip(_load_lines(loads, block_len, mix, records[a], profile), _load_lines(loads, block_len, mix, records[b], profile)) if boot
                   else [(([], records[a:a + 1]), ([], records[b:b + 1]))])
            for (lk, ra), (_, rb) in per:
                sp = summary.paired_spread(ra, rb, sa, sb, level=level)
                w.writerow(_pair_keys(flag_sets[b], flag_sets[a]) + lk + [len(ra), level]
                           + summary.paired_flat(sp))


def write_summary_csv(path, flag_sets, records):
    """one line per configuration: its flags (SUMMARY_KEYS), the summary fields and the derived numbers (summary.py)"""
    import csv
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(SUMMARY_KEYS + summary.columns())
        for fl, rec in zip(flag_sets, records):
            cl = Infrastructure(fl).gs_cluster()
            w.writerow([fl.trace_file, fl.scheme, fl.schedule, fl.num_buffer, fl.num_queue, fl.seed]
                       + summary.flat(rec, cl.num_switch * cl.num_node_p_switch, cl.num_gpu_p_node, cl.gpu_mem_cap_mib))


def main(argv=None):
    ap = argparse.ArgumentParser(description="run a sweep of simulator configurations as one batched GPU launch")
    ap.add_argument("--trace", nargs="+", required=True, help="trace CSV file(s)")
    ap.add_argument("--schedule", nargs="+", default=["fifo"])
    ap.add_argument("--scheme", default=None, help="placement scheme; default: the schedule's own (yarn for fifo / sjf / dlas / gittins)")
    ap.add_argument("--num_buffer", type=int, default=5)
    ap.add_argument("--num_switch", type=int, default=4)
    ap.add_argument("--num_node_p_switch", type=int, default=32)
    ap.add_argument("--num_queue", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=1)
    ap.add_argument("--seed", type=int, default=-1)
    ap.add_argument("--summary", default=None, metavar="FILE",
                    help="write one CSV line of run summary per configuration to FILE instead of the per-run logs")
    ap.add_argument("--bootstrap", type=int, default=None, metavar="R",
                    help="run R bootstrap replicas of every configuration, drawn on the GPU from its trace (needs --summary; "
                         "the Philox key is (--seed, or 0 when it is negative, replica index))")
    ap.add_argument("--load", type=float, nargs="+", default=None, metavar="L",
                    help="with --bootstrap: offered loads, the trace's inter-arrival gaps scaled by 1/L (default 1)")
    ap.add_argument("--jobs", type=int, default=None, metavar="N", help="with --bootstrap: jobs per replica (default: the trace's)")
    ap.add_argument("--block-len", type=int, default=None, metavar="L",
                    help="with --bootstrap: draw block bootstrap replicas with mean block length L (1..2^32 - 1), which keep runs "
                         "of consecutive jobs and their gaps together; every output file gets a block_len column after load")
    ap.add_argument("--mix", nargs="+", default=None, metavar="SPEC",
                    help="with --bootstrap and --mix-classes: draw the replicas from each job mix SPEC, k + 1 non-negative integer "
                         "weights joined by ':' (one per class of --mix-classes, each <= 2^32 - 1): a job of class c is drawn "
                         "with weight SPEC[c] instead of uniformly; every output file gets a mix column after load (after "
                         "block_len with --block-len)")
    ap.add_argument("--mix-classes", type=int, nargs="+", default=None, metavar="B",
                    help="with --mix: class bounds B1 < ... < Bk of the mixes (a job's class is the number of bounds <= its num_gpu)")
    ap.add_argument("--load-profile", nargs="+", default=None, metavar="SPEC",
                    help="with --bootstrap: give the replicas each time-varying offered load SPEC, T0:F0,T1:F1,...[@P]: from tick "
                         "Tk on the load is Fk times --load (integer ticks from 0, strictly increasing; positive load factors), "
                         "repeating every P ticks when @P is given.  Example: 0:1,20000:3,22000:1 is a 3x surge for 2000 ticks.  "
                         "Every output file gets a profile column after mix (after load / block_len without --mix)")
    ap.add_argument("--summary-ci", default=None, metavar="FILE",
                    help="with --bootstrap: one CSV line per (configuration, load) with the mean, std and 95%% interval across replicas")
    ap.add_argument("--timeline", default=None, metavar="FILE",
                    help="with --summary: also bin every run's rows by delta on the GPU and write one CSV line per (configuration, bin) "
                         "to FILE; with --bootstrap one line per (configuration, load, bin) with the spread across replicas")
    ap.add_argument("--bin-width", type=int, default=None, metavar="W", help="with --timeline: ticks of delta per bin")
    ap.add_argument("--bins", type=int, default=None, metavar="B",
                    help=f"with --timeline: bins (1..{capi.TIMELINE_MAX_BINS}, default 128); the last one is open-ended")
    ap.add_argument("--jobdist", default=None, metavar="FILE",
                    help="with --summary: also compute job statistics by job size (num_gpu classes) on the GPU and write one CSV "
                         "line per (configuration, class) to FILE; with --bootstrap one line per (configuration, load, class) "
                         "with the spread across replicas")
    ap.add_argument("--gpu-classes", type=int, nargs="+", default=None, metavar="B",
                    help="with --jobdist: class bounds B1 < ... < Bk (a job's class is the number of bounds <= its num_gpu; "
                         f"at most {capi.JOBDIST_MAX_CLASSES - 1}); default: one class")
    ap.add_argument("--cdf-edges", type=int, nargs="+", default=None, metavar="E",
                    help=f"with --jobdist: CDF edges in ticks (strictly increasing, at most {capi.JOBDIST_MAX_EDGES}; default 1 2 4 ... 2^30)")
    ap.add_argument("--jobdist-cdf", default=None, metavar="FILE",
                    help="with --jobdist: one CSV line per (configuration[, load], class, quantity, edge) with the CDF value or its spread")
    ap.add_argument("--compare", default=None, metavar="BASE",
                    help="with --summary: pair every other --schedule with BASE (one of the --schedule values) on the same trace and "
                         "repeat (with --bootstrap: the same load and replica) and compare them job by job on the GPU")
    ap.add_argument("--paired", default=None, metavar="FILE",
                    help="with --compare: one CSV line per (configuration, class, quantity) with the per-job differences "
                         "d = x - x_BASE of wait / turnaround / jct; with --bootstrap one line per (configuration, load, class, "
                         "quantity) with their spread across replicas.  Classes: --gpu-classes")
    ap.add_argument("--paired-cdf", default=None, metavar="FILE", help="with --paired: the CDF of d at the --diff-edges")
    ap.add_argument("--diff-edges", type=int, nargs="+", default=None, metavar="E",
                    help=f"with --compare: signed CDF edges of d in ticks (strictly increasing, at most {capi.JOBDIST_MAX_EDGES}; "
                         "default -2^30 ... -2 -1 0 1 2 ... 2^30)")
    ap.add_argument("--paired-summary", default=None, metavar="FILE",
                    help="with --compare: one CSV line per configuration (with --bootstrap: per configuration and load) with the "
                         "replica-level differences from BASE of the makespan and of every derived number")
    ap.add_argument("--slowdown", default=None, metavar="FILE",
                    help="with --summary: also compute job statistics by --job-key classes with bounded slowdown on the GPU and "
                         "write one CSV line per (configuration, class) to FILE; with --bootstrap one line per (configuration, "
                         "load, class) with the spread across replicas")
    ap.add_argument("--job-key", choices=tuple(capi.JKEYS), default=None,
                    help="with --slowdown: the class key, num_gpu, the run length jct or gpus * jct (default length)")
    ap.add_argument("--key-classes", type=int, nargs="+", default=None, metavar="B",
                    help="with --slowdown: class bounds B1 < ... < Bk (a job's class is the number of bounds <= its key; at most "
                         f"{capi.JOBDIST_MAX_CLASSES - 1}); default: one class")
    ap.add_argument("--slowdown-bound", type=int, default=None, metavar="TAU",
                    help="with --slowdown: bounded slowdown turnaround / max(jct, TAU), TAU >= 1 in ticks (default 1: plain slowdown)")
    ap.add_argument("--slowdown-cdf", default=None, metavar="FILE",
                    help="with --slowdown: one CSV line per (configuration[, load], class, quantity, edge) with the CDF value or its "
                         "spread; wait / turnaround / jct at --cdf-edges, slowdown at --sd-edges")
    ap.add_argument("--sd-edges", type=int, nargs="+", default=None, metavar="E",
                    help=f"with --slowdown: CDF edges of the slowdown in units of 1/1024 (strictly increasing, at most "
                         f"{capi.SLOWDOWN_MAX_EDGES}; default 1024 * 2^i for i = 0 ... 20)")
    ap.add_argument("--occupancy", default=None, metavar="FILE",
                    help="with --summary: also compute each run's time-weighted occupancy on the GPU (busy GPUs, queue length and "
                         "GPUs left idle while jobs wait, every row weighed by the ticks it stands for) and write one CSV line per "
                         "configuration to FILE; with --bootstrap one line per (configuration, load) with the spread across replicas")
    ap.add_argument("--queue-edges", type=int, nargs="+", default=None, metavar="E",
                    help=f"with --occupancy: queue-length CDF edges (>= 0, strictly increasing, at most {capi.OCC_MAX_EDGES}; "
                         "default 0 and 2^i for i = 0 ... 30)")
    ap.add_argument("--occupancy-cdf", default=None, metavar="FILE",
                    help="with --occupancy: one CSV line per (configuration[, load], quantity, point): the time share with at most "
                         "b busy GPUs for every b, over all time and over the time with jobs queued, and with a queue length at "
                         "most each queue edge")
    ap.add_argument("--interference", default=None, metavar="FILE",
                    help="with --summary: also compute the interference statistics of the utilisation-aware configurations "
                         "(horus, horus+, gandiva) on the GPU -- the jobs co-location slowed (actual > original duration), their "
                         "jct, the actual durations, the GPU time lost -- and write one CSV line per (configuration, seed, class) "
                         "to FILE.  Classes: --gpu-classes")
    ap.add_argument("--interference-ci", default=None, metavar="FILE",
                    help="with --interference and --repeats R >= 2: one CSV line per (configuration, class) with the spread of "
                         "the interference numbers over the R seeded repeats")
    ap.add_argument("--arrivals", default=None, metavar="FILE",
                    help="with --summary and --arrival-width: also compute job statistics by arrival time on the GPU -- wait, "
                         "turnaround, jct and bounded slowdown of the jobs that arrived in each bin of --arrival-width ticks -- "
                         "and write one CSV line per (configuration, bin) to FILE; with --bootstrap one line per (configuration, "
                         "load, bin) with the spread across the replicas with finished jobs in the bin")
    ap.add_argument("--arrival-width", type=int, default=None, metavar="W",
                    help="with --arrivals: arrival ticks per bin (the ticks of --bin-width, so both may share W)")
    ap.add_argument("--arrival-bins", type=int, default=None, metavar="B",
                    help=f"with --arrivals: bins (1..{capi.ARRIVALS_MAX_BINS}, default 128); the last one is open-ended")
    ap.add_argument("--arrival-bound", type=int, default=None, metavar="TAU",
                    help="with --arrivals: bounded slowdown turnaround / max(jct, TAU), TAU >= 1 in ticks (default 1: plain slowdown)")
    a = ap.parse_args(argv)
    arrivals = None
    if a.arrivals is not None:
        if not a.summary:
            ap.error("--arrivals needs --summary FILE")
        if a.arrival_width is None:
            ap.error("--arrivals needs --arrival-width W")
        try:
            arrivals = check_arrivals((a.arrival_width, 128 if a.arrival_bins is None else a.arrival_bins,
                                       1 if a.arrival_bound is None else a.arrival_bound))
        except ValueError as e:
            ap.error(str(e))
    elif a.arrival_width is not None or a.arrival_bins is not None or a.arrival_bound is not None:
        ap.error("--arrival-width, --arrival-bins and --arrival-bound need --arrivals FILE")
    interference = None
    if a.interference is not None:
        if not a.summary:
            ap.error("--interference needs --summary FILE")
        try:
            interference = check_interference(a.gpu_classes or ())
        except ValueError as e:
            ap.error(str(e))
    if a.interference_ci is not None and (a.interference is None or a.repeats < 2):
        ap.error("--interference-ci needs --interference FILE and --repeats R >= 2")
    occupancy = None
    if a.occupancy is not None:
        if not a.summary:
            ap.error("--occupancy needs --summary FILE")
        try:
            occupancy = check_occupancy(DEFAULT_QUEUE_EDGES if a.queue_edges is None else a.queue_edges)
        except ValueError as e:
            ap.error(str(e))
    elif a.queue_edges is not None or a.occupancy_cdf is not None:
        ap.error("--queue-edges and --occupancy-cdf need --occupancy FILE")
    slowdown = None
    if a.slowdown is not None:
        if not a.summary:
            ap.error("--slowdown needs --summary FILE")
        try:
            slowdown = check_slowdown(("length" if a.job_key is None else a.job_key, a.key_classes or (),
                                       1 if a.slowdown_bound is None else a.slowdown_bound,
                                       DEFAULT_CDF_EDGES if a.cdf_edges is None else a.cdf_edges,
                                       DEFAULT_SD_EDGES if a.sd_edges is None else a.sd_edges))
        except ValueError as e:
            ap.error(str(e))
    elif (a.job_key is not None or a.key_classes is not None or a.slowdown_bound is not None or a.slowdown_cdf is not None
          or a.sd_edges is not None):
        ap.error("--job-key, --key-classes, --slowdown-bound, --slowdown-cdf and --sd-edges need --slowdown FILE")
    jobdist = None
    if a.jobdist is not None:
        if not a.summary:
            ap.error("--jobdist needs --summary FILE")
        try:
            jobdist = check_jobdist((a.gpu_classes or (), DEFAULT_CDF_EDGES if a.cdf_edges is None else a.cdf_edges))
        except ValueError as e:
            ap.error(str(e))
    elif ((a.cdf_edges is not None and a.slowdown is None) or a.jobdist_cdf is not None
          or (a.gpu_classes is not None and a.paired is None and a.interference is None)):
        ap.error("--gpu-classes, --cdf-edges and --jobdist-cdf need --jobdist FILE (--gpu-classes: or --paired FILE or "
                 "--interference FILE; --cdf-edges: or --slowdown FILE)")
    if a.compare is None:
        if a.paired is not None or a.paired_cdf is not None or a.diff_edges is not None or a.paired_summary is not None:
            ap.error("--paired, --paired-cdf, --diff-edges and --paired-summary need --compare BASE")
    else:
        if not a.summary:
            ap.error("--compare needs --summary FILE")
        if a.schedule.count(a.compare) != 1:
            ap.error(f"--compare: {a.compare} must be exactly one of the --schedule values")
        if a.paired_cdf is not None and a.paired is None:
            ap.error("--paired-cdf needs --paired FILE")
    timeline = None
    if a.timeline is not None:
        if not a.summary:
            ap.error("--timeline needs --summary FILE")
        if a.bin_width is None:
            ap.error("--timeline needs --bin-width W")
        try:
            timeline = check_timeline((a.bin_width, 128 if a.bins is None else a.bins))
        except ValueError as e:
            ap.error(str(e))
    elif a.bin_width is not None or a.bins is not None:
        ap.error("--bin-width and --bins need --timeline FILE")
    if a.bootstrap is None and (a.load is not None or a.jobs is not None or a.summary_ci is not None or a.block_len is not None):
        ap.error("--load, --jobs, --block-len and --summary-ci need --bootstrap")
    mix = mix_text = None
    if a.mix is not None or a.mix_classes is not None:
        if a.bootstrap is None:
            ap.error("--mix and --mix-classes need --bootstrap")
        if a.mix is None or a.mix_classes is None:
            ap.error("--mix and --mix-classes go together")
        try:
            mix = check_mix((a.mix_classes, [parse_mix_spec(m, len(a.mix_classes) + 1) for m in a.mix]))
        except ValueError as e:
            ap.error(str(e))
        mix_text = list(a.mix)
    profile = profile_text = None
    if a.load_profile is not None:
        if a.bootstrap is None:
            ap.error("--load-profile needs --bootstrap")
        try:
            profile = [parse_profile_spec(p) for p in a.load_profile]
        except ValueError as e:
            ap.error(str(e))
        profile_text = list(a.load_profile)
    if a.bootstrap is not None:
        if not a.summary:
            ap.error("--bootstrap needs --summary FILE")
        if a.repeats != 1:
            ap.error("--bootstrap replaces --repeats")
    sets = []
    for tr in a.trace:
        for sc in a.schedule:
            for rep in range(a.repeats):
                tag = os.path.splitext(os.path.basename(tr))[0]
                scheme = a.scheme or (sc if sc in Scheduler.UTILISATION_AWARE else "yarn")
                sets.append(make_flags(trace_file=tr, schedule=sc, scheme=scheme, num_switch=a.num_switch,
                                       num_node_p_switch=a.num_node_p_switch, num_queue=a.num_queue, num_buffer=a.num_buffer,
                                       log_path=os.path.join(f"batched_{tag}", f"{scheme}_{sc}"),
                                       seed=a.seed if a.seed < 0 else a.seed + rep))
    if interference is not None and not any(_is_utilisation_aware(fl) for fl in sets):
        ap.error("--interference: no configuration runs on the utilisation-aware engine (--schedule horus, horus+ or gandiva)")
    compare = None
    if a.compare is not None:
        pairs, S, R = [], len(a.schedule), a.repeats
        base = a.schedule.index(a.compare)
        for i, fl in enumerate(sets):                     # sets[(trace * S + schedule) * R + repeat]
            if fl.schedule == a.compare:
                continue
            j = (i // (S * R) * S + base) * R + i % R
            if _is_utilisation_aware(fl) != _is_utilisation_aware(sets[j]):
                ap.error(f"--compare: {fl.schedule} and {a.compare} run on different engines; such pairs are not supported")
            pairs.append((j, i))
        try:
            compare = check_compare((pairs, a.gpu_classes or (), DEFAULT_DIFF_EDGES if a.diff_edges is None else a.diff_edges), sets)
        except ValueError as e:
            ap.error(str(e))
    if a.bootstrap is not None:
        loads = a.load or [1.0]
        try:
            _check_bootstrap_args(sets, a.bootstrap, loads, a.jobs, 1 if a.block_len is None else a.block_len, mix, profile)
        except ValueError as e:
            ap.error(str(e))
        bl = a.block_len
        res = summarize_bootstrap(sets, a.bootstrap, loads, seed=max(a.seed, 0), n=a.jobs, timeline=timeline, jobdist=jobdist,
                                  block_len=1 if bl is None else bl, compare=compare, mix=mix, slowdown=slowdown, occupancy=occupancy,
                                  profile=profile, arrivals=arrivals)
        recs, rest = (res, ()) if (timeline is None and jobdist is None and compare is None and slowdown is None
                                   and occupancy is None and arrivals is None) else (res[0], res[1:])
        if arrivals is not None:
            arec = rest[-1]
            rest = rest[:-1]
            write_arrivals_ci_csv(a.arrivals, sets, loads, arec, arrivals, block_len=bl, mix=mix_text, profile=profile_text)
        if occupancy is not None:
            orec, obusy, oq = rest[-1]
            rest = rest[:-1]
            write_occupancy_ci_csv(a.occupancy, sets, loads, orec, obusy, oq, occupancy, block_len=bl, mix=mix_text, profile=profile_text)
            if a.occupancy_cdf:
                write_occupancy_cdf_csv(a.occupancy_cdf, sets, orec, obusy, oq, occupancy, loads=loads, block_len=bl, mix=mix_text, profile=profile_text)
        if compare is not None:
            pairs, cmp_bounds, cmp_edges = compare
            prec, phist = rest[-1]
            rest = rest[:-1]
            if a.paired:
                write_paired_ci_csv(a.paired, sets, pairs, loads, prec, phist, cmp_bounds, cmp_edges, block_len=bl, mix=mix_text, profile=profile_text)
            if a.paired_cdf:
                write_paired_cdf_csv(a.paired_cdf, sets, pairs, prec, phist, cmp_bounds, cmp_edges, loads=loads, block_len=bl, mix=mix_text, profile=profile_text)
            if a.paired_summary:
                write_paired_summary_csv(a.paired_summary, sets, pairs, recs, loads=loads, block_len=bl, mix=mix_text, profile=profile_text)
        if slowdown is not None:
            srec, shist = rest[-1]
            rest = rest[:-1]
            write_slowdown_ci_csv(a.slowdown, sets, loads, srec, shist, slowdown, block_len=bl, mix=mix_text, profile=profile_text)
            if a.slowdown_cdf:
                write_slowdown_cdf_csv(a.slowdown_cdf, sets, srec, shist, slowdown, loads=loads, block_len=bl, mix=mix_text, profile=profile_text)
        if timeline is not None:
            write_timeline_ci_csv(a.timeline, sets, loads, rest[0], timeline[0], block_len=bl, mix=mix_text, profile=profile_text)
        if jobdist is not None:
            cls, hist = rest[-1]
            write_jobdist_ci_csv(a.jobdist, sets, loads, cls, hist, *jobdist, block_len=bl, mix=mix_text, profile=profile_text)
            if a.jobdist_cdf:
                write_jobdist_cdf_ci_csv(a.jobdist_cdf, sets, loads, cls, hist, *jobdist, block_len=bl, mix=mix_text, profile=profile_text)
        write_bootstrap_csv(a.summary, sets, loads, recs, block_len=bl, mix=mix_text, profile=profile_text)
        if a.summary_ci:
            write_bootstrap_ci_csv(a.summary_ci, sets, loads, recs, block_len=bl, mix=mix_text, profile=profile_text)
        print(f"{a.summary}: {len(sets)} configurations x {len(loads)} loads"
              + (f" x {len(mix_text)} mixes" if mix_text else "") + (f" x {len(profile_text)} load profiles" if profile_text else "")
              + f" x {a.bootstrap} replicas")
        return
    if a.summary:
        res = summarize_batched(sets, timeline=timeline, jobdist=jobdist, compare=compare, slowdown=slowdown, occupancy=occupancy,
                                interference=interference, arrivals=arrivals)
        recs, rest = (res, ()) if (timeline is None and jobdist is None and compare is None and slowdown is None
                                   and occupancy is None and interference is None and arrivals is None) else (res[0], res[1:])
        if arrivals is not None:
            arec = rest[-1]
            rest = rest[:-1]
            write_arrivals_csv(a.arrivals, sets, arec, arrivals)
        if interference is not None:
            irec = rest[-1]
            rest = rest[:-1]
            write_interference_csv(a.interference, sets, irec, interference)
            if a.interference_ci:
                write_interference_ci_csv(a.interference_ci, sets, a.repeats, irec, interference)
        if occupancy is not None:
            orec, obusy, oq = rest[-1]
            rest = rest[:-1]
            write_occupancy_csv(a.occupancy, sets, orec, obusy, oq, occupancy)
            if a.occupancy_cdf:
                write_occupancy_cdf_csv(a.occupancy_cdf, sets, orec, obusy, oq, occupancy)
        if compare is not None:
            pairs, cmp_bounds, cmp_edges = compare
            prec, phist = rest[-1]
            rest = rest[:-1]
            if a.paired:
                write_paired_csv(a.paired, sets, pairs, prec, phist, cmp_bounds, cmp_edges)
            if a.paired_cdf:
                write_paired_cdf_csv(a.paired_cdf, sets, pairs, prec, phist, cmp_bounds, cmp_edges)
            if a.paired_summary:
                write_paired_summary_csv(a.paired_summary, sets, pairs, recs)
        if slowdown is not None:
            srec, shist = rest[-1]
            rest = rest[:-1]
            write_slowdown_csv(a.slowdown, sets, srec, shist, slowdown)
            if a.slowdown_cdf:
                write_slowdown_cdf_csv(a.slowdown_cdf, sets, srec, shist, slowdown)
        if timeline is not None:
            write_timeline_csv(a.timeline, sets, rest[0], timeline[0])
        if jobdist is not None:
            cls, hist = rest[-1]
            write_jobdist_csv(a.jobdist, sets, cls, hist, *jobdist)
            if a.jobdist_cdf:
                write_jobdist_cdf_csv(a.jobdist_cdf, sets, cls, hist, *jobdist)
        write_summary_csv(a.summary, sets, recs)
        print(f"{a.summary}: {len(sets)} configurations")
        return
    for out_dir, st in run_batched(sets):
        print(f"{out_dir}: ticks={st.ticks} events={st.events} finished={st.finished}")


if __name__ == "__main__":
    main()

"""ctypes binding of libgsched.so (include/gsched.h).  No torch types cross this
boundary: numpy arrays in, numpy arrays out.  There is no CPU fallback -- if the
shared library or a CUDA device is missing every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .log_manager import CSPAN_DTYPE, EVROW_DTYPE, JOB_DTYPE, JOBRUN_DTYPE, NODEEV_DTYPE, QROW_DTYPE, ROW_DTYPE, SPAN_DTYPE

GS_MAX_QUEUES = 8
SCHEDULES = {"fifo": 0, "sjf": 1, "dlas": 2, "dlas-gpu": 3, "gittins": 4}
SCHEMES = {"yarn": 0, "count": 1}

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgsched.so")     # the in-tree nvcc build; there is no override
CUDA_BUILD_TAG = b"cuda:sm_90a"


class GsCluster(C.Structure):
    _fields_ = [("num_switch", C.c_int32), ("num_node_p_switch", C.c_int32),
                ("num_gpu_p_node", C.c_int32), ("num_cpu_p_node", C.c_int32),
                ("mem_p_node", C.c_int32), ("gpu_mem_cap_mib", C.c_int32),
                ("enable_network_costs", C.c_int32), ("cpu_per_task", C.c_int32),
                ("mem_per_task", C.c_int32), ("reserved0", C.c_int32),
                ("bandwidth", C.c_double), ("internode_latency", C.c_double)]

    @property
    def n_nodes(self):
        return self.num_switch * self.num_node_p_switch


class GsPolicy(C.Structure):
    _fields_ = [("schedule", C.c_int32), ("scheme", C.c_int32), ("num_queue", C.c_int32),
                ("gittins_n", C.c_int32), ("queue_limit", C.c_double * GS_MAX_QUEUES),
                ("gittins_delta", C.c_double), ("gittins_data", C.c_void_p),
                ("gittins_index", C.c_void_p)]


class GsRunStats(C.Structure):
    _fields_ = [("ticks", C.c_int64), ("events", C.c_int64), ("finished", C.c_int64),
                ("started", C.c_int64), ("placement_evals", C.c_int64), ("done", C.c_int32),
                ("status", C.c_int32), ("kernel_ms", C.c_double), ("h2d_ms", C.c_double),
                ("d2h_ms", C.c_double)]


SWITCH_CLUSTER_DTYPE = np.dtype([("num_switch", "<i4"), ("num_node_p_switch", "<i4"), ("num_gpu_p_node", "<i4"), ("reserved", "<i4"),
                                 ("node_off", "<i8"), ("job_off", "<i8"), ("job_cnt", "<i8")])
SWITCH_NODE_DTYPE = np.dtype([("free_gpus", "<i4"), ("free_cpus", "<i4"), ("free_mem", "<f8"), ("net_in", "<f8")])
SWITCH_JOB_DTYPE = np.dtype([("num_gpu", "<i4"), ("n_ps", "<i4"), ("ps_off", "<i8"), ("span_off", "<i8"), ("model_size", "<f8")])
SWITCH_ANS_DTYPE = np.dtype([("n_nodes", "<i4"), ("sw", "<i4")])
SWITCH_SPAN_DTYPE = np.dtype([("node", "<i4"), ("num_gpu", "<i4"), ("num_cpu", "<i4"), ("reserved", "<i4"), ("mem", "<f8"), ("network", "<f8")])
SWITCH_MEM = (5.0, 8.0, 0.2)          # worker_mem, ps_mem, p_w_mem: core/models.py:24-26 of the reference


class GsWindowInfo(C.Structure):
    _fields_ = [("row_first", C.c_int64), ("ticks", C.c_int64), ("ev_rows", C.c_int64), ("q_rows", C.c_int64),
                ("node_events", C.c_int64), ("spans_used", C.c_int64), ("admitted", C.c_int64), ("finished", C.c_int64), ("n", C.c_int64)]


class GsResultLayout(C.Structure):
    _fields_ = [("block_bytes", C.c_int64), ("off_ev", C.c_int64), ("off_q", C.c_int64), ("off_nodeev", C.c_int64), ("off_jobs", C.c_int64),
                ("off_duration", C.c_int64), ("off_finish_order", C.c_int64), ("off_spans", C.c_int64),
                ("cap_ev", C.c_int64), ("cap_q", C.c_int64), ("cap_nodeev", C.c_int64), ("cap_spans", C.c_int64), ("n", C.c_int64), ("span_bytes", C.c_int64)]


# gs_summary (include/gsched.h): one replica's run reduced to what the notebooks compute from cluster.csv / job.csv
SUMMARY_DTYPE = np.dtype([("n", "<i8"), ("rows", "<i8"), ("done", "<i4"), ("status", "<i4"), ("makespan", "<i8"),
                          ("busy_gpus_sum", "<i8"), ("running_sum", "<i8"), ("queued_sum", "<i8"),
                          ("busy_gpus_max", "<i4"), ("running_max", "<i4"), ("queued_max", "<i4"), ("pend_max_max", "<i4"),
                          ("pend_sum_lo", "<u8"), ("pend_sum_hi", "<u8"), ("mem_busy_lo", "<u8"), ("mem_busy_hi", "<u8"),
                          ("pending_rows", "<i8"), ("avg_pending_sum", "<f8"), ("util_sum", "<f8"), ("finished", "<i8"),
                          ("wait_sum", "<i8"), ("turnaround_sum", "<i8"), ("jct_sum", "<i8"), ("preempt_sum", "<i8"),
                          ("gpu_ticks_sum", "<i8"), ("wait_q", "<i4", (5,)), ("turnaround_q", "<i4", (5,)), ("jct_q", "<i4", (5,)),
                          ("reserved", "<i4", (5,))])
assert SUMMARY_DTYPE.itemsize == 256
# gs_tbin (include/gsched.h): one bin of a replica's timeline -- gs_summary's row part restricted to the rows with
# min(delta // W, B - 1) == bin, their smallest / largest delta and the `finished` counter of the bin's last row
TBIN_DTYPE = np.dtype([("rows", "<i8"), ("busy_gpus_sum", "<i8"), ("running_sum", "<i8"), ("queued_sum", "<i8"),
                       ("busy_gpus_max", "<i4"), ("running_max", "<i4"), ("queued_max", "<i4"), ("pend_max_max", "<i4"),
                       ("pend_sum_lo", "<u8"), ("pend_sum_hi", "<u8"), ("mem_busy_lo", "<u8"), ("mem_busy_hi", "<u8"),
                       ("pending_rows", "<i8"), ("avg_pending_sum", "<f8"), ("util_sum", "<f8"),
                       ("delta_min", "<i8"), ("delta_max", "<i8"), ("finished_last", "<i8")])
assert TBIN_DTYPE.itemsize == 128
TIMELINE_MAX_BINS = 1024
# gs_jclass (include/gsched.h): one job-size class of a replica's finished jobs -- gs_summary's job part restricted to
# the class, with exact 128-bit sums of squares; CDF counts come separately as uint32 (replica, class, 3, E + 1)
JCLASS_DTYPE = np.dtype([("jobs", "<i8"), ("wait_sum", "<i8"), ("turnaround_sum", "<i8"), ("jct_sum", "<i8"), ("preempt_sum", "<i8"),
                         ("gpu_ticks_sum", "<i8"), ("wait_sq_lo", "<u8"), ("wait_sq_hi", "<u8"), ("turnaround_sq_lo", "<u8"),
                         ("turnaround_sq_hi", "<u8"), ("jct_sq_lo", "<u8"), ("jct_sq_hi", "<u8"),
                         ("wait_q", "<i4", (5,)), ("turnaround_q", "<i4", (5,)), ("jct_q", "<i4", (5,)), ("reserved", "<i4")])
assert JCLASS_DTYPE.itemsize == 160
JOBDIST_MAX_CLASSES = 8
JOBDIST_MAX_EDGES = 255
# gs_sdclass (include/gsched.h): one class of a replica's finished jobs under a chosen key (GS_JKEY_*) -- its gs_jclass,
# then the bounded slowdown sd (units of 1/1024): exact sum, 128-bit sum of squares, order statistics, minimum, the
# jobs saturated at 2^31 - 1, and the exact 128-bit sum of the keys.  CDF counts come separately as uint32
# (replica, class, 3 * (E + 1) + Esd + 1): the wait, turnaround and jct rows, then the sd row.
SDCLASS_DTYPE = np.dtype([("jc", JCLASS_DTYPE), ("sd_sum", "<i8"), ("sd_sq_lo", "<u8"), ("sd_sq_hi", "<u8"), ("sd_q", "<i4", (5,)),
                          ("sd_min", "<i4"), ("sd_clamped", "<i8"), ("key_sum_lo", "<u8"), ("key_sum_hi", "<u8")])
assert SDCLASS_DTYPE.itemsize == 232
JKEYS = {"gpus": 0, "length": 1, "gpu-time": 2}           # GS_JKEY_GPUS, GS_JKEY_LENGTH, GS_JKEY_GPU_TIME
SLOWDOWN_MAX_EDGES = 255
SLOWDOWN_ONE = 1024                                       # sd units per unit of slowdown
SLOWDOWN_MAX = 2 ** 31 - 1                                # the saturated sd
# gs_abin (include/gsched.h): one arrival bin of a replica -- slowdown's record of the bin's finished jobs with the
# arrival tick as the key, then the jobs of the trace that arrived in the bin, finished or not.
ABIN_DTYPE = np.dtype([("s", SDCLASS_DTYPE), ("arrived", "<i8")])
assert ABIN_DTYPE.itemsize == 240
ARRIVALS_MAX_BINS = 1024
# gs_occ (include/gsched.h): a replica's rows weighed by the ticks they stand for -- rows weighed, T, the sums of
# w * busy_gpus / running / queued, the ticks with a queue, the idle GPU-ticks while jobs wait, the maxima and M * G.
# Histograms come separately as uint64 ticks: busy (replica, [all, waiting], total_gpus + 1), queue (replica, E + 1).
OCC_DTYPE = np.dtype([("rows", "<i8"), ("ticks", "<i8"), ("busy_sum", "<i8"), ("running_sum", "<i8"), ("queued_sum", "<i8"),
                      ("wait_ticks", "<i8"), ("idle_wait_sum", "<i8"), ("running_max", "<i4"), ("queued_max", "<i4"),
                      ("total_gpus", "<i4"), ("reserved", "<i4")])
assert OCC_DTYPE.itemsize == 72
OCC_MAX_EDGES = 255
# gs_ifclass (include/gsched_horus.h): one job-size class of a horus-engine replica's finished jobs split by
# interference -- jobdist's record of the degraded jobs (actual > original) and of the clean ones, then the
# fixed-point (units of 2^-10 tick) actual durations' sum, 128-bit sum of squares and order statistics, the original
# durations' sum, the degraded jobs' excess and lost GPU time, the jobs gandiva preempted, and the saturated jobs.
IFCLASS_DTYPE = np.dtype([("degraded", JCLASS_DTYPE), ("clean", JCLASS_DTYPE), ("actual_sum", "<i8"), ("actual_sq_lo", "<u8"),
                          ("actual_sq_hi", "<u8"), ("original_sum", "<i8"), ("excess_sum", "<i8"), ("lost_gpu_time_lo", "<u8"),
                          ("lost_gpu_time_hi", "<u8"), ("preempted_jobs", "<i8"), ("clamped", "<i8"), ("degraded_jct_mid", "<i4", (2,)),
                          ("actual_q", "<i4", (5,)), ("actual_mid", "<i4", (2,)), ("excess_max", "<i4"), ("preempt_max", "<i4"),
                          ("reserved", "<i4")])
assert IFCLASS_DTYPE.itemsize == 440
OCC_MAX_GPUS = 65535


class GsSlowdownCfg(C.Structure):
    _fields_ = [("key", C.c_int32), ("nclasses", C.c_int32), ("bounds", C.c_int64 * (JOBDIST_MAX_CLASSES - 1)), ("tau", C.c_int64),
                ("nedges", C.c_int32), ("nsd_edges", C.c_int32), ("edges", C.c_void_p), ("sd_edges", C.c_void_p)]


assert C.sizeof(GsSlowdownCfg) == 96
# gs_jpair (include/gsched.h): one job-size class of a pair of replicas on the same trace -- per quantity (wait,
# turnaround, jct) the per-job differences d = x_b - x_a over the jobs finished in both runs: counts by sign, exact
# sums, 128-bit sums of squares, and the nearest-rank points of d ascending (q_hi) and descending (q_lo)
JPAIR_DTYPE = np.dtype([("jobs", "<i8"), ("only_a", "<i8"), ("only_b", "<i8"), ("lt", "<i8", (3,)), ("eq", "<i8", (3,)), ("gt", "<i8", (3,)),
                        ("d_sum", "<i8", (3,)), ("d_sq_lo", "<u8", (3,)), ("d_sq_hi", "<u8", (3,)), ("q_hi", "<i4", (3, 5)), ("q_lo", "<i4", (3, 5))])
assert JPAIR_DTYPE.itemsize == 288

JOBIN_DTYPE = np.dtype([("arrive_tick", "<i4"), ("gpus", "<i4"), ("gpu_per_task", "<i4"), ("ps_count", "<i4"),
                        ("mem_bytes", "<i8"), ("duration", "<f8")])
# gs_boot_params (include/gsched.h): one bootstrap replica -- Philox key (seed, stream), jobs, gap scale gap_num / gap_den
BOOT_PARAMS_DTYPE = np.dtype([("seed", "<u8"), ("stream", "<u8"), ("n", "<i8"), ("gap_num", "<i4"), ("gap_den", "<i4")])
assert BOOT_PARAMS_DTYPE.itemsize == 32
# gs_boot_seg (include/gsched.h): one segment of a load profile -- start tick, gap scale gap_num / gap_den, reserved 0
BOOT_SEG_DTYPE = np.dtype([("start", "<i4"), ("gap_num", "<i4"), ("gap_den", "<i4"), ("reserved", "<i4")])
assert BOOT_SEG_DTYPE.itemsize == 16
BOOT_MAX_SEGMENTS = 64
NODE_DTYPE = np.dtype([("busy_mask", "<u8"), ("cpu_used", "<i4"), ("mem_used", "<i4")])
JOBREQ_DTYPE = np.dtype([("gpus", "<i4"), ("gpu_per_task", "<i4"), ("mem_bytes", "<i8")])


def make_cluster(num_switch=4, num_node_p_switch=32, num_gpu_p_node=8, num_cpu_p_node=128,
                 mem_p_node=512, gpu_memory_capacity=32, enable_network_costs=False,
                 bandwidth=1250, internode_latency=0.015, cpu_per_task=12, mem_per_task=60):
    """gs_cluster from the reference's flag values (infrastructure.py:26-43; job.py:105-106)."""
    return GsCluster(int(num_switch), int(num_node_p_switch), int(num_gpu_p_node),
                     int(num_cpu_p_node), int(mem_p_node), int(gpu_memory_capacity) * 1024,
                     1 if enable_network_costs else 0, int(cpu_per_task), int(mem_per_task), 0,
                     float(bandwidth), float(internode_latency))


def make_policy(schedule="fifo", scheme="yarn", num_queue=1, queue_limit=(), gittins_delta=3250.0,
                gittins_table=None):
    """gs_policy.  `gittins_table` = (data, index) float64 arrays from policies.build_gittins_table;
    the arrays are kept alive on the returned object."""
    p = GsPolicy()
    p.schedule = SCHEDULES[schedule]
    p.scheme = SCHEMES[scheme]
    p.num_queue = int(num_queue)
    for i, v in enumerate(list(queue_limit)[:GS_MAX_QUEUES]):
        p.queue_limit[i] = float(v)
    p.gittins_delta = float(gittins_delta)
    if gittins_table is not None:
        data = np.ascontiguousarray(gittins_table[0], dtype=np.float64)
        idx = np.ascontiguousarray(gittins_table[1], dtype=np.float64)
        p._keep = (data, idx)
        p.gittins_n = len(data)
        p.gittins_data = data.ctypes.data
        p.gittins_index = idx.ctypes.data
    return p


GS_OK, GS_ERR_ARG, GS_ERR_CUDA, GS_ERR_STATE, GS_ERR_CAPACITY, GS_ERR_COMM = 0, -1, -2, -3, -4, -5      # enum gs_status
GS_MAX_RANKS = 8


class GsError(RuntimeError):
    def __init__(self, msg, code=None):
        super().__init__(msg)
        self.code = code            # gs_status of the failing call, when there was one


class PinnedBuffer:
    """Page-locked host memory from gs_host_alloc, viewed as numpy arrays."""

    def __init__(self, nbytes):
        lib = load_library()
        self.ptr = C.c_void_p()
        rc = lib.gs_host_alloc(int(nbytes), C.byref(self.ptr))
        if rc != 0:
            raise GsError(f"gs_host_alloc failed ({rc})")
        self.nbytes = int(nbytes)
        self._lib = lib
        self._raw = (C.c_uint8 * max(self.nbytes, 1)).from_address(self.ptr.value)

    def view(self, dtype, count, offset=0):
        return np.frombuffer(self._raw, dtype=dtype, count=int(count), offset=int(offset))

    def free(self):
        if self.ptr and self.ptr.value:
            self._raw = None
            self._lib.gs_host_free(self.ptr)
            self.ptr = C.c_void_p()


_lib = None


def _ptr(a, ctype):
    return None if a is None else a.ctypes.data_as(C.POINTER(ctype))


def declare_horus_prototypes(lib):
    """ctypes prototypes of include/gsched_horus.h on `lib` (libgsched.so; tests/emu also builds the library's host side
    against a stand-in CUDA runtime and declares the same prototypes on it)"""
    i32p, i64p, f64p = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_double)
    u8p = C.POINTER(C.c_uint8)
    lib.gs_horus_create.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    lib.gs_horus_destroy.argtypes = [C.c_void_p]
    lib.gs_horus_config.argtypes = [C.c_void_p, C.c_int32, C.POINTER(GsCluster), C.POINTER(GsHorusParams)]
    lib.gs_horus_load_trace.argtypes = [C.c_void_p, C.c_int32, C.c_int64, i32p, i32p, i32p, f64p, i64p, f64p, f64p, f64p]
    lib.gs_horus_load_words.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_uint32), C.c_int64]
    lib.gs_horus_load_stream.argtypes = [C.c_void_p, C.c_int32, f64p, C.c_int64]
    lib.gs_horus_run.argtypes = [C.c_void_p, C.c_int64, C.c_int64]
    lib.gs_horus_stats.argtypes = [C.c_void_p, C.c_int32, C.POINTER(GsHorusRunStats)]
    lib.gs_horus_fetch.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, f64p, u8p, C.c_int64, C.c_void_p, i32p, i64p, i64p]
    lib.gs_horus_set_lanes.argtypes = [C.c_void_p, C.c_int]
    lib.gs_horus_set_lanes.restype = C.c_int
    lib.gs_horus_launch_count.argtypes = [C.c_void_p]
    lib.gs_horus_launch_count.restype = C.c_int64
    lib.gs_horus_last_error.argtypes = [C.c_void_p]
    lib.gs_horus_last_error.restype = C.c_char_p
    lib.gs_horus_build_tag.restype = C.c_char_p
    lib.gs_horus_summarize.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, f64p]
    lib.gs_horus_set_timeline.argtypes = [C.c_void_p, C.c_int64, C.c_int32]
    lib.gs_horus_fetch_timeline.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    lib.gs_horus_set_jobdist.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
    lib.gs_horus_fetch_jobdist.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.gs_horus_compare.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                     C.c_void_p, C.c_void_p, f64p]
    lib.gs_horus_compare.restype = C.c_int
    lib.gs_horus_set_slowdown.argtypes = [C.c_void_p, C.c_void_p]
    lib.gs_horus_fetch_slowdown.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.gs_horus_set_slowdown.restype = lib.gs_horus_fetch_slowdown.restype = C.c_int
    lib.gs_horus_set_arrivals.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int64]
    lib.gs_horus_fetch_arrivals.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    lib.gs_horus_set_arrivals.restype = lib.gs_horus_fetch_arrivals.restype = C.c_int
    lib.gs_horus_set_occupancy.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    lib.gs_horus_fetch_occupancy.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    lib.gs_horus_set_occupancy.restype = lib.gs_horus_fetch_occupancy.restype = C.c_int
    lib.gs_horus_set_interference.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    lib.gs_horus_fetch_interference.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    lib.gs_horus_set_interference.restype = lib.gs_horus_fetch_interference.restype = C.c_int
    for name in ("gs_horus_summarize", "gs_horus_set_timeline", "gs_horus_fetch_timeline", "gs_horus_set_jobdist", "gs_horus_fetch_jobdist", "gs_horus_create", "gs_horus_destroy", "gs_horus_config", "gs_horus_load_trace", "gs_horus_load_stream", "gs_horus_load_words",
                 "gs_horus_run", "gs_horus_stats", "gs_horus_fetch"):
        getattr(lib, name).restype = C.c_int
    return lib


def load_library():
    """Load libgsched.so and declare its prototypes; raises if it is not built or is not the CUDA build."""
    global _lib
    if _lib is not None:
        return _lib
    path = LIB_PATH
    if not os.path.exists(path):
        raise GsError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                      "(there is no CPU fallback)")
    lib = C.CDLL(path)
    i32p, i64p, f64p = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_double)
    lib.gs_abi_version.restype = C.c_int
    lib.gs_last_error.restype = C.c_char_p
    lib.gs_last_error.argtypes = [C.c_void_p]
    lib.gs_create.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    lib.gs_destroy.argtypes = [C.c_void_p]
    lib.gs_destroy.restype = None
    lib.gs_config_sim.argtypes = [C.c_void_p, C.c_int, C.POINTER(GsCluster), C.POINTER(GsPolicy)]
    lib.gs_load_trace.argtypes = [C.c_void_p, C.c_int, C.c_int64, i32p, i32p, i32p, f64p, i64p,
                                  f64p, f64p, i32p]
    lib.gs_load_trace_packed.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, f64p, f64p]
    lib.gs_load_trace_packed.restype = C.c_int
    lib.gs_fetch_all.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, i32p, i64p,
                                 C.c_void_p, C.c_int64, i64p]
    lib.gs_fetch_all.restype = C.c_int
    lib.gs_run.argtypes = [C.c_void_p, C.c_int64, C.c_int64]
    lib.gs_stats.argtypes = [C.c_void_p, C.c_int, C.POINTER(GsRunStats)]
    lib.gs_fetch_rows.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p]
    lib.gs_fetch_jobs.argtypes = [C.c_void_p, C.c_int, C.c_void_p, i32p]
    lib.gs_fetch_spans.argtypes = [C.c_void_p, C.c_int, i64p, C.c_void_p, C.c_int64, i64p]
    lib.gs_place_batch.argtypes = [C.c_void_p, C.POINTER(GsCluster), C.c_void_p, C.c_int32,
                                   C.c_void_p, C.c_int64, i32p, i32p, i64p, i32p, f64p]
    lib.gs_net_cost.argtypes = [C.c_void_p, C.POINTER(GsCluster), C.c_int64, i64p, i32p,
                                C.POINTER(C.c_uint8), i32p, f64p, f64p, f64p]
    lib.gs_set_span_budget.argtypes = [C.c_void_p, C.c_double]
    lib.gs_set_span_budget.restype = C.c_int
    lib.gs_reset.argtypes = [C.c_void_p]
    lib.gs_set_engine.argtypes = [C.c_void_p, C.c_int]
    lib.gs_set_engine.restype = C.c_int
    lib.gs_launch_count.argtypes = [C.c_void_p]
    lib.gs_launch_count.restype = C.c_int64
    lib.gs_window.argtypes = [C.c_void_p, C.c_int, C.POINTER(GsWindowInfo)]
    lib.gs_fetch_compact.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gs_sync.argtypes = [C.c_void_p]
    lib.gs_set_async.argtypes = [C.c_void_p, C.c_int]
    lib.gs_set_queue_rows_cap.argtypes = [C.c_void_p, C.c_int64]
    for name in ("gs_window", "gs_fetch_compact", "gs_sync", "gs_set_async", "gs_set_queue_rows_cap"):
        getattr(lib, name).restype = C.c_int
    lib.gs_load_traces_packed.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, i64p]
    lib.gs_result_layout.argtypes = [C.c_void_p, C.c_int, C.POINTER(GsResultLayout)]
    lib.gs_fetch_results.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    lib.gs_summarize.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, f64p]
    lib.gs_boot_population.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    lib.gs_boot_traces.argtypes = [C.c_void_p, C.c_void_p, f64p]
    lib.gs_boot_traces_blocked.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, f64p]
    lib.gs_boot_mixes.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    lib.gs_boot_traces_mixed.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, f64p]
    lib.gs_boot_profiles.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gs_boot_traces_profiled.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, f64p]
    lib.gs_boot_profiles.restype = lib.gs_boot_traces_profiled.restype = C.c_int
    lib.gs_fetch_trace.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.gs_set_timeline.argtypes = [C.c_void_p, C.c_int64, C.c_int32]
    lib.gs_fetch_timeline.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.gs_set_jobdist.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
    lib.gs_fetch_jobdist.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.gs_compare.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                               C.c_void_p, C.c_void_p, f64p]
    lib.gs_compare.restype = C.c_int
    lib.gs_set_slowdown.argtypes = [C.c_void_p, C.c_void_p]
    lib.gs_fetch_slowdown.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.gs_set_slowdown.restype = lib.gs_fetch_slowdown.restype = C.c_int
    lib.gs_set_arrivals.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int64]
    lib.gs_fetch_arrivals.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.gs_set_arrivals.restype = lib.gs_fetch_arrivals.restype = C.c_int
    lib.gs_set_occupancy.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    lib.gs_fetch_occupancy.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    lib.gs_set_occupancy.restype = lib.gs_fetch_occupancy.restype = C.c_int
    for name in ("gs_load_traces_packed", "gs_result_layout", "gs_fetch_results", "gs_summarize", "gs_boot_population", "gs_boot_traces",
                 "gs_boot_traces_blocked", "gs_boot_mixes", "gs_boot_traces_mixed", "gs_fetch_trace", "gs_set_timeline", "gs_fetch_timeline", "gs_set_jobdist", "gs_fetch_jobdist"):
        getattr(lib, name).restype = C.c_int
    lib.gs_switch_yarn.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, f64p, C.c_int64,
                                   C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_int64]
    lib.gs_switch_yarn.restype = C.c_int
    lib.gs_comm_prepare.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    lib.gs_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.gs_comm_stats.argtypes = [C.c_void_p, i64p, f64p]
    lib.gs_comm_set_min_runnable.argtypes = [C.c_void_p, C.c_int]
    for name in ("gs_comm_prepare", "gs_comm_init", "gs_comm_stats", "gs_comm_set_min_runnable"):
        getattr(lib, name).restype = C.c_int
    lib.gs_logcol_open.argtypes = [C.c_int64, C.c_int32, C.c_int64, i64p, i64p, i32p, i32p]
    lib.gs_logcol_open.restype = C.c_void_p
    lib.gs_logcol_close.argtypes = [C.c_void_p]
    lib.gs_logcol_close.restype = None
    lib.gs_logcol_counts.argtypes = [C.c_void_p, i64p]
    lib.gs_logcol_rows.argtypes = [C.c_void_p, C.c_int64, f64p, f64p, f64p, C.c_int64, f64p, i32p]
    lib.gs_logcol_counts.restype = lib.gs_logcol_rows.restype = C.c_int
    lib.gs_host_alloc.argtypes = [C.c_size_t, C.POINTER(C.c_void_p)]
    lib.gs_host_free.argtypes = [C.c_void_p]
    for name in ("gs_reset", "gs_host_alloc", "gs_host_free", "gs_create", "gs_config_sim", "gs_load_trace", "gs_run", "gs_stats",
                 "gs_fetch_rows", "gs_fetch_jobs", "gs_fetch_spans", "gs_place_batch",
                 "gs_net_cost"):
        getattr(lib, name).restype = C.c_int
    if lib.gs_abi_version() != 4:
        raise GsError("libgsched.so ABI version mismatch")
    declare_horus_prototypes(lib)
    lib.gs_build_tag.restype = C.c_char_p
    if lib.gs_build_tag() != CUDA_BUILD_TAG or lib.gs_horus_build_tag() != CUDA_BUILD_TAG:
        raise GsError(f"{path} is not the nvcc sm_90a build (there is no CPU path)")
    _lib = lib
    return lib


def warm_device_async(device=0):
    """Start creating the CUDA context of `device` on a helper thread (the driver call releases the GIL), so that a command
    line can parse its trace meanwhile.  Nothing is reported from here: the Engine constructor that follows raises whatever
    is wrong with the device or the library."""
    import threading

    def work():
        try:
            with Engine(device=device, nsims=1):
                pass
        except Exception:                                   # noqa: BLE001 - see the docstring
            pass
    t = threading.Thread(target=work, name="gs-warm-device", daemon=True)
    t.start()
    return t


class LogColumn:
    """Host walk of the sampled cluster.csv column (include/gsched.h gs_logcol_*): holdings in, per-row sums out."""

    def __init__(self, n_rows, width, first, last, key, job):
        self.lib = load_library()
        self.n_rows = int(n_rows)
        self._keep = (first, last, key, job)
        self.h = self.lib.gs_logcol_open(self.n_rows, int(width), len(first), _ptr(first, C.c_int64), _ptr(last, C.c_int64),
                                         _ptr(key, C.c_int32), _ptr(job, C.c_int32))
        if not self.h:
            raise GsError("gs_logcol_open: holdings must be sorted by first row, with device keys inside the cluster")
        self.row = 0

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        if self.h:
            self.lib.gs_logcol_close(self.h)
            self.h = None

    def counts(self):
        out = np.zeros(self.n_rows, dtype=np.int64)
        rc = self.lib.gs_logcol_counts(self.h, _ptr(out, C.c_int64))
        if rc:
            raise GsError("gs_logcol_counts", rc)
        return out

    def rows(self, r_end, loc, scale, z):
        k = int(r_end) - self.row
        acc, nun = np.zeros(k, dtype=np.float64), np.zeros(k, dtype=np.int32)
        z = np.ascontiguousarray(z, dtype=np.float64)
        rc = self.lib.gs_logcol_rows(self.h, int(r_end), _ptr(loc, C.c_double), _ptr(scale, C.c_double), _ptr(z, C.c_double), len(z),
                                     _ptr(acc, C.c_double), _ptr(nun, C.c_int32))
        if rc:
            raise GsError("gs_logcol_rows: the values passed are not the ones these rows consume", rc)
        self.row = int(r_end)
        return acc, nun


class GsHorusParams(C.Structure):
    _fields_ = [("score", C.c_int32), ("schedule", C.c_int32), ("num_buffer", C.c_int32), ("num_queue", C.c_int32),
                ("placement", C.c_int32), ("reserved", C.c_int32)]


class GsHorusRunStats(C.Structure):
    _fields_ = [("ticks", C.c_int64), ("events", C.c_int64), ("draws", C.c_int64), ("finished", C.c_int32),
                ("queued", C.c_int32), ("running", C.c_int32), ("done", C.c_int32), ("status", C.c_int32),
                ("reserved", C.c_int32), ("kernel_ms", C.c_float), ("reserved2", C.c_float)]


HORUS_REC_DTYPE = np.dtype([("start", "<i4"), ("end", "<i4"), ("jct", "<i4"), ("preempt", "<i4"),
                            ("original", "<f8"), ("actual", "<f8")])
# --scheme horus | horus+ | gandiva all select horus_placement, yarn selects ms_yarn_placement
# (core/scheduling/algorithm.py:182-187); WHICH score
# function it uses is decided by the --schedule name, because Scheduler._schedule passes self.schedule down as the
# `scheme` argument that indexes score_fn (schedule.py:47, algorithm.py:9-13,58,196).  With --schedule fifo that
# lookup raises KeyError in the reference, so the combination is rejected here as well.
HORUS_SCHEMES = {"horus": 0, "horus+": 0, "gandiva": 0, "yarn": 1}  # placement routine: horus_placement / ms_yarn_placement
HORUS_SCHEDULES = {"horus": 1, "horus+": 2, "gandiva": 3}          # --schedule (algorithm.py:292-298)
HORUS_SCORE_OF_SCHEDULE = {"horus": 0, "horus+": 0, "gandiva": 1}  # score_fn[schedule] (algorithm.py:9-13)


def make_horus_params(scheme="horus", schedule="horus", num_buffer=5, num_queue=1):
    if scheme not in HORUS_SCHEMES:
        raise NotImplementedError(f"scheme {scheme!r}: the utilisation-aware engine serves the horus, horus+, gandiva and yarn schemes")
    if schedule not in HORUS_SCHEDULES:
        raise NotImplementedError(f"schedule {schedule!r} with scheme {scheme!r}: the reference raises KeyError in "
                                  "score_fn[schedule] (core/scheduling/algorithm.py:58); use horus, horus+ or gandiva")
    return GsHorusParams(HORUS_SCORE_OF_SCHEDULE[schedule], HORUS_SCHEDULES[schedule], int(num_buffer), int(num_queue),
                         HORUS_SCHEMES[scheme], 0)


class HorusEngine:
    """`nsims` independent horus / gandiva simulations on one CUDA device (include/gsched_horus.h)."""

    def __init__(self, device=0, nsims=1):
        self.lib = self._library()
        self.h = C.c_void_p()
        self.nsims = int(nsims)
        self._n = [0] * self.nsims
        rc = self.lib.gs_horus_create(int(device), self.nsims, C.byref(self.h))
        if rc != 0:
            msg = self.lib.gs_horus_last_error(None)
            self.h = C.c_void_p()
            raise GsError(f"gs_horus_create failed ({rc}): {msg.decode() if msg else ''}")

    @staticmethod
    def _library():
        return load_library()       # always the CUDA build (load_library checks the build tag)

    def _check(self, rc, what):
        if rc != 0:
            msg = self.lib.gs_horus_last_error(self.h)
            raise GsError(f"{what} failed ({rc}): {msg.decode() if msg else ''}", rc)

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.lib.gs_horus_destroy(self.h)
            self.h = C.c_void_p()

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def config(self, sim, cluster: GsCluster, params: GsHorusParams):
        self._check(self.lib.gs_horus_config(self.h, sim, C.byref(cluster), C.byref(params)), "gs_horus_config")

    def load_trace(self, sim, table):
        arr = lambda a, dt: np.ascontiguousarray(a, dtype=dt)
        a, g, c = arr(table.arrive_tick, np.int32), arr(table.gpus, np.int32), arr(table.gpu_per_task, np.int32)
        d, m = arr(table.duration, np.float64), arr(table.mem_bytes, np.int64)
        ua, um = arr(table.util_avg, np.float64), arr(table.util_max, np.float64)
        ma = table.extra.get("mem_avg_mib")
        ma = None if ma is None else arr(ma, np.float64)
        self._check(self.lib.gs_horus_load_trace(self.h, sim, table.n, _ptr(a, C.c_int32), _ptr(g, C.c_int32), _ptr(c, C.c_int32),
                                                 _ptr(d, C.c_double), _ptr(m, C.c_int64), _ptr(ua, C.c_double),
                                                 _ptr(um, C.c_double), _ptr(ma, C.c_double)), "gs_horus_load_trace")
        self._n[sim] = table.n

    def set_lanes(self, lanes):
        """simulations per warp: 1 (lane 0 of every warp) or 32; 0 = one per warp, all lanes cooperate in the scoring"""
        self._check(self.lib.gs_horus_set_lanes(self.h, int(lanes)), "gs_horus_set_lanes")

    def load_stream(self, sim, standard_normal):
        g = np.ascontiguousarray(standard_normal, dtype=np.float64)
        self._check(self.lib.gs_horus_load_stream(self.h, sim, _ptr(g, C.c_double), len(g)), "gs_horus_load_stream")

    def load_words(self, sim, mt19937_words):
        """raw generator words (numpy.random.randint(0, 2**32, n, dtype=uint32)); required for horus+"""
        w = np.ascontiguousarray(mt19937_words, dtype=np.uint32)
        self._check(self.lib.gs_horus_load_words(self.h, sim, _ptr(w, C.c_uint32), len(w)), "gs_horus_load_words")

    def run(self, max_ticks=0, rows_cap=1 << 16):
        self._check(self.lib.gs_horus_run(self.h, int(max_ticks), int(rows_cap)), "gs_horus_run")

    def stats(self, sim) -> GsHorusRunStats:
        st = GsHorusRunStats()
        self._check(self.lib.gs_horus_stats(self.h, sim, C.byref(st)), "gs_horus_stats")
        return st

    def fetch(self, sim):
        """(rows, utilisation values, is-array flags, job records, finish order)"""
        from .log_manager import ROW_DTYPE
        st = self.stats(sim)
        n, t = self._n[sim], int(st.ticks)
        rows = np.zeros(max(t, 1), dtype=ROW_DTYPE)
        util = np.zeros(max(t, 1), dtype=np.float64)
        flags = np.zeros(max(t, 1), dtype=np.uint8)
        recs = np.zeros(max(n, 1), dtype=HORUS_REC_DTYPE)
        order = np.zeros(max(n, 1), dtype=np.int32)
        nr, nf = C.c_int64(0), C.c_int64(0)
        self._check(self.lib.gs_horus_fetch(self.h, sim, rows.ctypes.data_as(C.c_void_p), _ptr(util, C.c_double),
                                            _ptr(flags, C.c_uint8), len(rows), recs.ctypes.data_as(C.c_void_p),
                                            _ptr(order, C.c_int32), C.byref(nr), C.byref(nf)), "gs_horus_fetch")
        return rows[:nr.value], util[:nr.value], flags[:nr.value], recs[:n], order[:nf.value]

    def summarize(self, first=0, count=None, with_time=False):
        """SUMMARY_DTYPE records of replicas [first, first+count) over every row they hold (include/gsched_horus.h);
        with_time: (records, kernel milliseconds)"""
        count = self.nsims - first if count is None else int(count)
        out = np.zeros(max(count, 1), dtype=SUMMARY_DTYPE)
        ms = C.c_double(0.0)
        self._check(self.lib.gs_horus_summarize(self.h, int(first), count, out.ctypes.data_as(C.c_void_p), C.byref(ms)),
                    "gs_horus_summarize")
        return (out[:count], ms.value) if with_time else out[:count]

    def set_timeline(self, width, nbins):
        """bin every summarised row by min(delta // width, nbins - 1) on the device; nbins = 0 turns it off
        (include/gsched_horus.h: gs_horus_set_timeline)"""
        self._check(self.lib.gs_horus_set_timeline(self.h, int(width), int(nbins)), "gs_horus_set_timeline")
        self._tl_nbins = int(nbins)

    def timeline(self, first=0, count=None):
        """TBIN_DTYPE bins of replicas [first, first+count) as of the last summarize(): shape (count, nbins)"""
        return _fetch_timeline(self, self.lib.gs_horus_fetch_timeline, "gs_horus_fetch_timeline", first, count)

    def set_jobdist(self, bounds, edges):
        """job statistics by job size, filled by every summarize(): len(bounds) + 1 classes by num_gpu, CDF counts at
        `edges`; bounds=None turns it off (include/gsched_horus.h: gs_horus_set_jobdist)"""
        _set_jobdist(self, self.lib.gs_horus_set_jobdist, "gs_horus_set_jobdist", bounds, edges)

    def jobdist(self, first=0, count=None):
        """(JCLASS_DTYPE records (count, C), uint32 CDF counts (count, C, 3, E + 1)) as of the last summarize()"""
        return _fetch_jobdist(self, self.lib.gs_horus_fetch_jobdist, "gs_horus_fetch_jobdist", first, count)

    def set_slowdown(self, key=None, bounds=(), tau=1, edges=(), sd_edges=()):
        """job statistics by `key` ("gpus", "length" or "gpu-time") with bounded slowdown, filled by every summarize():
        len(bounds) + 1 classes, tau the slowdown's lower bound on the run length, CDF counts at `edges` and `sd_edges`
        (units of 1/1024); key=None turns it off (include/gsched_horus.h: gs_horus_set_slowdown)"""
        _set_slowdown(self, self.lib.gs_horus_set_slowdown, "gs_horus_set_slowdown", key, bounds, tau, edges, sd_edges)

    def slowdown(self, first=0, count=None):
        """(SDCLASS_DTYPE records (count, C), uint32 CDF counts (count, C, 3 * (E + 1) + Esd + 1)) as of the last
        summarize()"""
        return _fetch_slowdown(self, self.lib.gs_horus_fetch_slowdown, "gs_horus_fetch_slowdown", first, count)

    def set_arrivals(self, width, bins, tau=1):
        """job statistics by arrival time, filled by every summarize(): `bins` bins of `width` ticks by
        min(arrival // width, bins - 1), bounded slowdown with lower bound tau; bins = 0 turns it off
        (include/gsched_horus.h: gs_horus_set_arrivals)"""
        _set_arrivals(self, self.lib.gs_horus_set_arrivals, "gs_horus_set_arrivals", width, bins, tau)

    def arrivals(self, first=0, count=None):
        """ABIN_DTYPE records (count, bins) as of the last summarize()"""
        return _fetch_arrivals(self, self.lib.gs_horus_fetch_arrivals, "gs_horus_fetch_arrivals", first, count)

    def set_occupancy(self, queue_edges=None):
        """time-weighted occupancy filled by every summarize(), with queue-length CDF counts at `queue_edges`;
        None turns it off (include/gsched_horus.h: gs_horus_set_occupancy)"""
        _set_occupancy(self, self.lib.gs_horus_set_occupancy, "gs_horus_set_occupancy", queue_edges)

    def occupancy(self, first=0, count=None):
        """(OCC_DTYPE records (count,), uint64 busy histograms (count, 2, max total_gpus + 1): all time, waiting time,
        uint64 queue histograms (count, E + 1)) as of the last summarize()"""
        return _fetch_occupancy(self, self.lib.gs_horus_fetch_occupancy, "gs_horus_fetch_occupancy", first, count)

    def set_interference(self, bounds):
        """interference statistics filled by every summarize(): len(bounds) + 1 classes by num_gpu, each split into
        degraded (actual > original) and clean jobs; bounds=None turns it off (include/gsched_horus.h:
        gs_horus_set_interference)"""
        if bounds is None:
            self._check(self.lib.gs_horus_set_interference(self.h, 0, None), "gs_horus_set_interference")
            self._if_classes = 0
            return
        b = np.asarray(bounds, dtype=np.int64).reshape(-1)
        if b.size and (b.min() < -2 ** 31 or b.max() >= 2 ** 31):
            raise GsError("gs_horus_set_interference: bounds must be int32", GS_ERR_ARG)
        b = np.ascontiguousarray(b, dtype=np.int32)
        self._check(self.lib.gs_horus_set_interference(self.h, len(b) + 1, b.ctypes.data_as(C.c_void_p) if len(b) else None),
                    "gs_horus_set_interference")
        self._if_classes = len(b) + 1

    def interference(self, first=0, count=None):
        """IFCLASS_DTYPE records (count, C) as of the last summarize()"""
        count = self.nsims - first if count is None else int(count)
        nc = getattr(self, "_if_classes", 0)
        out = np.zeros((max(count, 1), max(nc, 1)), dtype=IFCLASS_DTYPE)
        self._check(self.lib.gs_horus_fetch_interference(self.h, int(first), count, out.ctypes.data_as(C.c_void_p)),
                    "gs_horus_fetch_interference")
        return out[:count, :nc]

    def compare(self, a, b, bounds=(), edges=(), with_time=False):
        """paired per-job comparison of replicas b[i] against a[i] on the same trace (include/gsched_horus.h:
        gs_horus_compare): (JPAIR_DTYPE records (P, C), uint32 CDF counts of d (P, C, 3, E + 1)); with_time: and the
        kernel milliseconds"""
        return _compare(self, self.lib.gs_horus_compare, "gs_horus_compare", a, b, bounds, edges, with_time)


def _fetch_timeline(eng, fn, what, first, count):
    count = eng.nsims - first if count is None else int(count)
    b = getattr(eng, "_tl_nbins", 0)
    out = np.zeros((max(count, 1), max(b, 1)), dtype=TBIN_DTYPE)
    eng._check(fn(eng.h, int(first), count, out.ctypes.data_as(C.c_void_p)), what)
    return out[:count, :b]


def _set_jobdist(eng, fn, what, bounds, edges):
    if bounds is None:
        eng._check(fn(eng.h, 0, None, 0, None), what)
        eng._jd_shape = (0, 0)
        return
    b = np.ascontiguousarray(np.asarray(bounds, dtype=np.int64).reshape(-1))
    e = np.ascontiguousarray(np.asarray(edges, dtype=np.int64).reshape(-1))
    if (b.size and (b.min() < -2 ** 31 or b.max() >= 2 ** 31)) or (e.size and (e.min() < -2 ** 31 or e.max() >= 2 ** 31)):
        raise GsError(f"{what}: bounds and edges must be int32", GS_ERR_ARG)
    b, e = b.astype(np.int32), e.astype(np.int32)
    eng._check(fn(eng.h, len(b) + 1, b.ctypes.data_as(C.c_void_p) if len(b) else None, len(e),
                  e.ctypes.data_as(C.c_void_p) if len(e) else None), what)
    eng._jd_shape = (len(b) + 1, len(e))


def _set_arrivals(eng, fn, what, width, bins, tau):
    bins, width, tau = int(bins), int(width), int(tau)
    if not (-2 ** 31 <= bins < 2 ** 31 and -2 ** 63 <= width < 2 ** 63 and -2 ** 63 <= tau < 2 ** 63):
        raise GsError(what + ": bins must be int32, width and tau int64", GS_ERR_ARG)
    eng._check(fn(eng.h, int(width), bins, int(tau)), what)
    eng._arr_bins = bins


def _fetch_arrivals(eng, fn, what, first, count):
    count = eng.nsims - first if count is None else int(count)
    nb = getattr(eng, "_arr_bins", 0)
    out = np.zeros((max(count, 1), max(nb, 1)), dtype=ABIN_DTYPE)
    eng._check(fn(eng.h, int(first), count, out.ctypes.data_as(C.c_void_p)), what)
    return out[:count, :nb]


def slowdown_cfg(key, bounds=(), tau=1, edges=(), sd_edges=()):
    """(GsSlowdownCfg, the arrays it points to) of a setting; GsError(GS_ERR_ARG) for an unknown key or values that do
    not fit the struct's fields (the library checks the rest)"""
    if key not in JKEYS:
        raise GsError(f"slowdown: key must be one of {sorted(JKEYS)}", GS_ERR_ARG)
    b = np.asarray(bounds, dtype=object).reshape(-1)
    e, se = (np.asarray(x, dtype=np.int64).reshape(-1) for x in (edges, sd_edges))
    if len(b) > JOBDIST_MAX_CLASSES - 1 or any(not -2 ** 63 <= int(x) < 2 ** 63 for x in b) or not -2 ** 63 <= int(tau) < 2 ** 63:
        raise GsError(f"slowdown: at most {JOBDIST_MAX_CLASSES - 1} int64 bounds and an int64 tau", GS_ERR_ARG)
    for arr in (e, se):
        if arr.size and (arr.min() < -2 ** 31 or arr.max() >= 2 ** 31):
            raise GsError("slowdown: edges must be int32", GS_ERR_ARG)
    e, se = np.ascontiguousarray(e, dtype=np.int32), np.ascontiguousarray(se, dtype=np.int32)
    cfg = GsSlowdownCfg(JKEYS[key], len(b) + 1)
    for i, x in enumerate(b):
        cfg.bounds[i] = int(x)
    cfg.tau = int(tau)
    cfg.nedges, cfg.nsd_edges = len(e), len(se)
    cfg.edges = e.ctypes.data if len(e) else None
    cfg.sd_edges = se.ctypes.data if len(se) else None
    return cfg, (e, se)


def _set_slowdown(eng, fn, what, key, bounds, tau, edges, sd_edges):
    if key is None:
        eng._check(fn(eng.h, None), what)
        eng._sd_shape = (0, 0)
        return
    cfg, keep = slowdown_cfg(key, bounds, tau, edges, sd_edges)
    eng._check(fn(eng.h, C.byref(cfg)), what)
    del keep
    eng._sd_shape = (cfg.nclasses, 3 * (cfg.nedges + 1) + cfg.nsd_edges + 1)


def _fetch_slowdown(eng, fn, what, first, count):
    count = eng.nsims - first if count is None else int(count)
    nc, row = getattr(eng, "_sd_shape", (0, 0))
    recs = np.zeros((max(count, 1), max(nc, 1)), dtype=SDCLASS_DTYPE)
    hist = np.zeros((max(count, 1), max(nc, 1), max(row, 1)), dtype=np.uint32)
    eng._check(fn(eng.h, int(first), count, recs.ctypes.data_as(C.c_void_p), hist.ctypes.data_as(C.c_void_p)), what)
    return recs[:count, :nc], hist[:count, :nc, :row]


def _set_occupancy(eng, fn, what, queue_edges):
    if queue_edges is None:
        eng._check(fn(eng.h, 0, 0, None), what)
        eng._occ_edges = 0
        return
    e = np.asarray(queue_edges, dtype=np.int64).reshape(-1)
    if e.size and (e.min() < -2 ** 31 or e.max() >= 2 ** 31):
        raise GsError(f"{what}: queue edges must be int32", GS_ERR_ARG)
    e = np.ascontiguousarray(e, dtype=np.int32)
    eng._check(fn(eng.h, 1, len(e), e.ctypes.data_as(C.c_void_p) if len(e) else None), what)
    eng._occ_edges = len(e)


def _fetch_occupancy(eng, fn, what, first, count):
    count = eng.nsims - first if count is None else int(count)
    E = getattr(eng, "_occ_edges", 0)
    recs = np.zeros(max(count, 1), dtype=OCC_DTYPE)
    eng._check(fn(eng.h, int(first), count, recs.ctypes.data_as(C.c_void_p), None, 0, None), what)
    pitch = int(recs["total_gpus"][:count].max()) + 1 if count else 1
    busy = np.zeros((max(count, 1), 2, pitch), dtype=np.uint64)
    queue = np.zeros((max(count, 1), E + 1), dtype=np.uint64)
    eng._check(fn(eng.h, int(first), count, None, busy.ctypes.data_as(C.c_void_p), pitch, queue.ctypes.data_as(C.c_void_p)), what)
    return recs[:count], busy[:count], queue[:count]


def _compare(eng, fn, what, a, b, bounds, edges, with_time):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.int64).reshape(-1))
    b = np.ascontiguousarray(np.asarray(b, dtype=np.int64).reshape(-1))
    if a.shape != b.shape:
        raise GsError(f"{what}: a and b must have the same length", GS_ERR_ARG)
    bd = np.asarray(bounds, dtype=np.int64).reshape(-1)
    ed = np.asarray(edges, dtype=np.int64).reshape(-1)
    for arr in (a, b, bd, ed):
        if arr.size and (arr.min() < -2 ** 31 or arr.max() >= 2 ** 31):
            raise GsError(f"{what}: indices, bounds and edges must be int32", GS_ERR_ARG)
    a, b, bd, ed = (np.ascontiguousarray(x, dtype=np.int32) for x in (a, b, bd, ed))
    P, nc, ne = len(a), len(bd) + 1, len(ed)
    recs = np.zeros((max(P, 1), nc), dtype=JPAIR_DTYPE)
    hist = np.zeros((max(P, 1), nc, 3, ne + 1), dtype=np.uint32)
    vp = lambda x: x.ctypes.data_as(C.c_void_p) if len(x) else None
    ms = C.c_double(0.0)
    eng._check(fn(eng.h, P, vp(a), vp(b), nc, vp(bd), ne, vp(ed), recs.ctypes.data_as(C.c_void_p), hist.ctypes.data_as(C.c_void_p),
                  C.byref(ms)), what)
    return (recs[:P], hist[:P], ms.value) if with_time else (recs[:P], hist[:P])


def _fetch_jobdist(eng, fn, what, first, count):
    count = eng.nsims - first if count is None else int(count)
    nc, ne = getattr(eng, "_jd_shape", (0, 0))
    classes = np.zeros((max(count, 1), max(nc, 1)), dtype=JCLASS_DTYPE)
    hist = np.zeros((max(count, 1), max(nc, 1), 3, ne + 1), dtype=np.uint32)
    eng._check(fn(eng.h, int(first), count, classes.ctypes.data_as(C.c_void_p), hist.ctypes.data_as(C.c_void_p)), what)
    return classes[:count, :nc], hist[:count, :nc]


class Engine:
    """One handle == `nsims` independent replicas on one CUDA device."""

    def __init__(self, device=0, nsims=1):
        self.lib = load_library()
        self.h = C.c_void_p()
        self.nsims = int(nsims)
        self._n = [0] * self.nsims
        self._keep = []
        rc = self.lib.gs_create(int(device), self.nsims, C.byref(self.h))
        if rc != 0:
            msg = self.lib.gs_last_error(None)
            self.h = C.c_void_p()
            raise GsError(f"gs_create failed ({rc}): {msg.decode() if msg else ''}")

    def _check(self, rc, what):
        if rc != 0:
            msg = self.lib.gs_last_error(self.h)
            raise GsError(f"{what} failed ({rc}): {msg.decode() if msg else ''}", rc)

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.lib.gs_destroy(self.h)
            self.h = C.c_void_p()

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def config(self, sim, cluster: GsCluster, policy: GsPolicy | None = None):
        policy = policy or make_policy()
        self._check(self.lib.gs_config_sim(self.h, sim, C.byref(cluster), C.byref(policy)), "gs_config_sim")

    def load_trace(self, sim, table):
        def arr(a, dt):
            return None if a is None else np.ascontiguousarray(a, dtype=dt)
        a = arr(table.arrive_tick, np.int32)
        g = arr(table.gpus, np.int32)
        c = arr(table.gpu_per_task, np.int32)
        d = arr(table.duration, np.float64)
        m = arr(table.mem_bytes, np.int64)
        mm = arr(table.model_mb, np.float64)
        it = arr(table.iterations, np.float64)
        ps = arr(table.ps_count, np.int32)
        self._check(self.lib.gs_load_trace(
            self.h, sim, int(table.n), _ptr(a, C.c_int32), _ptr(g, C.c_int32), _ptr(c, C.c_int32),
            _ptr(d, C.c_double), _ptr(m, C.c_int64), _ptr(mm, C.c_double), _ptr(it, C.c_double),
            _ptr(ps, C.c_int32)), "gs_load_trace")
        self._n[sim] = int(table.n)                 # only once the replica holds the trace (fetch_trace sizes by it)

    def set_engine(self, mode):
        """event-driven policies: 0 / 1 = warp per replica, 2 = thread per replica (the fifo engine has one mapping)"""
        self._check(self.lib.gs_set_engine(self.h, int(mode)), "gs_set_engine")

    def load_trace_packed(self, sim, packed, model_mb=None, iterations=None):
        """`packed`: JOBIN_DTYPE array (JobTable.packed())."""
        packed = np.ascontiguousarray(packed, dtype=JOBIN_DTYPE)
        mm = None if model_mb is None else np.ascontiguousarray(model_mb, dtype=np.float64)
        it = None if iterations is None else np.ascontiguousarray(iterations, dtype=np.float64)
        self._check(self.lib.gs_load_trace_packed(self.h, sim, len(packed), packed.ctypes.data_as(C.c_void_p),
                                                  _ptr(mm, C.c_double), _ptr(it, C.c_double)), "gs_load_trace_packed")
        self._n[sim] = len(packed)

    def fetch_all(self, sim, rows_out, jobs_out, order_out, off_out, spans_out, first=0, count=None):
        """One call: rows of the last window, job records, finish order, spans by job (into caller buffers)."""
        st = self.stats(sim)
        if count is None:
            count = st.ticks - first
        used = C.c_int64(0)
        self._check(self.lib.gs_fetch_all(self.h, sim, int(first), int(count), rows_out.ctypes.data_as(C.c_void_p),
                                          jobs_out.ctypes.data_as(C.c_void_p), _ptr(order_out, C.c_int32),
                                          _ptr(off_out, C.c_int64), spans_out.ctypes.data_as(C.c_void_p),
                                          len(spans_out), C.byref(used)), "gs_fetch_all")
        n = self._n[sim]
        return (rows_out[:int(count)], jobs_out[:n], order_out[:int(st.finished)], off_out[:n + 1],
                spans_out[:used.value])

    # ---- compact, asynchronous result path (fifo engine)
    def window(self, sim=0) -> GsWindowInfo:
        w = GsWindowInfo()
        self._check(self.lib.gs_window(self.h, sim, C.byref(w)), "gs_window")
        return w

    def set_async(self, on=True):
        self._check(self.lib.gs_set_async(self.h, 1 if on else 0), "gs_set_async")

    def set_queue_rows_cap(self, cap):
        self._check(self.lib.gs_set_queue_rows_cap(self.h, int(cap)), "gs_set_queue_rows_cap")

    def sync(self):
        self._check(self.lib.gs_sync(self.h), "gs_sync")

    def fetch_compact_into(self, sim, ev=None, qr=None, ne=None, jobs=None, dur=None, order=None, spans=None):
        """Enqueue the copies of one replica's compact results into caller buffers (numpy views, ideally of
        PinnedBuffer memory, each at least as long as window(sim) says); returns at once -- call sync()."""
        def vp(a):
            return None if a is None else a.ctypes.data_as(C.c_void_p)
        self._check(self.lib.gs_fetch_compact(self.h, sim, vp(ev), vp(qr), vp(ne), vp(jobs), vp(dur), vp(order), vp(spans)),
                    "gs_fetch_compact")

    def load_traces_packed(self, block, pitch_bytes, n_each):
        """every replica's trace from one host block (numpy uint8 / record view; trace i at i * pitch_bytes): one strided upload"""
        n_each = np.ascontiguousarray(n_each, dtype=np.int64)
        assert len(n_each) == self.nsims
        self._keep_block = (block, n_each)
        self._check(self.lib.gs_load_traces_packed(self.h, block.ctypes.data_as(C.c_void_p), int(pitch_bytes), _ptr(n_each, C.c_int64)),
                    "gs_load_traces_packed")
        self._n = [int(k) for k in n_each.tolist()]

    # ---- bootstrap replicas generated on the device (include/gsched.h: gs_boot_*)
    def boot_population(self, table_or_packed):
        """the base trace every replica is drawn from: a JobTable or JOBIN_DTYPE records (validated, copied to the device)"""
        packed = table_or_packed.packed() if hasattr(table_or_packed, "packed") else table_or_packed
        packed = np.ascontiguousarray(packed, dtype=JOBIN_DTYPE)
        self._check(self.lib.gs_boot_population(self.h, packed.ctypes.data_as(C.c_void_p), len(packed)), "gs_boot_population")
        self._pop_k = len(packed)

    def boot_mixes(self, weights):
        """the job mixes of the current population (gs_boot_mixes): `weights` holds one row of uint32 weights per mix,
        one weight per population record (shape (mixes, k)); mix m draws record i with probability w_i / sum(w).
        An empty array (shape (0, k) or (0,)) clears them"""
        w = np.asarray(weights)
        if w.size == 0:
            self._check(self.lib.gs_boot_mixes(self.h, 0, None), "gs_boot_mixes")
            return
        if w.ndim != 2 or w.dtype.kind not in "iu" or (w < 0).any() or (w > 2 ** 32 - 1).any():
            raise ValueError("boot_mixes: expected a 2-d array of uint32 weights (mixes, population records)")
        k = getattr(self, "_pop_k", None)
        if k is not None and w.shape[1] != k:
            raise ValueError(f"boot_mixes: expected one weight per population record ({k}), got {w.shape[1]}")
        w = np.ascontiguousarray(w, dtype=np.uint32)
        self._check(self.lib.gs_boot_mixes(self.h, len(w), w.ctypes.data_as(C.c_void_p)), "gs_boot_mixes")

    def boot_profiles(self, profiles):
        """the load profiles of the handle (gs_boot_profiles): a list of (segments, period), segments being
        BOOT_SEG_DTYPE records or (start, gap_num, gap_den) triples; an empty list clears them"""
        from .tracegen import check_profile
        segs, nseg, period = [], [], []
        for prof in profiles:
            t, num, den, P = check_profile(*prof)
            segs += [(a, b, c, 0) for a, b, c in zip(t, num, den)]
            nseg.append(len(t))
            period.append(P)
        if not nseg:
            self._check(self.lib.gs_boot_profiles(self.h, 0, None, None, None), "gs_boot_profiles")
            return
        S = np.array(segs, dtype=np.int64).astype(np.int32).view(BOOT_SEG_DTYPE).reshape(-1)
        N, P = np.array(nseg, dtype=np.int32), np.array(period, dtype=np.int32)
        self._check(self.lib.gs_boot_profiles(self.h, len(N), N.ctypes.data_as(C.c_void_p), P.ctypes.data_as(C.c_void_p),
                                              S.ctypes.data_as(C.c_void_p)), "gs_boot_profiles")

    def boot_traces(self, params, with_time=False, block_len=None, mix=None, profile=None):
        """draw every replica's trace from the population: `params` holds one BOOT_PARAMS_DTYPE record per replica.
        block_len: the mean block length L of a block bootstrap (gs_boot_traces_blocked), one integer for every
        replica or one per replica; None draws iid replicas (gs_boot_traces).  mix: the job mix of boot_mixes each
        replica draws its rows from (gs_boot_traces_mixed), one index for every replica or one per replica, -1 for
        the unweighted bootstrap; None draws every replica unweighted.  profile: the load profile of boot_profiles
        each replica takes its arrivals from (gs_boot_traces_profiled; a profiled replica's gap scale must be 1 / 1),
        one index for every replica or one per replica, -1 for none; None profiles no replica.  with_time: returns the
        generator's kernel milliseconds"""
        params = np.ascontiguousarray(params, dtype=BOOT_PARAMS_DTYPE)
        if params.shape != (self.nsims,):
            raise ValueError(f"boot_traces: one parameter record per replica ({self.nsims}), got shape {params.shape}")
        ms = C.c_double(0.0)
        if block_len is not None:
            L = np.asarray(block_len)
            if L.dtype.kind not in "iu" or L.shape not in ((), (self.nsims,)) or (L < 0).any() or (L > 2 ** 32 - 1).any():
                raise ValueError(f"boot_traces: block_len must be one uint32 or one per replica ({self.nsims})")
            L = np.ascontiguousarray(np.broadcast_to(L, (self.nsims,)), dtype=np.uint32)
        if mix is not None:
            M = np.asarray(mix)
            if M.dtype.kind not in "iu" or M.shape not in ((), (self.nsims,)) or (M < -2 ** 31).any() or (M > 2 ** 31 - 1).any():
                raise ValueError(f"boot_traces: mix must be one int32 or one per replica ({self.nsims})")
            M = np.ascontiguousarray(np.broadcast_to(M, (self.nsims,)), dtype=np.int32)
        if profile is not None:
            Q = np.asarray(profile)
            if Q.dtype.kind not in "iu" or Q.shape not in ((), (self.nsims,)) or (Q < -2 ** 31).any() or (Q > 2 ** 31 - 1).any():
                raise ValueError(f"boot_traces: profile must be one int32 or one per replica ({self.nsims})")
            Q = np.ascontiguousarray(np.broadcast_to(Q, (self.nsims,)), dtype=np.int32)
            self._check(self.lib.gs_boot_traces_profiled(self.h, params.ctypes.data_as(C.c_void_p),
                                                         None if block_len is None else L.ctypes.data_as(C.c_void_p),
                                                         None if mix is None else M.ctypes.data_as(C.c_void_p),
                                                         Q.ctypes.data_as(C.c_void_p), C.byref(ms)), "gs_boot_traces_profiled")
        elif mix is not None:
            self._check(self.lib.gs_boot_traces_mixed(self.h, params.ctypes.data_as(C.c_void_p),
                                                      None if block_len is None else L.ctypes.data_as(C.c_void_p),
                                                      M.ctypes.data_as(C.c_void_p), C.byref(ms)), "gs_boot_traces_mixed")
        elif block_len is None:
            self._check(self.lib.gs_boot_traces(self.h, params.ctypes.data_as(C.c_void_p), C.byref(ms)), "gs_boot_traces")
        else:
            self._check(self.lib.gs_boot_traces_blocked(self.h, params.ctypes.data_as(C.c_void_p), L.ctypes.data_as(C.c_void_p), C.byref(ms)),
                        "gs_boot_traces_blocked")
        self._n = [int(k) for k in params["n"].tolist()]
        return ms.value if with_time else None

    def fetch_trace(self, sim=0):
        """the JOBIN_DTYPE records of the trace replica `sim` holds on the device (loaded or generated)"""
        out = np.zeros(max(self._n[sim], 1), dtype=JOBIN_DTYPE)
        self._check(self.lib.gs_fetch_trace(self.h, sim, out.ctypes.data_as(C.c_void_p)), "gs_fetch_trace")
        return out[:self._n[sim]]

    def result_layout(self, sim=0) -> GsResultLayout:
        lay = GsResultLayout()
        self._check(self.lib.gs_result_layout(self.h, sim, C.byref(lay)), "gs_result_layout")
        return lay

    def fetch_results(self, out, out_pitch, first=0, count=None):
        """enqueue ONE strided copy of the result blocks of replicas [first, first+count) into `out`; call sync()"""
        count = self.nsims - first if count is None else count
        self._check(self.lib.gs_fetch_results(self.h, int(first), int(count), out.ctypes.data_as(C.c_void_p), int(out_pitch)), "gs_fetch_results")

    @staticmethod
    def result_views(buf, pitch, index, lay: "GsResultLayout", win: "GsWindowInfo"):
        """numpy views (records, queue records, node events, job starts, finish order, span pool) of replica `index` inside a fetched block buffer"""
        base = index * pitch
        ev = np.frombuffer(buf, dtype=EVROW_DTYPE, count=int(win.ev_rows), offset=base + lay.off_ev)
        qr = np.frombuffer(buf, dtype=QROW_DTYPE, count=int(win.q_rows), offset=base + lay.off_q)
        ne = np.frombuffer(buf, dtype=NODEEV_DTYPE, count=int(win.node_events), offset=base + lay.off_nodeev)
        jobs = np.frombuffer(buf, dtype=JOBRUN_DTYPE, count=int(win.n), offset=base + lay.off_jobs)
        order = np.frombuffer(buf, dtype=np.int32, count=int(win.finished), offset=base + lay.off_finish_order)
        spans = np.frombuffer(buf, dtype=CSPAN_DTYPE if lay.span_bytes == 8 else SPAN_DTYPE, count=int(win.spans_used), offset=base + lay.off_spans)
        return ev, qr, ne, jobs, order, spans

    def fetch_compact(self, sim=0):
        """(window info, gs_evrow[], gs_qrow[], gs_nodeev[], gs_job_start[], duration-after-network-cost or None, finish order, span pool)"""
        w = self.window(sim)
        n = int(w.n)
        ev = np.empty(max(int(w.ev_rows), 1), dtype=EVROW_DTYPE)
        qr = np.empty(max(int(w.q_rows), 1), dtype=QROW_DTYPE)
        ne = np.empty(max(int(w.node_events), 1), dtype=NODEEV_DTYPE)
        jobs = np.empty(max(n, 1), dtype=JOBRUN_DTYPE)
        dur = np.full(max(n, 1), np.nan)
        order = np.empty(max(int(w.finished), 1), dtype=np.int32)
        spans = np.empty(max(int(w.spans_used), 1), dtype=CSPAN_DTYPE if self.result_layout(sim).span_bytes == 8 else SPAN_DTYPE)
        self.fetch_compact_into(sim, ev, qr, ne, jobs, dur, order, spans)
        self.sync()
        return (w, ev[:int(w.ev_rows)], qr[:int(w.q_rows)], ne[:int(w.node_events)], jobs[:n], (None if n == 0 or np.isnan(dur[0]) else dur[:n]),
                order[:int(w.finished)], spans[:int(w.spans_used)])

    def switch_yarn(self, clusters, mem=SWITCH_MEM):
        """Legacy switch-local yarn placement with PS traffic (include/gsched.h: gs_switch_yarn).
        clusters: list of dicts {num_switch, num_node_p_switch, num_gpu_p_node, free_gpus[], free_cpus[], free_mem[],
        jobs: [(num_gpu, model_size, ps_network list)]}.  Returns per cluster (answers[(n_nodes, switch, spans)], node table)."""
        ncl = len(clusters)
        cl = np.zeros(ncl, dtype=SWITCH_CLUSTER_DTYPE)
        nodes, jobs, ps = [], [], []
        n_spans = 0
        for i, c in enumerate(clusters):
            m = c["num_switch"] * c["num_node_p_switch"]
            cl[i] = (c["num_switch"], c["num_node_p_switch"], c["num_gpu_p_node"], 0, len(nodes), len(jobs), len(c["jobs"]))
            for k in range(m):
                nodes.append((c["free_gpus"][k], c["free_cpus"][k], c["free_mem"][k], 0.0))
            for g, model, psn in c["jobs"]:
                jobs.append((g, len(psn), len(ps), n_spans, model))
                ps.extend(psn)
                n_spans += g // c["num_gpu_p_node"] + 1
        nodes = np.array(nodes, dtype=SWITCH_NODE_DTYPE)
        jobs = np.array(jobs, dtype=SWITCH_JOB_DTYPE) if jobs else np.zeros(0, dtype=SWITCH_JOB_DTYPE)
        ps = np.ascontiguousarray(ps, dtype=np.float64)
        ans = np.zeros(max(len(jobs), 1), dtype=SWITCH_ANS_DTYPE)
        spans = np.zeros(max(n_spans, 1), dtype=SWITCH_SPAN_DTYPE)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        self._check(self.lib.gs_switch_yarn(self.h, ncl, vp(cl), vp(nodes), len(nodes), vp(jobs), len(jobs), _ptr(ps, C.c_double), len(ps),
                                            mem[0], mem[1], mem[2], vp(ans), vp(spans), n_spans), "gs_switch_yarn")
        out = []
        for i in range(ncl):
            jo, jc, no = int(cl["job_off"][i]), int(cl["job_cnt"][i]), int(cl["node_off"][i])
            res = []
            for j in range(jo, jo + jc):
                k, so = int(ans["n_nodes"][j]), int(jobs["span_off"][j])
                res.append((k, int(ans["sw"][j]), spans[so:so + k].copy()))
            out.append((res, nodes[no:no + clusters[i]["num_switch"] * clusters[i]["num_node_p_switch"]].copy()))
        return out

    # ---- one simulation on several GPUs of one box (gittins; include/gsched.h: gs_comm_*)
    def comm_prepare(self, max_jobs) -> bytes:
        """allocate this handle's exchange buffer; returns its 64-byte IPC handle (send it to every rank)"""
        buf = (C.c_uint8 * 64)()
        self._check(self.lib.gs_comm_prepare(self.h, int(max_jobs), C.cast(buf, C.c_void_p)), "gs_comm_prepare")
        return bytes(buf)

    def comm_init(self, rank, handles):
        """handles: the 64-byte IPC handles of ALL ranks, in rank order (own at [rank])"""
        blob = b"".join(bytes(hb) for hb in handles)
        assert len(blob) == 64 * len(handles)
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        self._check(self.lib.gs_comm_init(self.h, int(rank), len(handles), C.cast(buf, C.c_void_p)), "gs_comm_init")

    def comm_set_min_runnable(self, k):
        """events with at most k runnable jobs are evaluated locally by every rank; 0 = always exchange; default: never exchange (include/gsched.h)"""
        self._check(self.lib.gs_comm_set_min_runnable(self.h, int(k)), "gs_comm_set_min_runnable")

    def comm_stats(self):
        """(exchanges of the last run, mean microseconds from publishing to having seen every peer)"""
        n, us = C.c_int64(0), C.c_double(0.0)
        self._check(self.lib.gs_comm_stats(self.h, C.byref(n), C.byref(us)), "gs_comm_stats")
        return int(n.value), float(us.value)

    def set_span_budget(self, spans_per_job):
        self._check(self.lib.gs_set_span_budget(self.h, float(spans_per_job)), "gs_set_span_budget")

    def reset(self):
        self._check(self.lib.gs_reset(self.h), "gs_reset")

    def launch_count(self):
        return int(self.lib.gs_launch_count(self.h))

    def run(self, max_ticks=0, rows_cap=0):
        self._check(self.lib.gs_run(self.h, int(max_ticks), int(rows_cap)), "gs_run")

    def run_all(self, rows_cap=0, collect_rows=True):
        """Run every replica to its exit condition.  The device keeps a window of
        `rows_cap` statistics rows per replica; it is drained after every launch.
        Returns one concatenated row array per replica (or None)."""
        parts = [[] for _ in range(self.nsims)]
        seen = [0] * self.nsims
        while True:
            self.run(0, rows_cap)
            pending = 0
            for s in range(self.nsims):
                st = self.stats(s)
                if collect_rows and st.ticks > seen[s]:
                    parts[s].append(self.fetch_rows(s, seen[s], st.ticks - seen[s]))
                seen[s] = st.ticks
                pending += 0 if st.done else 1
            if pending == 0:
                break
        if not collect_rows:
            return None
        return [np.concatenate(p) if p else np.empty(0, dtype=ROW_DTYPE) for p in parts]

    def summarize(self, first=0, count=None, with_time=False):
        """SUMMARY_DTYPE records of replicas [first, first+count): folds the rows of the last window not folded yet,
        recomputes the job part (include/gsched.h: gs_summarize).  Call it after every run() of a multi-window run.
        with_time: (records, kernel milliseconds)"""
        count = self.nsims - first if count is None else int(count)
        out = np.zeros(max(count, 1), dtype=SUMMARY_DTYPE)
        ms = C.c_double(0.0)
        self._check(self.lib.gs_summarize(self.h, int(first), count, out.ctypes.data_as(C.c_void_p), C.byref(ms)), "gs_summarize")
        return (out[:count], ms.value) if with_time else out[:count]

    def set_timeline(self, width, nbins):
        """while nbins > 0, every summarize() also bins the rows it folds by min(delta // width, nbins - 1) on the
        device; nbins = 0 turns it off.  Set it before the first summarize() of a run (include/gsched.h: gs_set_timeline)"""
        self._check(self.lib.gs_set_timeline(self.h, int(width), int(nbins)), "gs_set_timeline")
        self._tl_nbins = int(nbins)

    def timeline(self, first=0, count=None):
        """TBIN_DTYPE bins of replicas [first, first+count) as of the last summarize(): shape (count, nbins)"""
        return _fetch_timeline(self, self.lib.gs_fetch_timeline, "gs_fetch_timeline", first, count)

    def set_jobdist(self, bounds, edges):
        """while set, every summarize() also computes per-replica job statistics by job size on the device:
        len(bounds) + 1 classes (a job's class is the number of bounds <= its num_gpu) and CDF counts of wait /
        turnaround / jct at `edges`; bounds=None turns it off.  May be called at any time (include/gsched.h: gs_set_jobdist)"""
        _set_jobdist(self, self.lib.gs_set_jobdist, "gs_set_jobdist", bounds, edges)

    def jobdist(self, first=0, count=None):
        """(JCLASS_DTYPE records (count, C), uint32 CDF counts (count, C, 3, E + 1)) of replicas [first, first+count)
        as of the last summarize(); count[..., m, b] = #(value m <= edges[b]) - #(value m <= edges[b - 1])"""
        return _fetch_jobdist(self, self.lib.gs_fetch_jobdist, "gs_fetch_jobdist", first, count)

    def set_slowdown(self, key=None, bounds=(), tau=1, edges=(), sd_edges=()):
        """while set, every summarize() also computes per-replica job statistics by `key` ("gpus", "length" = jct or
        "gpu-time" = gpus * jct) on the device: len(bounds) + 1 classes (a job's class is the number of bounds <= its
        key), bounded slowdown sd = 1024 * turnaround / max(jct, tau) in units of 1/1024 (at least 1024, at most
        2^31 - 1), CDF counts of wait / turnaround / jct at `edges` and of sd at `sd_edges`; key=None turns it off.  May
        be called at any time (include/gsched.h: gs_set_slowdown)"""
        _set_slowdown(self, self.lib.gs_set_slowdown, "gs_set_slowdown", key, bounds, tau, edges, sd_edges)

    def slowdown(self, first=0, count=None):
        """(SDCLASS_DTYPE records (count, C), uint32 CDF counts (count, C, 3 * (E + 1) + Esd + 1): the wait, turnaround
        and jct rows of E + 1 counts, then the sd row of Esd + 1) of replicas [first, first+count) as of the last
        summarize()"""
        return _fetch_slowdown(self, self.lib.gs_fetch_slowdown, "gs_fetch_slowdown", first, count)

    def set_arrivals(self, width, bins, tau=1):
        """while bins > 0, every summarize() also computes per-replica job statistics by arrival time on the device:
        a job that arrived at tick a falls in bin min(a // width, bins - 1), and each bin holds slowdown's record of
        its finished jobs (bounded slowdown with lower bound tau, the arrival tick as the key) and the count of its
        trace jobs; bins = 0 turns it off.  May be called at any time (include/gsched.h: gs_set_arrivals)"""
        _set_arrivals(self, self.lib.gs_set_arrivals, "gs_set_arrivals", width, bins, tau)

    def arrivals(self, first=0, count=None):
        """ABIN_DTYPE records (count, bins) of replicas [first, first+count) as of the last summarize()"""
        return _fetch_arrivals(self, self.lib.gs_fetch_arrivals, "gs_fetch_arrivals", first, count)

    def set_occupancy(self, queue_edges=None):
        """time-weighted occupancy filled by every summarize(): each row weighed by the ticks it stands for, busy-GPU
        histograms over all time and over the ticks with a queue, queue-length CDF counts at `queue_edges`; None turns it
        off.  Set it before the first summarize() of a run (include/gsched.h: gs_set_occupancy)"""
        _set_occupancy(self, self.lib.gs_set_occupancy, "gs_set_occupancy", queue_edges)

    def occupancy(self, first=0, count=None):
        """(OCC_DTYPE records (count,), uint64 busy histograms (count, 2, max total_gpus + 1): all time, waiting time,
        uint64 queue histograms (count, E + 1)) of replicas [first, first+count) as of the last summarize()"""
        return _fetch_occupancy(self, self.lib.gs_fetch_occupancy, "gs_fetch_occupancy", first, count)

    def compare(self, a, b, bounds=(), edges=(), with_time=False):
        """paired per-job comparison of replicas b[i] against a[i], which hold the same trace, over the jobs finished so
        far (include/gsched.h: gs_compare): len(bounds) + 1 classes by num_gpu, per quantity d = x_b - x_a of wait /
        turnaround / jct.  Returns (JPAIR_DTYPE records (P, C), uint32 CDF counts of d at `edges` (P, C, 3, E + 1));
        with_time: and the kernel milliseconds"""
        return _compare(self, self.lib.gs_compare, "gs_compare", a, b, bounds, edges, with_time)

    def run_summarized(self, rows_cap=0):
        """Run every replica to its exit condition, summarising after every launch and fetching no rows; returns
        the final SUMMARY_DTYPE records of all replicas."""
        while True:
            self.run(0, rows_cap)
            out = self.summarize()
            if out["done"].all():
                return out

    def stats(self, sim=0) -> GsRunStats:
        st = GsRunStats()
        self._check(self.lib.gs_stats(self.h, sim, C.byref(st)), "gs_stats")
        return st

    def fetch_rows(self, sim=0, first=0, count=None, out=None):
        if count is None:
            count = self.stats(sim).ticks - first
        rows = np.empty(int(count), dtype=ROW_DTYPE) if out is None else out[:int(count)]
        self._check(self.lib.gs_fetch_rows(self.h, sim, int(first), int(count),
                                           rows.ctypes.data_as(C.c_void_p)), "gs_fetch_rows")
        return rows

    def fetch_jobs(self, sim=0, out_recs=None, out_order=None):
        n = self._n[sim]
        recs = np.empty(n, dtype=JOB_DTYPE) if out_recs is None else out_recs[:n]
        order = np.empty(max(n, 1), dtype=np.int32) if out_order is None else out_order
        self._check(self.lib.gs_fetch_jobs(self.h, sim, recs.ctypes.data_as(C.c_void_p),
                                           _ptr(order, C.c_int32)), "gs_fetch_jobs")
        return recs, order[:int(self.stats(sim).finished)]

    def fetch_spans(self, sim=0, out_off=None, out_spans=None):
        """(span_off[n+1], spans) grouped by job; optional caller (pinned) buffers."""
        n = self._n[sim]
        off = np.zeros(n + 1, dtype=np.int64) if out_off is None else out_off[:n + 1]
        used = C.c_int64(0)
        if out_spans is None:
            self._check(self.lib.gs_fetch_spans(self.h, sim, None, None, 0, C.byref(used)), "gs_fetch_spans")
            out_spans = np.empty(max(int(used.value), 1), dtype=SPAN_DTYPE)
        self._check(self.lib.gs_fetch_spans(self.h, sim, _ptr(off, C.c_int64),
                                            out_spans.ctypes.data_as(C.c_void_p), len(out_spans),
                                            C.byref(used)), "gs_fetch_spans")
        return off, out_spans[:used.value]

    def place_batch(self, cluster: GsCluster, nodes, jobs, task_off=None):
        nodes = np.ascontiguousarray(nodes, dtype=NODE_DTYPE)
        jobs = np.ascontiguousarray(jobs, dtype=JOBREQ_DTYPE)
        b = len(jobs)
        first = np.empty(b, dtype=np.int32)
        used = np.empty(b, dtype=np.int32)
        task_node = None
        if task_off is not None:
            task_off = np.ascontiguousarray(task_off, dtype=np.int64)
            task_node = np.empty(int(task_off[-1]), dtype=np.int32)
        ms = C.c_double(0.0)
        self._check(self.lib.gs_place_batch(
            self.h, C.byref(cluster), nodes.ctypes.data_as(C.c_void_p), len(nodes),
            jobs.ctypes.data_as(C.c_void_p), b, _ptr(first, C.c_int32), _ptr(used, C.c_int32),
            _ptr(task_off, C.c_int64), _ptr(task_node, C.c_int32), C.byref(ms)), "gs_place_batch")
        return first, used, task_node, ms.value

    def net_cost(self, cluster: GsCluster, task_off, task_node, is_ps, ps_count, model_mb, iterations):
        task_off = np.ascontiguousarray(task_off, dtype=np.int64)
        task_node = np.ascontiguousarray(task_node, dtype=np.int32)
        is_ps = None if is_ps is None else np.ascontiguousarray(is_ps, dtype=np.uint8)
        ps_count = np.ascontiguousarray(ps_count, dtype=np.int32)
        model_mb = np.ascontiguousarray(model_mb, dtype=np.float64)
        iterations = np.ascontiguousarray(iterations, dtype=np.float64)
        b = len(ps_count)
        out = np.empty(b, dtype=np.float64)
        self._check(self.lib.gs_net_cost(
            self.h, C.byref(cluster), b, _ptr(task_off, C.c_int64), _ptr(task_node, C.c_int32),
            _ptr(is_ps, C.c_uint8), _ptr(ps_count, C.c_int32), _ptr(model_mb, C.c_double),
            _ptr(iterations, C.c_double), _ptr(out, C.c_double)), "gs_net_cost")
        return out

// gsched.cu -- sm_90a (H100) discrete-event engine + C ABI (include/gsched.h).
//
// Execution model (GPU-first, not a translation of the Python object graph):
//   * one WARP owns one simulation replica ("sim").  The cluster's node table
//     lives in shared memory as (busy-device mask, charged task slots) -- the
//     reference's cpu_used/mem_used always move together in units of 12/60 per
//     task (job.py:105-106, node.py:204-205), so both collapse into one slot
//     counter k with  free_slots = min(cpu/12, mem/60) - k.
//   * lanes stripe over nodes; single-node first fit is a ballot + ffs (argmin
//     over node id), cross-node fill is a warp prefix sum over per-node task
//     capacities with a cut-off -- no per-device objects are ever walked.
//   * all reference per-tick re-scans (pandas filters, _construct_info,
//     pending-time aging, time_processed stepping) are replaced by closed
//     forms and O(1) incremental counters; completions come from a timing
//     wheel keyed by finish tick, appended in start order.
//   * the loop is event stepped: ticks on which nothing arrives, starts or
//     finishes are jumped over; every other tick leaves one 24-byte record of
//     integer aggregates (+ one for the queue while it is non-empty) from which
//     the 64-byte gs_tick_row of EVERY tick is rebuilt on demand; the job table
//     is streamed once from HBM, results are written once (4-byte start tick per job +
//     8-byte gs_cspan per (job,node) + finish order).
//   * thousands of replicas run per launch (one warp each, 132 SMs x 28
//     warps); a single replica is latency bound by construction.
//
// Reference semantics followed (paths relative to the reference root):
//   Scheduler.start            core/scheduling/schedule.py:178-215
//   Scheduler._schedule        core/scheduling/schedule.py:40-60
//   schedule_fifo              core/scheduling/algorithm.py:189-202
//   ms_yarn_placement          core/scheduling/algorithm.py:28-32
//   try_single_node_alloc_ms   core/scheduling/algorithm.py:396-417
//   try_cross_node_alloc_ms    core/scheduling/algorithm.py:301-393
//   Node fit/reserve/release   infra/node.py:71-91,109-127,146-171,200-275
//   Device.can_fit             infra/device.py:67-77
//   gen_jobs / step / finish   core/jobs/jobs_manager.py:65-87,143-148,228-250
//   calculate_network_costs    core/network/network_service.py:3-39
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "gsched.h"

#include "gs_common.cuh"
#include "gs_tick2.cuh"
#include "gs_policy.cuh"
#include "gs_aux.cuh"
#include "gs_switch.cuh"
#include "gs_summary.cuh"
#include "gs_boot.cuh"

// ------------------------------------------------------------------ host side

// Per-replica device layout.  The RESULT arrays come first and contiguously (gs_result_layout): statistics records,
// queue records, per-job results, (durations,) finish order, spans -- so that everything a caller reads back from a
// replica is ONE copy, and from all replicas of a handle ONE strided copy (the slabs live side by side in an arena).
struct SimLayout {
  size_t o_ev = 0, o_q = 0, o_ne = 0, o_rec2 = 0, o_dur2 = 0, o_fin = 0, o_spans = 0, out_bytes = 0;
  size_t o_rec = 0, o_rows = 0, o_jst = 0, o_stack = 0, o_wh = 0, o_wm = 0, o_nb = 0, o_nk = 0;
  size_t o_pj = 0, o_run = 0, o_qs = 0, o_end = 0, o_tmp = 0, o_ci = 0, o_ck = 0, o_stale = 0;
  size_t total = 0;
  int64_t rows_cap = 0, qrows_cap = 0;
  int W = 256;
};

struct SimHost {
  gs_cluster cl;
  gs_policy pol;
  bool configured = false, loaded = false, prepared = false;
  int64_t n = 0;
  void *trace_slab = nullptr;
  void *state_slab = nullptr;
  void *git_dev = nullptr;
  long long git_direct_n = 0;       // entries of the direct look-up table behind the two gittins tables in git_dev
  size_t trace_bytes = 0, state_bytes = 0;
  int64_t span_cap = 0, rows_cap = 0, qrows_cap = 0, last_arrive = 0;
  int max_need = 1;
  unsigned char *state_ptr = nullptr;     // the replica's slab: inside the handle's arena or its own allocation (state_slab)
  bool trace_in_arena = false;
  int64_t sum_rows = 0;                   // gs_summarize: rows folded into the replica's accumulator (its watermark)
  bool sum_fresh = true;                  // the accumulator is to be zeroed before the next fold (the replica was prepared afresh)
  bool tl_fresh = true;                   // gs_set_timeline: the bins are to be zeroed before the next fold
  bool tl_done = false;                   // summarised with the timeline on since it was prepared
  bool jd_done = false;                   // summarised with the current jobdist setting since it was prepared
  bool sd_done = false;                   // summarised with the current slowdown setting since it was prepared
  bool arr_done = false;                  // summarised with the current arrivals setting since it was prepared
  bool occ_fresh = true;                  // the occupancy record, carry and histograms are to be zeroed before the next fold
  bool occ_done = false;                  // summarised with the occupancy on since it was prepared
  SimDev dev;
  SimLayout layout;
};

struct gs_engine {
  int device = 0, nsims = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  cudaEvent_t e_wait = nullptr;   // blocking-sync event: in asynchronous mode the driving thread sleeps while it waits
  std::vector<SimHost> sims;
  SimDev *d_sims = nullptr;
  void *h_stage = nullptr;
  size_t h_stage_bytes = 0;
  void *d_scratch = nullptr;
  size_t d_scratch_bytes = 0;
  std::vector<SimDev> h_back;   // pinned-size-stable host mirror used by gs_run
  // arenas: the replicas' state slabs (result block first) / traces side by side with one stride, so that a whole
  // handle is read back or uploaded with ONE strided copy (gs_fetch_results / gs_load_traces_packed)
  void *arena = nullptr; size_t arena_bytes = 0, arena_stride = 0;
  void *tarena = nullptr; size_t tarena_bytes = 0, tarena_stride = 0;
  std::string err;
  double kernel_ms = 0, h2d_ms = 0, d2h_ms = 0;
  long long launches = 0;  // kernels launched by this handle
  int engine_mode = 0;     // event-driven policies: 0 warp-cooperative kernels, 2 one thread per replica
  double span_budget = 0;  // > 0: span pool = min(worst case, budget * n + 4096) records per replica
  int64_t qrows_cap = 0;   // 0: same as rows_cap
  bool async = false;      // gs_set_async
  // sharded single simulation (gs_comm_prepare / gs_comm_init)
  void *comm_buf = nullptr; int64_t comm_cap = 0; int comm_rank = 0, comm_n = 0;
  void *comm_peer[GS_MAX_RANKS] = {nullptr}; bool comm_opened[GS_MAX_RANKS] = {false};
  int comm_min_runnable = 0x7fffffff;      // gs_comm_set_min_runnable: no exchange unless the caller asks for one (include/gsched.h)
  unsigned long long comm_epoch = 0, comm_epoch0 = 0;   // exchange counter: continues across runs / value at the last prepare
  bool dirty = true;       // host mirror of SimDev newer than device copy
  gs_summary *d_sum = nullptr;   // gs_summarize: one accumulator per replica
  gs_tbin *d_tl = nullptr; size_t tl_bytes = 0;   // gs_set_timeline: nsims x tl_nbins bins
  int64_t tl_width = 0; int tl_nbins = 0;
  gs_jclass *d_jd = nullptr; size_t jd_bytes = 0;       // gs_set_jobdist: nsims x C class records
  unsigned *d_jd_hist = nullptr; size_t jd_hist_bytes = 0;   // and nsims x C x 3 x (E + 1) CDF counts
  GsJdCfg jd{};                                          // jd.nclasses = 0: off
  gs_sdclass *d_sd = nullptr; size_t sd_bytes = 0;      // gs_set_slowdown: nsims x C class records
  unsigned *d_sd_hist = nullptr; size_t sd_hist_bytes = 0;   // and nsims x C x (3 (E + 1) + Esd + 1) CDF counts
  GsSdCfg sd{};                                          // sd.nclasses = 0: off
  gs_abin *d_arr = nullptr; size_t arr_bytes = 0;       // gs_set_arrivals: nsims x B bin records, only while on
  GsArrCfg arr{};                                        // arr.nbins = 0: off
  bool occ_on = false; GsOccCfg occ{};                   // gs_set_occupancy
  gs_occ *d_occ = nullptr; GsOccCarry *d_occ_carry = nullptr;   // nsims records and carries
  unsigned long long *d_occ_busy = nullptr; int64_t occ_pitch = 0;   // nsims x [H_all, H_wait] x occ_pitch counters
  unsigned long long *d_occ_q = nullptr; size_t occ_q_bytes = 0;     // nsims x (E + 1) queue counters
  // gs_boot_population: the records of the base trace, then its k - 1 gaps (int32)
  void *d_pop = nullptr; int64_t pop_k = 0; int64_t pop_max_gap = 0; double pop_max_need = 1.0;
  // gs_boot_mixes: nmix alias tables of pop_k entries each, mix-major, and their weight sums
  GsBootAlias *d_mix = nullptr; int32_t nmix = 0; std::vector<uint64_t> mix_T;
  // gs_boot_profiles: the device form of nprof profiles, profile-major, with a host copy for the arrival bound
  GsBootProfSeg *d_prof = nullptr; int32_t nprof = 0;
  std::vector<GsBootProfSeg> prof_seg; std::vector<int32_t> prof_off, prof_nseg, prof_period; std::vector<long long> prof_B;
};

static std::string g_create_err;

static int fail(gs_handle h, int code, const std::string &msg) {
  if (h) h->err = msg; else g_create_err = msg;
  return code;
}
#define CU(call)                                                                          \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess)                                                                \
      return fail(h, GS_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));    \
  } while (0)

static size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// Wait for the handle's stream.  Asynchronous mode is what many host threads use side by side (one handle each): there the
// waiting thread sleeps on a blocking-sync event instead of spinning, which leaves the cores to the threads that work.
static cudaError_t wait_stream(gs_handle h) {
  if (!h->async) return cudaStreamSynchronize(h->stream);
  cudaError_t e = cudaEventRecord(h->e_wait, h->stream);
  return e != cudaSuccess ? e : cudaEventSynchronize(h->e_wait);
}

extern "C" int gs_abi_version(void) { return GS_ABI_VERSION; }
extern "C" const char *gs_build_tag(void) {
#ifdef __CUDACC__
  return "cuda:sm_90a";
#else
  return "host-emulation";
#endif
}

extern "C" const char *gs_last_error(gs_handle h) { return h ? h->err.c_str() : g_create_err.c_str(); }

extern "C" int gs_create(int device, int nsims, gs_handle *out) {
  gs_handle h = nullptr;
  if (!out || nsims <= 0) return fail(nullptr, GS_ERR_ARG, "gs_create: bad arguments");
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0)
    return fail(nullptr, GS_ERR_CUDA, std::string("no usable CUDA device (there is no CPU fallback): ") +
                                          (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
  if (device < 0 || device >= count) return fail(nullptr, GS_ERR_ARG, "gs_create: device ordinal out of range");
  CU(cudaSetDevice(device));
  h = new gs_engine();
  h->device = device;
  h->nsims = nsims;
  h->sims.resize((size_t)nsims);
  h->h_back.resize((size_t)nsims);
  cudaError_t e1 = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  cudaError_t e2 = cudaEventCreate(&h->e0);
  cudaError_t e3 = cudaEventCreate(&h->e1);
  cudaError_t e4 = cudaMalloc(&h->d_sims, sizeof(SimDev) * (size_t)nsims);
  if (cudaEventCreateWithFlags(&h->e_wait, cudaEventBlockingSync | cudaEventDisableTiming) != cudaSuccess) e4 = cudaErrorUnknown;
  if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess || e4 != cudaSuccess) {
    delete h;
    return fail(nullptr, GS_ERR_CUDA, "gs_create: stream/event/alloc failed");
  }
  *out = h;
  return GS_OK;
}

extern "C" void gs_destroy(gs_handle h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (auto &s : h->sims) { if (s.trace_slab) cudaFree(s.trace_slab); if (s.state_slab) cudaFree(s.state_slab); if (s.git_dev) cudaFree(s.git_dev); }
  if (h->d_sims) cudaFree(h->d_sims);
  if (h->arena) cudaFree(h->arena);
  if (h->tarena) cudaFree(h->tarena);
  if (h->h_stage) cudaFreeHost(h->h_stage);
  if (h->d_scratch) cudaFree(h->d_scratch);
  if (h->d_sum) cudaFree(h->d_sum);
  if (h->d_tl) cudaFree(h->d_tl);
  if (h->d_jd) cudaFree(h->d_jd);
  if (h->d_jd_hist) cudaFree(h->d_jd_hist);
  if (h->d_sd) cudaFree(h->d_sd);
  if (h->d_sd_hist) cudaFree(h->d_sd_hist);
  if (h->d_arr) cudaFree(h->d_arr);
  if (h->d_occ) cudaFree(h->d_occ);
  if (h->d_occ_carry) cudaFree(h->d_occ_carry);
  if (h->d_occ_busy) cudaFree(h->d_occ_busy);
  if (h->d_occ_q) cudaFree(h->d_occ_q);
  if (h->d_pop) cudaFree(h->d_pop);
  if (h->d_mix) cudaFree(h->d_mix);
  if (h->d_prof) cudaFree(h->d_prof);
  for (int q = 0; q < GS_MAX_RANKS; ++q) if (h->comm_opened[q] && h->comm_peer[q]) cudaIpcCloseMemHandle(h->comm_peer[q]);
  if (h->comm_buf) cudaFree(h->comm_buf);
  if (h->e0) cudaEventDestroy(h->e0);
  if (h->e1) cudaEventDestroy(h->e1);
  if (h->e_wait) cudaEventDestroy(h->e_wait);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

static int check_cluster(gs_handle h, const gs_cluster *c) {
  if (!c) return fail(h, GS_ERR_ARG, "cluster is NULL");
  long long m = (long long)c->num_switch * c->num_node_p_switch;
  if (c->num_switch <= 0 || c->num_node_p_switch <= 0 || m > (1 << 20))
    return fail(h, GS_ERR_ARG, "cluster: num_switch * num_node_p_switch must be in 1..2^20");
  if (c->num_gpu_p_node <= 0 || c->num_gpu_p_node > GS_MAX_GPUS_PER_NODE)
    return fail(h, GS_ERR_ARG, "cluster: num_gpu_p_node must be in 1..64");
  if (c->cpu_per_task <= 0 || c->mem_per_task <= 0 || c->num_cpu_p_node < 0 || c->mem_p_node < 0)
    return fail(h, GS_ERR_ARG, "cluster: cpu/mem per task must be positive");
  if (c->gpu_mem_cap_mib <= 0) return fail(h, GS_ERR_ARG, "cluster: gpu_mem_cap_mib must be positive");
  return GS_OK;
}

extern "C" int gs_config_sim(gs_handle h, int sim, const gs_cluster *cluster, const gs_policy *policy) {
  if (!h) return GS_ERR_ARG;
  if (sim < 0 || sim >= h->nsims) return fail(h, GS_ERR_ARG, "gs_config_sim: sim index out of range");
  int rc = check_cluster(h, cluster);
  if (rc) return rc;
  SimHost &s = h->sims[(size_t)sim];
  if (s.prepared) return fail(h, GS_ERR_STATE, "gs_config_sim: replica already running");
  // validate into locals, commit only on success (a rejected call leaves the replica as it was)
  gs_policy pol;
  if (policy) pol = *policy; else { memset(&pol, 0, sizeof(pol)); pol.num_queue = 1; }
  if (pol.schedule < GS_SCHED_FIFO || pol.schedule > GS_SCHED_GITTINS)
    return fail(h, GS_ERR_ARG, "gs_config_sim: unknown schedule");
  if (pol.scheme != GS_SCHEME_YARN && pol.scheme != GS_SCHEME_COUNT)
    return fail(h, GS_ERR_ARG, "gs_config_sim: unknown scheme");
  if (pol.schedule == GS_SCHED_FIFO && pol.scheme != GS_SCHEME_YARN)
    return fail(h, GS_ERR_ARG, "gs_config_sim: fifo runs with the yarn scheme only");
  if (pol.schedule == GS_SCHED_FIFO &&
      ((long long)cluster->num_switch * cluster->num_node_p_switch * cluster->num_gpu_p_node > 65535 ||
       (long long)cluster->num_cpu_p_node / cluster->cpu_per_task > 32767))
    return fail(h, GS_ERR_ARG, "gs_config_sim: the fifo engine packs its counters for clusters of at most 65535 GPUs");
  if ((pol.schedule == GS_SCHED_DLAS || pol.schedule == GS_SCHED_DLAS_GPU) &&
      (pol.num_queue < 1 || pol.num_queue > GS_MAX_QUEUES))
    return fail(h, GS_ERR_ARG, "gs_config_sim: num_queue must be in 1..8 for dlas");
  void *git_dev = nullptr;
  long long git_direct_n = 0;
  if (pol.schedule == GS_SCHED_GITTINS) {
    if (pol.gittins_n < 1 || !pol.gittins_data || !pol.gittins_index)
      return fail(h, GS_ERR_ARG, "gs_config_sim: gittins needs the (data, index) tables");
    CU(cudaSetDevice(h->device));
    const size_t bytes = 8 * (size_t)pol.gittins_n;
    // direct form of the look-up "index of the first sample above a" for whole-number a (attained service always is one):
    // one entry per integer up to the largest sample, when that is not out of proportion with the table itself
    std::vector<double> direct;
    if (pol.gittins_n >= 2) {
      const double last = pol.gittins_data[pol.gittins_n - 2];
      if (last >= 0.0 && last < 8.0 * (double)pol.gittins_n + 65536.0 && last < 67108864.0) {
        direct.resize((size_t)last + 1);
        size_t idx = 0;
        for (size_t k = 0; k < direct.size(); ++k) {
          while (idx + 1 < (size_t)pol.gittins_n && !(pol.gittins_data[idx] > (double)k)) ++idx;
          direct[k] = pol.gittins_index[idx];
        }
      }
    }
    git_direct_n = (long long)direct.size();
    CU(cudaMalloc(&git_dev, 2 * bytes + 8 * direct.size()));
    cudaError_t e1 = cudaMemcpy(git_dev, pol.gittins_data, bytes, cudaMemcpyHostToDevice);
    cudaError_t e2 = cudaMemcpy((unsigned char *)git_dev + bytes, pol.gittins_index, bytes, cudaMemcpyHostToDevice);
    cudaError_t e3 = direct.empty() ? cudaSuccess : cudaMemcpy((unsigned char *)git_dev + 2 * bytes, direct.data(), 8 * direct.size(), cudaMemcpyHostToDevice);
    if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess) { cudaFree(git_dev); return fail(h, GS_ERR_CUDA, "gs_config_sim: gittins table upload failed"); }
  }
  if (s.git_dev) cudaFree(s.git_dev);
  s.git_dev = git_dev;
  s.git_direct_n = git_direct_n;
  s.cl = *cluster;
  s.pol = pol;
  s.pol.gittins_data = s.pol.gittins_index = nullptr;   // host pointers are not retained past this call
  s.loaded = false;       // load-time bounds (max_need, span_cap) depend on the cluster: a reconfigured replica needs its trace again
  s.configured = true;
  h->dirty = true;
  return GS_OK;
}

static int ensure_stage(gs_handle h, size_t bytes) {
  if (h->h_stage_bytes >= bytes) return GS_OK;
  if (h->h_stage) { cudaStreamSynchronize(h->stream); cudaFreeHost(h->h_stage); }
  h->h_stage = nullptr; h->h_stage_bytes = 0;
  CU(cudaMallocHost(&h->h_stage, bytes));
  h->h_stage_bytes = bytes;
  return GS_OK;
}

// Validation + load-time bounds over n packed records (read only).
static int scan_trace(gs_handle h, const SimHost &s, int64_t n, const JobIn *ji, bool net, const double *model_mb,
                      const double *iterations, int64_t *span_cap_out, double *max_need_out) {
  const int M = s.cl.num_switch * s.cl.num_node_p_switch;
  const bool netcost = net && s.cl.enable_network_costs;
  int64_t span_cap = 0;
  double max_need = 1.0;
  int prev = 0;
  for (int64_t j = 0; j < n; ++j) {
    const JobIn r = ji[j];
    if (r.arrive < prev) return fail(h, GS_ERR_ARG, "gs_load_trace: arrive_tick must be non-negative and non-decreasing");
    prev = r.arrive;
    if (r.gpc <= 0 || r.gpus < r.gpc || r.gpus % r.gpc != 0 || r.gpus >= (1 << 24) || r.gpc > 255)
      return fail(h, GS_ERR_ARG, "gs_load_trace: gpus must be a positive multiple of gpu_per_task below 2^24 (job.py:96-100)");
    if (r.memb < 0) return fail(h, GS_ERR_ARG, "gs_load_trace: negative mem_bytes");
    if (!(r.dur == r.dur)) return fail(h, GS_ERR_ARG, "gs_load_trace: NaN duration");
    const int64_t tasks = r.gpus / r.gpc;
    span_cap += tasks < M ? tasks : M;
    double d = r.dur;
    if (netcost && r.ps > 1) {
      const double cross = (double)(tasks < M ? tasks : M);
      const double extra = (model_mb[j] / s.cl.bandwidth + cross * s.cl.internode_latency) * (iterations[j] * 2.0);
      if (extra > 0) d += extra;
    }
    if (d > max_need) max_need = d;
  }
  *span_cap_out = span_cap; *max_need_out = max_need;
  return GS_OK;
}

static int load_common(gs_handle h, int sim, int64_t n, const JobIn *packed, const int32_t *arrive_tick,
                       const int32_t *gpus, const int32_t *gpu_per_task, const double *duration,
                       const int64_t *mem_bytes, const double *model_mb, const double *iterations,
                       const int32_t *ps_count) {
  if (!h) return GS_ERR_ARG;
  if (sim < 0 || sim >= h->nsims) return fail(h, GS_ERR_ARG, "gs_load_trace: sim index out of range");
  SimHost &s = h->sims[(size_t)sim];
  if (!s.configured) return fail(h, GS_ERR_STATE, "gs_load_trace: call gs_config_sim first");
  if (n < 0 || n >= (1ll << 31) - 64) return fail(h, GS_ERR_ARG, "gs_load_trace: n out of range");
  if (n > 0 && !packed && (!arrive_tick || !gpus || !gpu_per_task || !duration || !mem_bytes))
    return fail(h, GS_ERR_ARG, "gs_load_trace: NULL column");
  const bool net = model_mb && iterations && (packed || ps_count);
  CU(cudaSetDevice(h->device));
  const size_t N = (size_t)(n > 0 ? n : 1);
  const size_t off_model = align_up(sizeof(JobIn) * N), off_iters = align_up(off_model + (net ? 8 * N : 0));
  const size_t total = align_up(off_iters + (net ? 8 * N : 0));
  // asynchronous path: packed records in page-locked caller memory go to the device without staging
  bool direct = false;
  if (h->async && packed && !net && n > 0) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, packed) == cudaSuccess && at.type == cudaMemoryTypeHost) direct = true;
    else (void)cudaGetLastError();
  }
  const JobIn *ji = packed;
  if (!direct) {
    CU(cudaStreamSynchronize(h->stream));         // the staging buffer may still feed an earlier upload
    int rc = ensure_stage(h, total);
    if (rc) return rc;
    unsigned char *st = (unsigned char *)h->h_stage;
    JobIn *dst = (JobIn *)st;
    if (packed) memcpy(dst, packed, sizeof(JobIn) * (size_t)n);
    else
      for (int64_t j = 0; j < n; ++j) {
        JobIn r;
        r.arrive = arrive_tick[j]; r.gpus = gpus[j]; r.gpc = gpu_per_task[j]; r.ps = net ? ps_count[j] : 0;
        r.memb = mem_bytes[j]; r.dur = duration[j];
        dst[j] = r;
      }
    if (net && n > 0) {
      memcpy(st + off_model, model_mb, 8 * (size_t)n);
      memcpy(st + off_iters, iterations, 8 * (size_t)n);
    }
    ji = dst;
  }
  int64_t span_cap = 0;
  double max_need = 1.0;
  int rc = scan_trace(h, s, n, ji, net, model_mb, iterations, &span_cap, &max_need);
  if (rc) return rc;
  if (max_need > (double)(1 << 26)) return fail(h, GS_ERR_ARG, "gs_load_trace: job duration exceeds 2^26 ticks");
  if (s.trace_slab && s.trace_bytes < total) { CU(cudaStreamSynchronize(h->stream)); cudaFree(s.trace_slab); s.trace_slab = nullptr; }
  if (!s.trace_slab) { CU(cudaMalloc(&s.trace_slab, total)); s.trace_bytes = total; }
  if (direct) {
    CU(cudaMemcpyAsync(s.trace_slab, packed, sizeof(JobIn) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
  } else {
    CU(cudaEventRecord(h->e0, h->stream));
    CU(cudaMemcpyAsync(s.trace_slab, h->h_stage, total, cudaMemcpyHostToDevice, h->stream));
    CU(cudaEventRecord(h->e1, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    float ms = 0; cudaEventElapsedTime(&ms, h->e0, h->e1);
    h->h2d_ms += ms;
  }
  unsigned char *d = (unsigned char *)s.trace_slab;
  SimDev &D = s.dev;
  memset(&D, 0, sizeof(D));
  D.jobs = (const JobIn *)d;
  D.model_mb = net ? (const double *)(d + off_model) : nullptr;
  D.iters = net ? (const double *)(d + off_iters) : nullptr;
  if (h->span_budget > 0) {
    const int64_t lim = (int64_t)(h->span_budget * (double)n) + 4096;
    if (span_cap > lim) span_cap = lim;
  }
  s.n = n; s.span_cap = span_cap > 0 ? span_cap : 1;
  s.max_need = (int)max_need + 2;
  s.last_arrive = n > 0 ? ji[n - 1].arrive : 0;
  s.loaded = true;
  s.trace_in_arena = false;
  s.prepared = false;      // (re)loading a trace restarts the replica; slabs are reused when big enough
  h->dirty = true;
  return GS_OK;
}

extern "C" int gs_load_trace(gs_handle h, int sim, int64_t n, const int32_t *arrive_tick, const int32_t *gpus,
                             const int32_t *gpu_per_task, const double *duration, const int64_t *mem_bytes,
                             const double *model_mb, const double *iterations, const int32_t *ps_count) {
  return load_common(h, sim, n, nullptr, arrive_tick, gpus, gpu_per_task, duration, mem_bytes, model_mb, iterations, ps_count);
}

// Same trace, already packed as 32-byte gs_jobin records (saves the column gather on the host).
extern "C" int gs_load_trace_packed(gs_handle h, int sim, int64_t n, const gs_jobin *jobs, const double *model_mb,
                                    const double *iterations) {
  static_assert(sizeof(gs_jobin) == sizeof(JobIn), "gs_jobin layout");
  if (n > 0 && !jobs) return fail(h, GS_ERR_ARG, "gs_load_trace_packed: NULL records");
  return load_common(h, sim, n, reinterpret_cast<const JobIn *>(jobs), nullptr, nullptr, nullptr, nullptr, nullptr,
                     model_mb, iterations, nullptr);
}

static SimLayout layout_sim(gs_handle h, const SimHost &s, int64_t rows_cap) {
  SimLayout L;
  const gs_cluster &c = s.cl;
  const int M = c.num_switch * c.num_node_p_switch;
  const size_t N = (size_t)(s.n > 0 ? s.n : 1);
  int W = 256; while (W < s.max_need + 1) W <<= 1;
  L.W = W;
  if (rows_cap <= 0) rows_cap = s.last_arrive + 2ll * s.max_need + 4096;
  L.rows_cap = rows_cap;
  L.qrows_cap = h->qrows_cap > 0 ? h->qrows_cap : rows_cap;
  const bool evd = s.pol.schedule != GS_SCHED_FIFO;        // event-driven policy: rows + extra scratch
  const bool net = c.enable_network_costs != 0;
  size_t total = 0;
  auto take = [&](size_t bytes) { const size_t o = total; total = align_up(total + bytes); return o; };
  if (evd) {
    L.o_fin = take(4 * N);
    L.o_rec = take(sizeof(gs_job_rec) * N);
    L.o_rows = take(sizeof(gs_tick_row) * (size_t)rows_cap);
    L.out_bytes = total;
    const size_t nql = (size_t)(s.pol.num_queue > 2 ? s.pol.num_queue : 2);
    L.o_pj = take(sizeof(PJob) * N); L.o_run = take(4 * N); L.o_qs = take(4 * N * nql); L.o_end = take(4 * N);
    L.o_tmp = take(4 * N); L.o_ci = take(4 * (size_t)M); L.o_ck = take(4 * (size_t)M); L.o_stale = take(4 * N);
  } else {
    L.o_ev = take(sizeof(gs_evrow) * (size_t)rows_cap);
    L.o_q = take(sizeof(gs_qrow) * (size_t)L.qrows_cap);
    L.o_ne = take(sizeof(gs_nodeev) * (size_t)(M + 2));          // at most one event per node + one per window
    L.o_rec2 = take(4 * N);
    if (net) L.o_dur2 = take(8 * N);
    L.o_fin = take(4 * N);
    L.o_spans = take((c.num_gpu_p_node > 32 ? sizeof(gs_span) : sizeof(gs_cspan)) * (size_t)s.span_cap);
    L.out_bytes = total;
    L.o_jst = take(sizeof(JobState2) * N);
    L.o_stack = take(8 * (N + 1));
    L.o_wh = take(4 * (size_t)W); L.o_wm = take(8 * (size_t)W);
    L.o_nb = take(8 * (size_t)M); L.o_nk = take(4 * (size_t)M);
  }
  L.total = total;
  return L;
}

static int bind_sim(gs_handle h, SimHost &s, const SimLayout &L, unsigned char *d) {
  const gs_cluster &c = s.cl;
  const int M = c.num_switch * c.num_node_p_switch;
  const int W = L.W;
  const int64_t rows_cap = L.rows_cap, qrows_cap = L.qrows_cap;
  const bool evd = s.pol.schedule != GS_SCHED_FIFO;
  const bool net = c.enable_network_costs != 0;
  const size_t o_fin = L.o_fin, o_rec = L.o_rec, o_rows = L.o_rows, o_rec2 = L.o_rec2, o_dur2 = L.o_dur2, o_jst = L.o_jst, o_stack = L.o_stack;
  const size_t o_wh = L.o_wh, o_wm = L.o_wm, o_spans = L.o_spans, o_ev = L.o_ev, o_q = L.o_q, o_nb = L.o_nb, o_nk = L.o_nk;
  const size_t o_pj = L.o_pj, o_run = L.o_run, o_qs = L.o_qs, o_end = L.o_end, o_tmp = L.o_tmp, o_ci = L.o_ci, o_ck = L.o_ck, o_stale = L.o_stale;
  s.layout = L;
  s.state_ptr = d;
  SimDev &D = s.dev;
  D.M = M; D.G = c.num_gpu_p_node;
  int kc = c.num_cpu_p_node / c.cpu_per_task, km = c.mem_p_node / c.mem_per_task;
  D.K = kc < km ? kc : km;
  D.netcost = net ? 1 : 0;
  D.n = (int)s.n; D.wheel_mask = W - 1; D.policy = s.pol.schedule;
  D.cap_bytes = (long long)c.gpu_mem_cap_mib << 20;
  D.fit_limit = D.cap_bytes - ((long long)500 << 20);      // cap - mem > 500 MiB  (device.py:75)
  D.bandwidth = c.bandwidth; D.latency = c.internode_latency;
  D.fin = (int *)(d + o_fin);
  D.rec = nullptr; D.rows = nullptr; D.jstart = nullptr; D.dur2 = nullptr; D.jst2 = nullptr; D.stack = nullptr;
  D.wheel_head = nullptr; D.wheel_mem = nullptr; D.spans = nullptr; D.evrows = nullptr; D.qrows = nullptr; D.nodeev = nullptr; D.nbusy = nullptr; D.nk = nullptr;
  if (evd) {
    D.rec = (gs_job_rec *)(d + o_rec); D.rows = (gs_tick_row *)(d + o_rows);
  } else {
    D.jstart = (int *)(d + o_rec2); D.dur2 = net ? (double *)(d + o_dur2) : nullptr;
    D.jst2 = (JobState2 *)(d + o_jst); D.stack = (int *)(d + o_stack);
    D.wheel_head = (int *)(d + o_wh); D.wheel_mem = (long long *)(d + o_wm);
    D.spans = (void *)(d + o_spans); D.evrows = (gs_evrow *)(d + o_ev); D.qrows = (gs_qrow *)(d + o_q); D.nodeev = (gs_nodeev *)(d + L.o_ne);
    D.nbusy = (unsigned long long *)(d + o_nb); D.nk = (int *)(d + o_nk);
  }
  D.span_cap = s.span_cap; D.rows_cap = rows_cap; D.qrows_cap = qrows_cap;
  s.rows_cap = rows_cap; s.qrows_cap = qrows_cap;
  if (evd) {
    D.pj = (PJob *)(d + o_pj); D.runnable = (int *)(d + o_run); D.queues = (int *)(d + o_qs);
    D.endj = (int *)(d + o_end); D.tmpl = (int *)(d + o_tmp); D.cidle = (int *)(d + o_ci); D.ckfree = (int *)(d + o_ck);
    D.stalej = (int *)(d + o_stale); D.stale_n = 0;
    D.num_queue = s.pol.num_queue > 0 ? s.pol.num_queue : 1;
    for (int q = 0; q < GS_MAX_QUEUES; ++q) { D.queue_limit[q] = s.pol.queue_limit[q]; D.qn[q] = 0; }
    D.gittins_delta = s.pol.gittins_delta; D.next_gittins_unit = s.pol.gittins_delta;
    D.git_n = s.pol.schedule == GS_SCHED_GITTINS ? s.pol.gittins_n : 0;
    D.git_data = (const double *)s.git_dev;
    D.git_index = s.git_dev ? (const double *)((unsigned char *)s.git_dev + 8 * (size_t)s.pol.gittins_n) : nullptr;
    D.git_direct_n = (s.git_dev && D.git_n > 0) ? s.git_direct_n : 0;
    D.git_direct = D.git_direct_n > 0 ? (const double *)((unsigned char *)s.git_dev + 16 * (size_t)s.pol.gittins_n) : nullptr;
    D.rn = 0; D.en = 0; D.end_time = 0x7fffffff; D.next_job_jump = 0x7fffffff;
  }
  D.comm_n = 0; D.comm_rank = 0; D.comm_cap = 0; D.comm_rk_in = nullptr; D.comm_flags = nullptr; D.comm_epoch = 0; D.comm_wait_cycles = 0;
  if (h->comm_n > 1 && s.pol.schedule == GS_SCHED_GITTINS) {
    if ((int64_t)s.n > h->comm_cap) return fail(h, GS_ERR_ARG, "gs_run: the trace has more jobs than gs_comm_prepare sized the exchange buffer for");
    // the event counter never restarts: a new run continues where the last one ended (all ranks execute the same
    // events, so their counters agree), which needs no reset of the flag words and no extra synchronisation
    D.comm_epoch = h->comm_epoch; h->comm_epoch0 = h->comm_epoch;
    D.comm_n = h->comm_n; D.comm_rank = h->comm_rank; D.comm_cap = h->comm_cap; D.comm_min_runnable = h->comm_min_runnable;
    D.comm_flags = (unsigned long long *)h->comm_buf;
    D.comm_rk_in = (double *)((unsigned char *)h->comm_buf + 256);
    for (int q = 0; q < h->comm_n; ++q) {
      D.comm_peer_flags[q] = (unsigned long long *)h->comm_peer[q];
      D.comm_peer_rk[q] = (double *)((unsigned char *)h->comm_peer[q] + 256);
    }
  }
  D.delta = D.p = D.top = D.running = D.finished = D.ever = D.busy_gpus = D.done = D.status = 0;
  D.blocked = D.nev = D.nq = D.nne = 0;
  D.mem_busy = D.sum_arr = D.span_used = D.events = D.evals = D.started = D.ticks = D.row_first = 0;
  D.need_init = 1;
  s.sum_rows = 0; s.sum_fresh = true;
  s.tl_fresh = true; s.tl_done = false; s.jd_done = false; s.sd_done = false; s.arr_done = false;
  s.occ_fresh = true; s.occ_done = false;
  s.prepared = true;
  return GS_OK;
}

extern "C" int gs_run(gs_handle h, int64_t max_ticks, int64_t rows_cap) {
  if (!h) return GS_ERR_ARG;
  CU(cudaSetDevice(h->device));
  int maxM = 1;
  bool none_prepared = true;
  for (auto &s : h->sims) {
    if (!s.loaded) return fail(h, GS_ERR_STATE, "gs_run: every replica needs gs_config_sim + gs_load_trace");
    none_prepared &= !s.prepared;
    int M = s.cl.num_switch * s.cl.num_node_p_switch;
    if (M > maxM) maxM = M;
  }
  if (none_prepared) {
    // a fresh start of every replica (the common case): the slabs go side by side into one arena with one stride
    std::vector<SimLayout> Ls((size_t)h->nsims);
    size_t stride = 0;
    for (int i = 0; i < h->nsims; ++i) { Ls[(size_t)i] = layout_sim(h, h->sims[(size_t)i], rows_cap); stride = std::max(stride, Ls[(size_t)i].total); }
    stride = align_up(stride, 512);
    const size_t need = stride * (size_t)h->nsims;
    if (h->arena_bytes < need) {
      CU(cudaStreamSynchronize(h->stream));
      if (h->arena) cudaFree(h->arena);
      h->arena = nullptr; h->arena_bytes = 0;
      CU(cudaMalloc(&h->arena, need));
      h->arena_bytes = need;
    }
    h->arena_stride = stride;
    for (int i = 0; i < h->nsims; ++i) {
      int rc = bind_sim(h, h->sims[(size_t)i], Ls[(size_t)i], (unsigned char *)h->arena + stride * (size_t)i);
      if (rc) return rc;
    }
    h->dirty = true;
  } else {
    for (auto &s : h->sims)
      if (!s.prepared) {   // one replica restarts while others keep running: it gets (or keeps) its own allocation
        const SimLayout L = layout_sim(h, s, rows_cap);
        if (s.state_slab && s.state_bytes < L.total) { CU(cudaStreamSynchronize(h->stream)); cudaFree(s.state_slab); s.state_slab = nullptr; }
        if (!s.state_slab) { CU(cudaMalloc(&s.state_slab, L.total)); s.state_bytes = L.total; }
        int rc = bind_sim(h, s, L, (unsigned char *)s.state_slab);
        if (rc) return rc;
        h->dirty = true;
      }
  }
  bool fifo_kind[4] = {false, false, false, false};   // [network costs][more than 32 GPUs per node]
  bool any_evd = false, evd_init = false;
  for (auto &s : h->sims) {
    if (s.pol.schedule == GS_SCHED_FIFO) fifo_kind[(s.cl.enable_network_costs ? 2 : 0) + (s.cl.num_gpu_p_node > 32 ? 1 : 0)] = true;
    else { any_evd = true; evd_init |= s.dev.need_init != 0; }
  }
  if (h->dirty) {
    for (int i = 0; i < h->nsims; ++i) h->h_back[(size_t)i] = h->sims[(size_t)i].dev;
    CU(cudaMemcpyAsync(h->d_sims, h->h_back.data(), sizeof(SimDev) * (size_t)h->nsims, cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->dirty = false;
  }
  CU(cudaEventRecord(h->e0, h->stream));
  if (any_evd) {
    if (evd_init) {      // state reset is part of the timed engine work
      gs_init_kernel<<<dim3(16, (unsigned)h->nsims), 256, 0, h->stream>>>(h->d_sims, h->nsims);
      CU(cudaGetLastError());
      h->launches += 1;
    }
    // engine mode 2: one thread per replica (first version); default: one warp per replica
    const int thread_map = h->engine_mode == 2 ? 1 : 0;
    if (thread_map) {
      gs_policy_kernel<<<(unsigned)((h->nsims + 31) / 32), 32, 0, h->stream>>>(h->d_sims, h->nsims, (long long)max_ticks, 1);
      CU(cudaGetLastError());
      h->launches += 1;
    } else {
      gs_dlas_warp_kernel<<<(unsigned)h->nsims, 32, 0, h->stream>>>(h->d_sims, h->nsims, (long long)max_ticks);
      CU(cudaGetLastError());
      const size_t pol_smem = 8 * (size_t)maxM;
      if (pol_smem > 48 * 1024)
        CU(cudaFuncSetAttribute(gs_sortpol_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pol_smem));
      gs_sortpol_warp_kernel<<<(unsigned)h->nsims, 32, pol_smem, h->stream>>>(h->d_sims, h->nsims, (long long)max_ticks);
      CU(cudaGetLastError());
      h->launches += 2;
    }
  }
  if (fifo_kind[0] || fifo_kind[1] || fifo_kind[2] || fifo_kind[3]) {
    const int stride = (int)align_up((size_t)maxM * 12 + 8 + SCACHE * 8, 16);
    if (stride > 200 * 1024) return fail(h, GS_ERR_ARG, "gs_run: node table does not fit shared memory (M too large)");
    // one instantiation per (network costs, mask width); each skips the replicas of the other kinds
#define GS_LAUNCH_TICK2(NET_, G64_)                                                                                              \
    do {                                                                                                                         \
      if (stride > 48 * 1024) CU(cudaFuncSetAttribute(gs_tick2_kernel<NET_, G64_>, cudaFuncAttributeMaxDynamicSharedMemorySize, stride)); \
      gs_tick2_kernel<NET_, G64_><<<(unsigned)h->nsims, 32, (size_t)stride, h->stream>>>(h->d_sims, h->nsims, (long long)max_ticks, stride); \
      CU(cudaGetLastError());                                                                                                    \
      h->launches += 1;                                                                                                          \
    } while (0)
    if (fifo_kind[0]) GS_LAUNCH_TICK2(false, false);
    if (fifo_kind[1]) GS_LAUNCH_TICK2(false, true);
    if (fifo_kind[2]) GS_LAUNCH_TICK2(true, false);
    if (fifo_kind[3]) GS_LAUNCH_TICK2(true, true);
#undef GS_LAUNCH_TICK2
  }
  CU(cudaEventRecord(h->e1, h->stream));
  CU(cudaMemcpyAsync(h->h_back.data(), h->d_sims, sizeof(SimDev) * (size_t)h->nsims, cudaMemcpyDeviceToHost, h->stream));
  CU(wait_stream(h));
  float ms = 0; cudaEventElapsedTime(&ms, h->e0, h->e1);
  h->kernel_ms += ms;
  if (h->comm_n > 1 && h->h_back[0].comm_n > 1) h->comm_epoch = h->h_back[0].comm_epoch;
  int worst = 0;
  for (int i = 0; i < h->nsims; ++i) {
    h->h_back[(size_t)i].need_init = 0;
    h->sims[(size_t)i].dev = h->h_back[(size_t)i];
    if (h->h_back[(size_t)i].status != 0 && worst == 0) worst = h->h_back[(size_t)i].status;
  }
  if (worst != 0) return fail(h, worst, "gs_run: a replica stopped with an in-kernel error (see gs_stats.status)");
  return GS_OK;
}

extern "C" int gs_stats(gs_handle h, int sim, gs_run_stats *out) {
  if (!h || !out) return GS_ERR_ARG;
  if (sim < 0 || sim >= h->nsims) return fail(h, GS_ERR_ARG, "gs_stats: sim index out of range");
  const SimDev &D = h->sims[(size_t)sim].dev;
  memset(out, 0, sizeof(*out));
  out->ticks = D.ticks; out->events = D.events; out->finished = D.finished; out->started = D.started;
  out->placement_evals = D.evals; out->done = D.done; out->status = D.status;
  out->kernel_ms = h->kernel_ms; out->h2d_ms = h->h2d_ms; out->d2h_ms = h->d2h_ms;
  return GS_OK;
}

extern "C" int gs_window(gs_handle h, int sim, gs_window_info *out) {
  if (!h || !out) return GS_ERR_ARG;
  if (sim < 0 || sim >= h->nsims) return fail(h, GS_ERR_ARG, "gs_window: sim index out of range");
  const SimHost &s = h->sims[(size_t)sim];
  if (!s.prepared) return fail(h, GS_ERR_STATE, "gs_window: nothing has run yet");
  const SimDev &D = s.dev;
  out->row_first = D.row_first; out->ticks = D.ticks;
  const bool fifo = s.pol.schedule == GS_SCHED_FIFO;
  out->ev_rows = fifo ? D.nev : 0; out->q_rows = fifo ? D.nq : 0; out->node_events = fifo ? D.nne : 0;
  out->spans_used = D.span_used; out->admitted = D.p; out->finished = D.finished; out->n = s.n;
  return GS_OK;
}

extern "C" int gs_comm_prepare(gs_handle h, int64_t max_jobs, gs_comm_handle *out) {
  if (!h || !out || max_jobs < 1) return fail(h, GS_ERR_ARG, "gs_comm_prepare: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) <= sizeof(gs_comm_handle), "IPC handle size");
  if (h->nsims != 1) return fail(h, GS_ERR_ARG, "gs_comm_prepare: a sharded simulation needs a handle with exactly one replica");
  if (h->comm_n > 0) return fail(h, GS_ERR_STATE, "gs_comm_prepare: already initialised");
  CU(cudaSetDevice(h->device));
  if (h->comm_buf) { cudaFree(h->comm_buf); h->comm_buf = nullptr; }
  const size_t bytes = 256 + 2 * 8 * (size_t)max_jobs;
  CU(cudaMalloc(&h->comm_buf, bytes));
  CU(cudaMemset(h->comm_buf, 0, bytes));
  h->comm_cap = max_jobs;
  cudaIpcMemHandle_t ih;
  CU(cudaIpcGetMemHandle(&ih, h->comm_buf));
  memset(out, 0, sizeof(*out));
  memcpy(out->bytes, &ih, sizeof(ih));
  return GS_OK;
}

extern "C" int gs_comm_init(gs_handle h, int rank, int nranks, const gs_comm_handle *all) {
  if (!h || !all || nranks < 1 || nranks > GS_MAX_RANKS || rank < 0 || rank >= nranks)
    return fail(h, GS_ERR_ARG, "gs_comm_init: bad arguments (1 <= nranks <= 8)");
  if (!h->comm_buf) return fail(h, GS_ERR_STATE, "gs_comm_init: call gs_comm_prepare first");
  if (h->comm_n > 0) return fail(h, GS_ERR_STATE, "gs_comm_init: already initialised");
  CU(cudaSetDevice(h->device));
  for (int q = 0; q < nranks; ++q) {
    if (q == rank) { h->comm_peer[q] = h->comm_buf; h->comm_opened[q] = false; continue; }
    cudaIpcMemHandle_t ih;
    memcpy(&ih, all[q].bytes, sizeof(ih));
    void *ptr = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&ptr, ih, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      for (int r = 0; r < q; ++r) if (h->comm_opened[r]) { cudaIpcCloseMemHandle(h->comm_peer[r]); h->comm_opened[r] = false; h->comm_peer[r] = nullptr; }
      return fail(h, GS_ERR_COMM, std::string("gs_comm_init: cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
    }
    h->comm_peer[q] = ptr; h->comm_opened[q] = true;
  }
  h->comm_rank = rank; h->comm_n = nranks;
  for (auto &s : h->sims) s.prepared = false;
  h->dirty = true;
  return GS_OK;
}

// Events whose runnable list has at most `k` entries are evaluated by every rank itself (identical state, identical
// result, nothing to send); longer lists are split and exchanged.  k = 0: exchange on every event.  Must be the same on
// every rank; takes effect for replicas prepared afterwards.
extern "C" int gs_comm_set_min_runnable(gs_handle h, int k) {
  if (!h) return GS_ERR_ARG;
  if (k < 0) return fail(h, GS_ERR_ARG, "gs_comm_set_min_runnable: must be >= 0");
  h->comm_min_runnable = k;
  for (auto &s : h->sims) s.prepared = false;
  h->dirty = true;
  return GS_OK;
}

extern "C" int gs_comm_stats(gs_handle h, int64_t *exchanges, double *mean_us) {
  if (!h) return GS_ERR_ARG;
  const SimDev &D = h->sims[0].dev;
  int khz = 0;
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, h->device);
  const unsigned long long done = D.comm_n > 1 ? D.comm_epoch - h->comm_epoch0 : 0ull;
  if (exchanges) *exchanges = (int64_t)done;
  if (mean_us) *mean_us = (done > 0 && khz > 0) ? (double)D.comm_wait_cycles / (double)done / ((double)khz / 1000.0) : 0.0;
  return GS_OK;
}

extern "C" int gs_sync(gs_handle h) {
  if (!h) return GS_ERR_ARG;
  CU(cudaSetDevice(h->device));
  CU(wait_stream(h));
  return GS_OK;
}

extern "C" int gs_set_async(gs_handle h, int on) {
  if (!h) return GS_ERR_ARG;
  h->async = on != 0;
  return GS_OK;
}

extern "C" int gs_set_queue_rows_cap(gs_handle h, int64_t qrows_cap) {
  if (!h) return GS_ERR_ARG;
  if (qrows_cap < 0) return fail(h, GS_ERR_ARG, "gs_set_queue_rows_cap: must be >= 0");
  h->qrows_cap = qrows_cap;
  return GS_OK;
}

extern "C" int gs_fetch_compact(gs_handle h, int sim, gs_evrow *ev_out, gs_qrow *q_out, gs_nodeev *nodeev_out, gs_job_start *jobs_out,
                                double *duration_out, int32_t *finish_order_out, void *spans_out) {
  if (!h) return GS_ERR_ARG;
  if (sim < 0 || sim >= h->nsims) return fail(h, GS_ERR_ARG, "gs_fetch_compact: sim index out of range");
  SimHost &s = h->sims[(size_t)sim];
  if (!s.prepared) return fail(h, GS_ERR_STATE, "gs_fetch_compact: nothing has run yet");
  if (s.pol.schedule != GS_SCHED_FIFO) return fail(h, GS_ERR_ARG, "gs_fetch_compact: the compact records are the fifo engine's output");
  static_assert(sizeof(gs_evrow) == 24 && sizeof(gs_qrow) == 24 && sizeof(gs_nodeev) == 8 && sizeof(gs_job_start) == 4 && sizeof(gs_cspan) == 8,
                "compact record layout");
  const size_t span_bytes = s.cl.num_gpu_p_node > 32 ? sizeof(gs_span) : sizeof(gs_cspan);
  const SimDev &D = s.dev;
  CU(cudaSetDevice(h->device));
  if (ev_out && D.nev > 0) CU(cudaMemcpyAsync(ev_out, D.evrows, sizeof(gs_evrow) * (size_t)D.nev, cudaMemcpyDeviceToHost, h->stream));
  if (q_out && D.nq > 0) CU(cudaMemcpyAsync(q_out, D.qrows, sizeof(gs_qrow) * (size_t)D.nq, cudaMemcpyDeviceToHost, h->stream));
  if (nodeev_out && D.nne > 0) CU(cudaMemcpyAsync(nodeev_out, D.nodeev, sizeof(gs_nodeev) * (size_t)D.nne, cudaMemcpyDeviceToHost, h->stream));
  if (jobs_out && s.n > 0) CU(cudaMemcpyAsync(jobs_out, D.jstart, 4 * (size_t)s.n, cudaMemcpyDeviceToHost, h->stream));
  if (duration_out && D.dur2 && s.n > 0) CU(cudaMemcpyAsync(duration_out, D.dur2, 8 * (size_t)s.n, cudaMemcpyDeviceToHost, h->stream));
  if (finish_order_out && D.finished > 0) CU(cudaMemcpyAsync(finish_order_out, D.fin, 4 * (size_t)D.finished, cudaMemcpyDeviceToHost, h->stream));
  if (spans_out && D.span_used > 0) CU(cudaMemcpyAsync(spans_out, D.spans, span_bytes * (size_t)D.span_used, cudaMemcpyDeviceToHost, h->stream));
  return GS_OK;
}

// The trace arena holds the traces of all replicas side by side, one stride apart (gs_load_traces_packed,
// gs_boot_traces).  reserve_trace_arena makes room for traces of up to nmax records each (h->tarena_stride);
// bind_arena_trace then points replica i at its slot: loaded, not prepared, the span budget applied.
static int reserve_trace_arena(gs_handle h, int64_t nmax) {
  const size_t stride = align_up(sizeof(JobIn) * (size_t)nmax, 512);
  const size_t need = stride * (size_t)h->nsims;
  CU(wait_stream(h));                                   // earlier work may still read the old traces
  if (h->tarena_bytes < need) {
    if (h->tarena) cudaFree(h->tarena);
    h->tarena = nullptr; h->tarena_bytes = 0;
    CU(cudaMalloc(&h->tarena, need));
    h->tarena_bytes = need;
  }
  h->tarena_stride = stride;
  return GS_OK;
}

static void bind_arena_trace(gs_handle h, int i, int64_t n, int64_t span_cap, double max_need, int64_t last_arrive) {
  SimHost &s = h->sims[(size_t)i];
  SimDev &D = s.dev;
  memset(&D, 0, sizeof(D));
  D.jobs = (const JobIn *)((unsigned char *)h->tarena + h->tarena_stride * (size_t)i);
  if (h->span_budget > 0) { const int64_t lim = (int64_t)(h->span_budget * (double)n) + 4096; if (span_cap > lim) span_cap = lim; }
  s.n = n; s.span_cap = span_cap > 0 ? span_cap : 1;
  s.max_need = (int)max_need + 2;
  s.last_arrive = last_arrive;
  s.loaded = true; s.prepared = false; s.trace_in_arena = true;
}

// Every replica of the handle at once, from ONE host block (record i*pitch_bytes is the trace of replica i): the traces
// go into a device arena with one stride and travel as a single strided copy.  With gs_set_async and a page-locked
// block nothing is staged and the call returns before the copy completes (keep the block until gs_run / gs_sync).
extern "C" int gs_load_traces_packed(gs_handle h, const gs_jobin *jobs, size_t pitch_bytes, const int64_t *n_each) {
  if (!h) return GS_ERR_ARG;
  if (!jobs || !n_each || pitch_bytes % sizeof(JobIn) != 0) return fail(h, GS_ERR_ARG, "gs_load_traces_packed: bad arguments (pitch must be a multiple of 32)");
  CU(cudaSetDevice(h->device));
  int64_t nmax = 1;
  for (int i = 0; i < h->nsims; ++i) {
    const SimHost &s = h->sims[(size_t)i];
    if (!s.configured) return fail(h, GS_ERR_STATE, "gs_load_traces_packed: call gs_config_sim for every replica first");
    if (s.cl.enable_network_costs) return fail(h, GS_ERR_ARG, "gs_load_traces_packed: traces with network columns go through gs_load_trace");
    if (n_each[i] < 0 || n_each[i] >= (1ll << 31) - 64 || (size_t)n_each[i] * sizeof(JobIn) > pitch_bytes)
      return fail(h, GS_ERR_ARG, "gs_load_traces_packed: a trace does not fit the pitch");
    nmax = std::max(nmax, n_each[i]);
  }
  // validate first (read only); nothing changes if a trace is rejected
  std::vector<int64_t> span_cap((size_t)h->nsims); std::vector<double> max_need((size_t)h->nsims);
  for (int i = 0; i < h->nsims; ++i) {
    const JobIn *ji = reinterpret_cast<const JobIn *>(reinterpret_cast<const unsigned char *>(jobs) + pitch_bytes * (size_t)i);
    int rc = scan_trace(h, h->sims[(size_t)i], n_each[i], ji, false, nullptr, nullptr, &span_cap[(size_t)i], &max_need[(size_t)i]);
    if (rc) return rc;
    if (max_need[(size_t)i] > (double)(1 << 26)) return fail(h, GS_ERR_ARG, "gs_load_trace: job duration exceeds 2^26 ticks");
  }
  int rc = reserve_trace_arena(h, nmax);
  if (rc) return rc;
  const size_t stride = h->tarena_stride;
  bool direct = false;
  if (h->async) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, jobs) == cudaSuccess && at.type == cudaMemoryTypeHost) direct = true;
    else (void)cudaGetLastError();
  }
  const void *src = jobs;
  if (!direct) {
    rc = ensure_stage(h, pitch_bytes * (size_t)h->nsims);
    if (rc) return rc;
    memcpy(h->h_stage, jobs, pitch_bytes * (size_t)h->nsims);
    src = h->h_stage;
  }
  CU(cudaEventRecord(h->e0, h->stream));
  CU(cudaMemcpy2DAsync(h->tarena, stride, src, pitch_bytes, sizeof(JobIn) * (size_t)nmax, (size_t)h->nsims, cudaMemcpyHostToDevice, h->stream));
  CU(cudaEventRecord(h->e1, h->stream));
  if (!direct) {
    CU(cudaStreamSynchronize(h->stream));
    float ms = 0; cudaEventElapsedTime(&ms, h->e0, h->e1);
    h->h2d_ms += ms;
  }
  for (int i = 0; i < h->nsims; ++i) {
    const JobIn *ji = reinterpret_cast<const JobIn *>(reinterpret_cast<const unsigned char *>(jobs) + pitch_bytes * (size_t)i);
    bind_arena_trace(h, i, n_each[i], span_cap[(size_t)i], max_need[(size_t)i], n_each[i] > 0 ? ji[n_each[i] - 1].arrive : 0);
  }
  h->dirty = true;
  return GS_OK;
}

// Where the results of a replica lie inside its result block, and how the blocks of the handle are spaced.
extern "C" int gs_result_layout(gs_handle h, int sim, gs_result_layout_t *out) {
  if (!h || !out) return GS_ERR_ARG;
  if (sim < 0 || sim >= h->nsims) return fail(h, GS_ERR_ARG, "gs_result_layout: sim index out of range");
  const SimHost &s = h->sims[(size_t)sim];
  if (!s.prepared) return fail(h, GS_ERR_STATE, "gs_result_layout: nothing has run yet");
  if (s.pol.schedule != GS_SCHED_FIFO) return fail(h, GS_ERR_ARG, "gs_result_layout: the compact records are the fifo engine's output");
  const SimLayout &L = s.layout;
  memset(out, 0, sizeof(*out));
  out->block_bytes = (int64_t)L.out_bytes;
  out->off_ev = (int64_t)L.o_ev; out->off_q = (int64_t)L.o_q; out->off_nodeev = (int64_t)L.o_ne; out->off_jobs = (int64_t)L.o_rec2;
  out->cap_nodeev = (int64_t)s.cl.num_switch * s.cl.num_node_p_switch + 2;
  out->off_duration = s.cl.enable_network_costs ? (int64_t)L.o_dur2 : -1;
  out->off_finish_order = (int64_t)L.o_fin; out->off_spans = (int64_t)L.o_spans;
  out->cap_ev = L.rows_cap; out->cap_q = L.qrows_cap; out->cap_spans = s.span_cap; out->n = s.n;
  out->span_bytes = s.cl.num_gpu_p_node > 32 ? (int64_t)sizeof(gs_span) : (int64_t)sizeof(gs_cspan);
  return GS_OK;
}

// The result blocks of replicas [first, first + count) in one strided copy (asynchronous: gs_sync waits).  Row i of
// `out` (out_pitch bytes apart) receives the first block_bytes bytes of replica first + i's block.
extern "C" int gs_fetch_results(gs_handle h, int first, int count, void *out, size_t out_pitch) {
  if (!h) return GS_ERR_ARG;
  if (first < 0 || count < 0 || first + count > h->nsims || (count > 0 && !out)) return fail(h, GS_ERR_ARG, "gs_fetch_results: bad arguments");
  if (count == 0) return GS_OK;
  CU(cudaSetDevice(h->device));
  size_t width = 0;
  bool in_arena = true;
  for (int i = first; i < first + count; ++i) {
    const SimHost &s = h->sims[(size_t)i];
    if (!s.prepared) return fail(h, GS_ERR_STATE, "gs_fetch_results: nothing has run yet");
    if (s.pol.schedule != GS_SCHED_FIFO) return fail(h, GS_ERR_ARG, "gs_fetch_results: the compact records are the fifo engine's output");
    width = std::max(width, s.layout.out_bytes);
    in_arena &= s.state_ptr == (unsigned char *)h->arena + h->arena_stride * (size_t)i;
  }
  if (width > out_pitch) return fail(h, GS_ERR_CAPACITY, "gs_fetch_results: out_pitch is smaller than a result block");
  if (in_arena) {
    CU(cudaMemcpy2DAsync(out, out_pitch, (unsigned char *)h->arena + h->arena_stride * (size_t)first, h->arena_stride, width, (size_t)count,
                         cudaMemcpyDeviceToHost, h->stream));
  } else {
    for (int i = first; i < first + count; ++i)
      CU(cudaMemcpyAsync((unsigned char *)out + out_pitch * (size_t)(i - first), h->sims[(size_t)i].state_ptr, h->sims[(size_t)i].layout.out_bytes,
                         cudaMemcpyDeviceToHost, h->stream));
  }
  return GS_OK;
}

static int ensure_scratch(gs_handle h, size_t bytes) {
  if (h->d_scratch_bytes >= bytes) return GS_OK;
  if (h->d_scratch) { cudaStreamSynchronize(h->stream); cudaFree(h->d_scratch); }
  h->d_scratch = nullptr; h->d_scratch_bytes = 0;
  CU(cudaMalloc(&h->d_scratch, bytes));
  h->d_scratch_bytes = bytes;
  return GS_OK;
}

static int timed_d2h(gs_handle h, void *dst, const void *src, size_t bytes) {
  if (bytes == 0) return GS_OK;
  CU(cudaEventRecord(h->e0, h->stream));
  CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaEventRecord(h->e1, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  float ms = 0; cudaEventElapsedTime(&ms, h->e0, h->e1);
  h->d2h_ms += ms;
  return GS_OK;
}

extern "C" int gs_fetch_rows(gs_handle h, int sim, int64_t first, int64_t count, gs_tick_row *rows_out) {
  if (!h) return GS_ERR_ARG;
  if (sim < 0 || sim >= h->nsims) return fail(h, GS_ERR_ARG, "gs_fetch_rows: sim index out of range");
  SimHost &s = h->sims[(size_t)sim];
  if (!s.prepared) return fail(h, GS_ERR_STATE, "gs_fetch_rows: nothing has run yet");
  const SimDev &D = s.dev;
  if (count < 0 || first < D.row_first || first + count > D.ticks)
    return fail(h, GS_ERR_ARG, "gs_fetch_rows: range is outside the rows of the last gs_run window");
  if (count == 0) return GS_OK;
  if (!rows_out) return fail(h, GS_ERR_ARG, "gs_fetch_rows: NULL output");
  CU(cudaSetDevice(h->device));
  if (s.pol.schedule != GS_SCHED_FIFO)
    return timed_d2h(h, rows_out, D.rows + (first - D.row_first), sizeof(gs_tick_row) * (size_t)count);
  // fifo: rebuild the rows of the whole window from its records on the device, copy the requested slice
  const int64_t wrows = D.ticks - D.row_first;
  int rc = ensure_scratch(h, sizeof(gs_tick_row) * (size_t)wrows);
  if (rc) return rc;
  if (D.nev > 0) {
    gs_expand_rows_kernel<<<(unsigned)((D.nev + 127) / 128), 128, 0, h->stream>>>(h->d_sims, sim, D.M, D.G, (gs_tick_row *)h->d_scratch);
    CU(cudaGetLastError());
    h->launches += 1;
  }
  return timed_d2h(h, rows_out, (gs_tick_row *)h->d_scratch + (first - D.row_first), sizeof(gs_tick_row) * (size_t)count);
}

extern "C" int gs_fetch_jobs(gs_handle h, int sim, gs_job_rec *jobs_out, int32_t *finish_order_out) {
  if (!h) return GS_ERR_ARG;
  if (sim < 0 || sim >= h->nsims) return fail(h, GS_ERR_ARG, "gs_fetch_jobs: sim index out of range");
  SimHost &s = h->sims[(size_t)sim];
  if (!s.prepared) return fail(h, GS_ERR_STATE, "gs_fetch_jobs: nothing has run yet");
  CU(cudaSetDevice(h->device));
  const SimDev &D = s.dev;
  const gs_job_rec *src = D.rec;
  if (jobs_out && s.n > 0 && s.pol.schedule == GS_SCHED_FIFO) {
    int rc = ensure_scratch(h, sizeof(gs_job_rec) * (size_t)s.n);
    if (rc) return rc;
    gs_expand_jobs_kernel<<<(unsigned)((s.n + 255) / 256), 256, 0, h->stream>>>(h->d_sims, sim, (gs_job_rec *)h->d_scratch);
    CU(cudaGetLastError());
    h->launches += 1;
    src = (const gs_job_rec *)h->d_scratch;
  }
  CU(cudaEventRecord(h->e0, h->stream));
  if (jobs_out && s.n > 0)
    CU(cudaMemcpyAsync(jobs_out, src, sizeof(gs_job_rec) * (size_t)s.n, cudaMemcpyDeviceToHost, h->stream));
  if (finish_order_out && D.finished > 0)
    CU(cudaMemcpyAsync(finish_order_out, D.fin, 4 * (size_t)D.finished, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaEventRecord(h->e1, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  float ms = 0; cudaEventElapsedTime(&ms, h->e0, h->e1);
  h->d2h_ms += ms;
  return GS_OK;
}

// Spans are pooled in START order while the simulation runs (bit 31 of ntasks marks the first span of a
// job); this entry point hands them out grouped by job (CSR).  Start ticks are unique (one start per
// tick), so the k-th marked span belongs to the job with the k-th smallest start tick.
extern "C" int gs_fetch_spans(gs_handle h, int sim, int64_t *span_off_out, gs_span *spans_out, int64_t spans_cap,
                              int64_t *spans_used) {
  if (!h) return GS_ERR_ARG;
  if (sim < 0 || sim >= h->nsims) return fail(h, GS_ERR_ARG, "gs_fetch_spans: sim index out of range");
  SimHost &s = h->sims[(size_t)sim];
  if (!s.prepared) return fail(h, GS_ERR_STATE, "gs_fetch_spans: nothing has run yet");
  CU(cudaSetDevice(h->device));
  const SimDev &D = s.dev;
  const int64_t used = s.pol.schedule == GS_SCHED_FIFO ? D.span_used : 0;
  if (spans_used) *spans_used = used;
  if (!spans_out && !span_off_out) return GS_OK;
  if (spans_out && spans_cap < used) return fail(h, GS_ERR_CAPACITY, "gs_fetch_spans: spans_out too small");
  const int64_t n = s.n;
  if (used == 0) {
    if (span_off_out) for (int64_t j = 0; j <= n; ++j) span_off_out[j] = 0;
    return GS_OK;
  }
  std::vector<gs_span> pool((size_t)used);
  std::vector<int32_t> r2((size_t)n);
  int rc;
  if (s.cl.num_gpu_p_node > 32) {
    rc = timed_d2h(h, pool.data(), D.spans, sizeof(gs_span) * (size_t)used);
    if (rc) return rc;
  } else {                  // compact 8-byte records on the device: widen them here
    std::vector<gs_cspan> cp((size_t)used);
    rc = timed_d2h(h, cp.data(), D.spans, sizeof(gs_cspan) * (size_t)used);
    if (rc) return rc;
    for (int64_t i = 0; i < used; ++i) {
      const uint32_t w = cp[(size_t)i].where;
      gs_span sp; sp.node = (int32_t)GS_CSPAN_NODE(w); sp.devmask = cp[(size_t)i].devmask;
      sp.ntasks = (int32_t)(GS_CSPAN_NTASKS(w) | (GS_CSPAN_FIRST(w) ? GS_SPAN_FIRST : 0u));
      pool[(size_t)i] = sp;
    }
  }
  rc = timed_d2h(h, r2.data(), D.jstart, 4 * (size_t)n);
  if (rc) return rc;
  // jobs in start order: bucket by start tick (unique, < ticks)
  std::vector<int32_t> by_tick((size_t)D.ticks + 1, -1);
  const int64_t admitted = D.p;
  for (int64_t j = 0; j < admitted; ++j) if (r2[(size_t)j] >= 0 && r2[(size_t)j] <= D.ticks) by_tick[(size_t)r2[(size_t)j]] = (int32_t)j;
  std::vector<int32_t> order; order.reserve((size_t)n);
  for (int64_t t = 0; t <= D.ticks; ++t) if (by_tick[(size_t)t] >= 0) order.push_back(by_tick[(size_t)t]);
  std::vector<int64_t> first((size_t)n, 0), cnt((size_t)n, 0);
  int64_t k = -1;
  for (int64_t i = 0; i < used; ++i) {
    if ((uint32_t)pool[(size_t)i].ntasks & GS_SPAN_FIRST) { ++k; if (k < (int64_t)order.size()) first[(size_t)order[(size_t)k]] = i; }
    if (k >= 0 && k < (int64_t)order.size()) cnt[(size_t)order[(size_t)k]] += 1;
  }
  if (k + 1 != (int64_t)order.size()) return fail(h, GS_ERR_STATE, "gs_fetch_spans: span pool and start records disagree");
  int64_t run = 0;
  for (int64_t j = 0; j < n; ++j) {
    if (span_off_out) span_off_out[j] = run;
    if (spans_out)
      for (int64_t i = 0; i < cnt[(size_t)j]; ++i) {
        gs_span sp = pool[(size_t)(first[(size_t)j] + i)];
        sp.ntasks = (int32_t)((uint32_t)sp.ntasks & ~GS_SPAN_FIRST);
        spans_out[run + i] = sp;
      }
    run += cnt[(size_t)j];
  }
  if (span_off_out) span_off_out[n] = run;
  return GS_OK;
}

// Everything a caller needs from one finished (or paused) replica in ONE call, in the row / record
// formats of the reference's LogInfo and job.csv (the compact, asynchronous route is gs_fetch_compact).
extern "C" int gs_fetch_all(gs_handle h, int sim, int64_t first, int64_t count, gs_tick_row *rows_out,
                            gs_job_rec *jobs_out, int32_t *finish_order_out, int64_t *span_off_out,
                            gs_span *spans_out, int64_t spans_cap, int64_t *spans_used) {
  if (!h) return GS_ERR_ARG;
  int rc = GS_OK;
  if (rows_out) rc = gs_fetch_rows(h, sim, first, count, rows_out);
  if (rc == GS_OK && (jobs_out || finish_order_out)) rc = gs_fetch_jobs(h, sim, jobs_out, finish_order_out);
  if (rc == GS_OK) rc = gs_fetch_spans(h, sim, span_off_out, spans_out, spans_cap, spans_used);
  return rc;
}

// ------------------------------------------------------------------ run summaries (gs_summary.cuh)
// Rows of the last window not folded yet (`delta` above the accumulator's watermark), one block per replica.
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_sum_rows_kernel(const SimDev *sims, int first, gs_summary *acc) {
  const int r = first + blockIdx.x;
  const SimDev &S = sims[r];
  gs_summary &A = acc[r];
  const long long wm = A.rows;
  const long long lo = wm > S.row_first ? wm : S.row_first, hi = S.ticks;
  GsSumPart p;
  gs_sum_zero(p);
  if (S.policy == GS_SCHED_FIFO) gs_sum_fold_records(p, S.evrows, S.nev, S.qrows, S.nq, S.ticks, wm);
  else
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) gs_sum_row(p, S.rows[i - S.row_first], 0.0);
  gs_sum_block_reduce(p);
  if (threadIdx.x == 0) {
    A.n = S.n; A.done = S.done; A.status = S.status;
    if (hi > lo) {
      gs_sum_add_rows(A, p);
      A.makespan = S.policy == GS_SCHED_FIFO ? hi : S.rows[hi - 1 - S.row_first].now;   // fifo: row i has delta i + 1
    }
    A.util_sum = __longlong_as_double(0x7ff8000000000000ll);    // sampled on the host after the run
  }
}

// Timeline: the same rows as gs_sum_rows_kernel into the replica's bins.  Launched before it, so `acc[r].rows` is still
// the watermark of the rows folded before this call.
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_tl_rows_kernel(const SimDev *sims, int first, const gs_summary *acc, gs_tbin *bins,
                                                                    long long W, int B) {
  const int r = first + blockIdx.x;
  const SimDev &S = sims[r];
  const long long wm = acc[r].rows;
  gs_tbin *T = bins + (size_t)r * (size_t)B;
  if (S.policy == GS_SCHED_FIFO) gs_tl_fold_records(T, B, W, S.evrows, S.nev, S.qrows, S.nq, S.ticks, wm);
  else gs_tl_fold_rows(T, B, W, S.rows, nullptr, S.row_first, wm > S.row_first ? wm : S.row_first, S.ticks);
  gs_tl_util_nan(T, B);
}

// Occupancy: the same rows as gs_sum_rows_kernel into the replica's gs_occ, carry and histograms.  Launched before it,
// like gs_tl_rows_kernel.  fifo folds the records alone: busy, running and queued are constant over a record.
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_occ_rows_kernel(const SimDev *sims, int first, const gs_summary *acc, GsOccCfg cfg,
                                                                     gs_occ *occ, GsOccCarry *carry, unsigned long long *busy,
                                                                     long long pitch, unsigned long long *queue) {
  extern __shared__ unsigned long long occ_dyn[];          // 2 * (G + 1) counters where they fit GS_OCC_SMEM_COUNTERS
  const int r = first + blockIdx.x;
  const SimDev &S = sims[r];
  const long long wm = acc[r].rows;
  unsigned long long *hall = busy + (size_t)r * 2 * (size_t)pitch, *hq = queue + (size_t)r * (size_t)(cfg.nedges + 1);
  if (S.policy == GS_SCHED_FIFO)
    gs_occ_fold(GS_OCC_FIFO, occ_dyn, occ + r, nullptr, hall, hall + pitch, hq, cfg, S.M * S.G, S.evrows, S.nev, S.ticks, wm, nullptr, 0, 0, 0, 1);
  else
    gs_occ_fold(GS_OCC_EVENTS, occ_dyn, occ + r, carry + r, hall, hall + pitch, hq, cfg, S.M * S.G, nullptr, 0, 0, 0, S.rows, S.row_first,
                wm > S.row_first ? wm : S.row_first, S.ticks, S.done);
}

// The finished jobs as job.csv prints them (gs_expand_jobs_kernel for fifo, the job records otherwise).  job(r, i) is
// the i-th job of the finish order, job_at(r, j) job j of the trace (meaningful once it has finished).
struct GsSumEngineJobs {
  const SimDev *sims;
  __device__ long long finished(int r) const { return sims[r].finished; }
  __device__ long long n(int r) const { return sims[r].n; }
  __device__ int order(int r, long long i) const { return sims[r].fin[i]; }
  __device__ GsSumJob job(int r, long long i) const { return job_at(r, sims[r].fin[i]); }
  __device__ int arrive_at(int r, int j) const { return sims[r].jobs[j].arrive; }
  // the gs_jobin records of job j in the traces of replicas ra and rb are byte-equal
  __device__ bool same_job(int ra, int rb, int j) const {
    const unsigned long long *x = reinterpret_cast<const unsigned long long *>(sims[ra].jobs + j);
    const unsigned long long *y = reinterpret_cast<const unsigned long long *>(sims[rb].jobs + j);
    static_assert(sizeof(JobIn) == 32, "JobIn is four 64-bit words");
    return x[0] == y[0] && x[1] == y[1] && x[2] == y[2] && x[3] == y[3];
  }
  __device__ GsSumJob job_at(int r, int j) const {
    const SimDev &S = sims[r];
    const JobIn jb = S.jobs[j];
    if (S.policy == GS_SCHED_FIFO) {
      const int st = S.jstart[j];
      const double d = S.netcost ? S.dur2[j] : jb.dur;
      const int need = gs_sum_run_length(d > jb.dur ? d : jb.dur);
      return gs_sum_job(jb.arrive, st, st + need, need, 1, jb.gpus);
    }
    const gs_job_rec rec = S.rec[j];
    return gs_sum_job(jb.arrive, rec.start, rec.end, rec.jct, rec.preempt, jb.gpus);
  }
};

// The busy histograms' pitch: G + 1 counters of the largest cluster summarised so far.  A larger one moves every
// replica's counters to the new pitch.
static int ensure_occ_pitch(gs_handle h, int first, int count) {
  int64_t need = 1;
  for (int i = first; i < first + count; ++i) need = std::max(need, (int64_t)h->sims[(size_t)i].dev.M * h->sims[(size_t)i].dev.G + 1);
  if (need <= h->occ_pitch) return GS_OK;
  const size_t bytes = 16 * (size_t)need * (size_t)h->nsims;
  unsigned long long *d = nullptr;
  CU(cudaMalloc(&d, bytes));
  CU(cudaMemsetAsync(d, 0, bytes, h->stream));
  if (h->d_occ_busy) {
    CU(cudaMemcpy2DAsync(d, 8 * (size_t)need, h->d_occ_busy, 8 * (size_t)h->occ_pitch, 8 * (size_t)h->occ_pitch, 2 * (size_t)h->nsims,
                         cudaMemcpyDeviceToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_occ_busy);
  }
  h->d_occ_busy = d; h->occ_pitch = need;
  return GS_OK;
}

extern "C" int gs_summarize(gs_handle h, int first, int count, gs_summary *out, double *kernel_ms) {
  if (!h) return GS_ERR_ARG;
  if (first < 0 || count < 0 || first + count > h->nsims || (count > 0 && !out)) return fail(h, GS_ERR_ARG, "gs_summarize: bad arguments");
  if (count == 0) { if (kernel_ms) *kernel_ms = 0.0; return GS_OK; }
  // every check before anything changes: a refused call leaves the accumulators as they were
  int64_t kmax = 1;
  for (int i = first; i < first + count; ++i) {
    const SimHost &s = h->sims[(size_t)i];
    if (!s.prepared) return fail(h, GS_ERR_STATE, "gs_summarize: a replica has not run yet");
    if (s.sum_rows < s.dev.row_first)
      return fail(h, GS_ERR_STATE, "gs_summarize: a replica ran a window that was not summarised (call gs_summarize after every gs_run)");
    kmax = std::max(kmax, (int64_t)s.dev.finished);
    if (h->occ_on && (int64_t)s.dev.M * s.dev.G > GS_OCC_MAX_GPUS)
      return fail(h, GS_ERR_ARG, "gs_summarize: the occupancy statistics take clusters of at most 65535 GPUs");
  }
  CU(cudaSetDevice(h->device));
  if (h->occ_on) { const int rc = ensure_occ_pitch(h, first, count); if (rc) return rc; }
  if (!h->d_sum) {
    CU(cudaMalloc(&h->d_sum, sizeof(gs_summary) * (size_t)h->nsims));
    CU(cudaMemset(h->d_sum, 0, sizeof(gs_summary) * (size_t)h->nsims));
  }
  int per_sm = 1, sms = 132;
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gs_sum_jobs_kernel<GsSumEngineJobs>, GS_SUM_THREADS, 0));
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
  const int grid = std::min(count, std::max(1, per_sm) * sms);
  const size_t pitch = (size_t)align_up((size_t)kmax, 64);
  const int Csd = h->sd.nclasses, Barr = h->arr.nbins;
  int grid_arr = 0;
  if (Barr > 0) {
    int per_arr = 1;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_arr, gs_arr_jobs_kernel<GsSumEngineJobs>, GS_SUM_THREADS, 0));
    grid_arr = std::min(grid, std::max(1, per_arr) * sms);
  }
  int rc = ensure_scratch(h, std::max((Csd > 0 ? 4 : 3) * sizeof(int) * pitch * (size_t)grid,    // gs_sd_jobs_kernel: a fourth row
                                      GS_ARR_ROWS * sizeof(int) * pitch * (size_t)grid_arr));
  if (rc) return rc;
  const int B = h->tl_nbins;
  for (int i = first; i < first + count; ++i) {
    SimHost &s = h->sims[(size_t)i];
    if (s.sum_fresh) { CU(cudaMemsetAsync(h->d_sum + i, 0, sizeof(gs_summary), h->stream)); s.sum_fresh = false; }
    if (B > 0 && s.tl_fresh) { CU(cudaMemsetAsync(h->d_tl + (size_t)i * B, 0, sizeof(gs_tbin) * (size_t)B, h->stream)); s.tl_fresh = false; }
    if (h->occ_on && s.occ_fresh) {
      CU(cudaMemsetAsync(h->d_occ + i, 0, sizeof(gs_occ), h->stream));
      CU(cudaMemsetAsync(h->d_occ_carry + i, 0, sizeof(GsOccCarry), h->stream));
      CU(cudaMemsetAsync(h->d_occ_busy + (size_t)i * 2 * (size_t)h->occ_pitch, 0, 16 * (size_t)h->occ_pitch, h->stream));
      CU(cudaMemsetAsync(h->d_occ_q + (size_t)i * (h->occ.nedges + 1), 0, 8 * (size_t)(h->occ.nedges + 1), h->stream));
      s.occ_fresh = false;
    }
  }
  CU(cudaEventRecord(h->e0, h->stream));
  if (h->occ_on) {        // before gs_sum_rows_kernel, which advances the watermark
    int gsm = 0;          // dynamic shared memory for the replicas whose busy histograms fit it
    for (int i = first; i < first + count; ++i) {
      const int g = h->sims[(size_t)i].dev.M * h->sims[(size_t)i].dev.G;
      if (2 * (g + 1) <= GS_OCC_SMEM_COUNTERS) gsm = std::max(gsm, g);
    }
    gs_occ_rows_kernel<<<(unsigned)count, GS_SUM_THREADS, 16 * (size_t)(gsm + 1), h->stream>>>(
        h->d_sims, first, h->d_sum, h->occ, h->d_occ, h->d_occ_carry, h->d_occ_busy, (long long)h->occ_pitch, h->d_occ_q);
    CU(cudaGetLastError());
    h->launches += 1;
  }
  if (B > 0) {            // before gs_sum_rows_kernel, which advances the watermark
    gs_tl_rows_kernel<<<(unsigned)count, GS_SUM_THREADS, 0, h->stream>>>(h->d_sims, first, h->d_sum, h->d_tl, (long long)h->tl_width, B);
    CU(cudaGetLastError());
    h->launches += 1;
  }
  gs_sum_rows_kernel<<<(unsigned)count, GS_SUM_THREADS, 0, h->stream>>>(h->d_sims, first, h->d_sum);
  CU(cudaGetLastError());
  GsSumEngineJobs src{h->d_sims};
  gs_sum_jobs_kernel<GsSumEngineJobs><<<(unsigned)grid, GS_SUM_THREADS, 0, h->stream>>>(src, first, count, h->d_sum, (int *)h->d_scratch,
                                                                                       (long long)pitch);
  CU(cudaGetLastError());
  h->launches += 2;
  const int C = h->jd.nclasses;
  if (C > 0) {            // after gs_sum_jobs_kernel, on the same scratch
    int per_jd = 1;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_jd, gs_jd_jobs_kernel<GsSumEngineJobs>, GS_SUM_THREADS, 0));
    const int grid_jd = std::min(grid, std::max(1, per_jd) * sms);
    gs_jd_jobs_kernel<GsSumEngineJobs><<<(unsigned)grid_jd, GS_SUM_THREADS, 0, h->stream>>>(src, first, count, h->jd, h->d_jd, h->d_jd_hist,
                                                                                           (int *)h->d_scratch, (long long)pitch);
    CU(cudaGetLastError());
    h->launches += 1;
  }
  if (Csd > 0) {          // after gs_sum_jobs_kernel (and gs_jd_jobs_kernel), on the same scratch
    int per_sd = 1;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sd, gs_sd_jobs_kernel<GsSumEngineJobs>, GS_SUM_THREADS, 0));
    const int grid_sd = std::min(grid, std::max(1, per_sd) * sms);
    gs_sd_jobs_kernel<GsSumEngineJobs><<<(unsigned)grid_sd, GS_SUM_THREADS, 0, h->stream>>>(src, first, count, h->sd, h->d_sd, h->d_sd_hist,
                                                                                           (int *)h->d_scratch, (long long)pitch);
    CU(cudaGetLastError());
    h->launches += 1;
  }
  if (Barr > 0) {         // after the other job kernels: its own GS_ARR_ROWS rows on the same scratch
    gs_arr_jobs_kernel<GsSumEngineJobs><<<(unsigned)grid_arr, GS_SUM_THREADS, 0, h->stream>>>(src, first, count, h->arr, h->d_arr,
                                                                                             (int *)h->d_scratch, (long long)pitch);
    CU(cudaGetLastError());
    h->launches += 1;
  }
  CU(cudaEventRecord(h->e1, h->stream));
  CU(cudaMemcpyAsync(out, h->d_sum + first, sizeof(gs_summary) * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  float ms = 0; cudaEventElapsedTime(&ms, h->e0, h->e1);
  if (kernel_ms) *kernel_ms = ms;
  for (int i = first; i < first + count; ++i) {
    h->sims[(size_t)i].sum_rows = out[i - first].rows;
    if (B > 0) h->sims[(size_t)i].tl_done = true;
    if (C > 0) h->sims[(size_t)i].jd_done = true;
    if (Csd > 0) h->sims[(size_t)i].sd_done = true;
    if (Barr > 0) h->sims[(size_t)i].arr_done = true;
    if (h->occ_on) h->sims[(size_t)i].occ_done = true;
  }
  return GS_OK;
}

extern "C" int gs_set_timeline(gs_handle h, int64_t bin_width, int32_t nbins) {
  if (!h) return GS_ERR_ARG;
  if (nbins < 0 || nbins > GS_TIMELINE_MAX_BINS || (nbins > 0 && (bin_width < 1 || bin_width > (1ll << 40))))
    return fail(h, GS_ERR_ARG, "gs_set_timeline: nbins must be in 0..1024 and, when it is not 0, bin_width in 1..2^40");
  for (const SimHost &s : h->sims)
    if (s.prepared && !s.sum_fresh && s.sum_rows > 0)
      return fail(h, GS_ERR_STATE, "gs_set_timeline: a replica has already folded rows (set the timeline before summarising a run, or after gs_reset)");
  const size_t need = sizeof(gs_tbin) * (size_t)h->nsims * (size_t)nbins;
  if (need > h->tl_bytes) {
    CU(cudaSetDevice(h->device));
    gs_tbin *d = nullptr;
    CU(cudaMalloc(&d, need));
    if (h->d_tl) { CU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_tl); }
    h->d_tl = d; h->tl_bytes = need;
  }
  h->tl_width = nbins > 0 ? bin_width : 0;
  h->tl_nbins = nbins;
  for (SimHost &s : h->sims) { s.tl_fresh = true; s.tl_done = false; }
  return GS_OK;
}

extern "C" int gs_fetch_timeline(gs_handle h, int first, int count, gs_tbin *out) {
  if (!h) return GS_ERR_ARG;
  if (first < 0 || count < 0 || first + count > h->nsims || (count > 0 && !out)) return fail(h, GS_ERR_ARG, "gs_fetch_timeline: bad arguments");
  if (h->tl_nbins == 0) return fail(h, GS_ERR_STATE, "gs_fetch_timeline: the timeline is off (gs_set_timeline)");
  for (int i = first; i < first + count; ++i) {
    const SimHost &s = h->sims[(size_t)i];
    if (!s.prepared || !s.tl_done) return fail(h, GS_ERR_STATE, "gs_fetch_timeline: a replica has not been summarised with the timeline on since it was prepared");
  }
  if (count == 0) return GS_OK;
  CU(cudaSetDevice(h->device));
  const size_t B = (size_t)h->tl_nbins;
  CU(cudaMemcpyAsync(out, h->d_tl + (size_t)first * B, sizeof(gs_tbin) * B * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  CU(wait_stream(h));
  return GS_OK;
}

extern "C" int gs_set_jobdist(gs_handle h, int32_t nclasses, const int32_t *bounds, int32_t nedges, const int32_t *edges) {
  if (!h) return GS_ERR_ARG;
  GsJdCfg cfg;
  const char *why = nullptr;
  if (!gs_jd_make_cfg(nclasses, bounds, nedges, edges, cfg, &why)) return fail(h, GS_ERR_ARG, std::string("gs_set_jobdist: ") + why);
  const size_t need = sizeof(gs_jclass) * (size_t)h->nsims * (size_t)cfg.nclasses;
  const size_t need_hist = sizeof(unsigned) * (size_t)h->nsims * (size_t)cfg.nclasses * 3 * (size_t)(cfg.nedges + 1);
  if (need > h->jd_bytes || need_hist > h->jd_hist_bytes) {
    CU(cudaSetDevice(h->device));
    gs_jclass *d = nullptr;
    unsigned *dh = nullptr;
    CU(cudaMalloc(&d, std::max(need, h->jd_bytes)));
    if (cudaMalloc(&dh, std::max(need_hist, h->jd_hist_bytes)) != cudaSuccess) {
      cudaFree(d);
      return fail(h, GS_ERR_CUDA, "gs_set_jobdist: cudaMalloc failed");
    }
    CU(cudaStreamSynchronize(h->stream));
    if (h->d_jd) cudaFree(h->d_jd);
    if (h->d_jd_hist) cudaFree(h->d_jd_hist);
    h->d_jd = d; h->jd_bytes = std::max(need, h->jd_bytes);
    h->d_jd_hist = dh; h->jd_hist_bytes = std::max(need_hist, h->jd_hist_bytes);
  }
  h->jd = cfg;
  for (SimHost &s : h->sims) s.jd_done = false;
  return GS_OK;
}

extern "C" int gs_fetch_jobdist(gs_handle h, int first, int count, gs_jclass *classes_out, uint32_t *hist_out) {
  if (!h) return GS_ERR_ARG;
  if (first < 0 || count < 0 || first + count > h->nsims) return fail(h, GS_ERR_ARG, "gs_fetch_jobdist: bad arguments");
  if (h->jd.nclasses == 0) return fail(h, GS_ERR_STATE, "gs_fetch_jobdist: the job statistics are off (gs_set_jobdist)");
  for (int i = first; i < first + count; ++i) {
    const SimHost &s = h->sims[(size_t)i];
    if (!s.prepared || !s.jd_done)
      return fail(h, GS_ERR_STATE, "gs_fetch_jobdist: a replica has not been summarised with this setting since it was prepared");
  }
  if (count == 0) return GS_OK;
  CU(cudaSetDevice(h->device));
  const size_t C = (size_t)h->jd.nclasses, per = C * 3 * (size_t)(h->jd.nedges + 1);
  if (classes_out)
    CU(cudaMemcpyAsync(classes_out, h->d_jd + (size_t)first * C, sizeof(gs_jclass) * C * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  if (hist_out)
    CU(cudaMemcpyAsync(hist_out, h->d_jd_hist + (size_t)first * per, sizeof(unsigned) * per * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  CU(wait_stream(h));
  return GS_OK;
}

extern "C" int gs_set_slowdown(gs_handle h, const gs_slowdown_cfg *in) {
  if (!h) return GS_ERR_ARG;
  GsSdCfg cfg;
  const char *why = nullptr;
  if (!gs_sd_make_cfg(in, cfg, &why)) return fail(h, GS_ERR_ARG, std::string("gs_set_slowdown: ") + why);
  const size_t need = sizeof(gs_sdclass) * (size_t)h->nsims * (size_t)cfg.nclasses;
  const size_t need_hist = sizeof(unsigned) * (size_t)h->nsims * (size_t)cfg.nclasses * (size_t)gs_sd_row_len(cfg);
  if (need > h->sd_bytes || need_hist > h->sd_hist_bytes) {
    CU(cudaSetDevice(h->device));
    gs_sdclass *d = nullptr;
    unsigned *dh = nullptr;
    CU(cudaMalloc(&d, std::max(need, h->sd_bytes)));
    if (cudaMalloc(&dh, std::max(need_hist, h->sd_hist_bytes)) != cudaSuccess) {
      cudaFree(d);
      return fail(h, GS_ERR_CUDA, "gs_set_slowdown: cudaMalloc failed");
    }
    CU(cudaStreamSynchronize(h->stream));
    if (h->d_sd) cudaFree(h->d_sd);
    if (h->d_sd_hist) cudaFree(h->d_sd_hist);
    h->d_sd = d; h->sd_bytes = std::max(need, h->sd_bytes);
    h->d_sd_hist = dh; h->sd_hist_bytes = std::max(need_hist, h->sd_hist_bytes);
  }
  h->sd = cfg;
  for (SimHost &s : h->sims) s.sd_done = false;
  return GS_OK;
}

extern "C" int gs_fetch_slowdown(gs_handle h, int first, int count, gs_sdclass *out, uint32_t *hist_out) {
  if (!h) return GS_ERR_ARG;
  if (first < 0 || count < 0 || first + count > h->nsims) return fail(h, GS_ERR_ARG, "gs_fetch_slowdown: bad arguments");
  if (h->sd.nclasses == 0) return fail(h, GS_ERR_STATE, "gs_fetch_slowdown: the slowdown statistics are off (gs_set_slowdown)");
  for (int i = first; i < first + count; ++i) {
    const SimHost &s = h->sims[(size_t)i];
    if (!s.prepared || !s.sd_done)
      return fail(h, GS_ERR_STATE, "gs_fetch_slowdown: a replica has not been summarised with this setting since it was prepared");
  }
  if (count == 0) return GS_OK;
  CU(cudaSetDevice(h->device));
  const size_t C = (size_t)h->sd.nclasses, per = C * (size_t)gs_sd_row_len(h->sd);
  if (out)
    CU(cudaMemcpyAsync(out, h->d_sd + (size_t)first * C, sizeof(gs_sdclass) * C * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  if (hist_out)
    CU(cudaMemcpyAsync(hist_out, h->d_sd_hist + (size_t)first * per, sizeof(unsigned) * per * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  CU(wait_stream(h));
  return GS_OK;
}

extern "C" int gs_set_arrivals(gs_handle h, int64_t bin_width, int32_t nbins, int64_t tau) {
  if (!h) return GS_ERR_ARG;
  GsArrCfg cfg;
  const char *why = nullptr;
  if (!gs_arr_make_cfg(bin_width, nbins, tau, cfg, &why)) return fail(h, GS_ERR_ARG, std::string("gs_set_arrivals: ") + why);
  CU(cudaSetDevice(h->device));
  const size_t need = sizeof(gs_abin) * (size_t)h->nsims * (size_t)cfg.nbins;
  if (need > h->arr_bytes) {
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    gs_abin *d = nullptr;
    if (need > free_b || cudaMalloc(&d, need) != cudaSuccess) {
      (void)cudaGetLastError();
      return fail(h, GS_ERR_CAPACITY, "gs_set_arrivals: the bin records (" + std::to_string(need) + " bytes) do not fit the device's free memory");
    }
    if (h->d_arr) { CU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_arr); }
    h->d_arr = d; h->arr_bytes = need;
  } else if (cfg.nbins == 0 && h->d_arr) {           // off: the records are not kept
    CU(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_arr);
    h->d_arr = nullptr; h->arr_bytes = 0;
  }
  h->arr = cfg;
  for (SimHost &s : h->sims) s.arr_done = false;
  return GS_OK;
}

extern "C" int gs_fetch_arrivals(gs_handle h, int first, int count, gs_abin *out) {
  if (!h) return GS_ERR_ARG;
  if (first < 0 || count < 0 || first + count > h->nsims || (count > 0 && !out)) return fail(h, GS_ERR_ARG, "gs_fetch_arrivals: bad arguments");
  if (h->arr.nbins == 0) return fail(h, GS_ERR_STATE, "gs_fetch_arrivals: the arrival statistics are off (gs_set_arrivals)");
  for (int i = first; i < first + count; ++i) {
    const SimHost &s = h->sims[(size_t)i];
    if (!s.prepared || !s.arr_done)
      return fail(h, GS_ERR_STATE, "gs_fetch_arrivals: a replica has not been summarised with this setting since it was prepared");
  }
  if (count == 0) return GS_OK;
  CU(cudaSetDevice(h->device));
  const size_t B = (size_t)h->arr.nbins;
  CU(cudaMemcpyAsync(out, h->d_arr + (size_t)first * B, sizeof(gs_abin) * B * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  CU(wait_stream(h));
  return GS_OK;
}

extern "C" int gs_set_occupancy(gs_handle h, int32_t on, int32_t nedges, const int32_t *edges) {
  if (!h) return GS_ERR_ARG;
  GsOccCfg cfg{};
  const char *why = nullptr;
  if (on && !gs_occ_make_cfg(nedges, edges, cfg, &why)) return fail(h, GS_ERR_ARG, std::string("gs_set_occupancy: ") + why);
  for (const SimHost &s : h->sims)
    if (s.prepared && !s.sum_fresh && s.sum_rows > 0)
      return fail(h, GS_ERR_STATE, "gs_set_occupancy: a replica has already folded rows (set the occupancy before summarising a run, or after gs_reset)");
  if (on) {
    CU(cudaSetDevice(h->device));
    const size_t need_q = 8 * (size_t)h->nsims * (size_t)(cfg.nedges + 1);
    if (!h->d_occ) {
      gs_occ *d = nullptr;
      GsOccCarry *c = nullptr;
      CU(cudaMalloc(&d, sizeof(gs_occ) * (size_t)h->nsims));
      if (cudaMalloc(&c, sizeof(GsOccCarry) * (size_t)h->nsims) != cudaSuccess) { cudaFree(d); return fail(h, GS_ERR_CUDA, "gs_set_occupancy: cudaMalloc failed"); }
      h->d_occ = d; h->d_occ_carry = c;
    }
    if (need_q > h->occ_q_bytes) {
      unsigned long long *d = nullptr;
      CU(cudaMalloc(&d, need_q));
      if (h->d_occ_q) { CU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_occ_q); }
      h->d_occ_q = d; h->occ_q_bytes = need_q;
    }
  }
  h->occ_on = on != 0;
  h->occ = cfg;
  for (SimHost &s : h->sims) { s.occ_fresh = true; s.occ_done = false; }
  return GS_OK;
}

extern "C" int gs_fetch_occupancy(gs_handle h, int first, int count, gs_occ *out, uint64_t *busy_hist, int32_t busy_pitch, uint64_t *queue_hist) {
  if (!h) return GS_ERR_ARG;
  if (first < 0 || count < 0 || first + count > h->nsims) return fail(h, GS_ERR_ARG, "gs_fetch_occupancy: bad arguments");
  if (!h->occ_on) return fail(h, GS_ERR_STATE, "gs_fetch_occupancy: the occupancy statistics are off (gs_set_occupancy)");
  int64_t width = 1;
  for (int i = first; i < first + count; ++i) {
    const SimHost &s = h->sims[(size_t)i];
    if (!s.prepared || !s.occ_done)
      return fail(h, GS_ERR_STATE, "gs_fetch_occupancy: a replica has not been summarised with the occupancy on since it was prepared");
    width = std::max(width, (int64_t)s.dev.M * s.dev.G + 1);
  }
  if (busy_hist && count > 0 && busy_pitch < width)
    return fail(h, GS_ERR_CAPACITY, "gs_fetch_occupancy: busy_pitch is smaller than total_gpus + 1 of a fetched replica");
  if (count == 0) return GS_OK;
  CU(cudaSetDevice(h->device));
  if (out) CU(cudaMemcpyAsync(out, h->d_occ + first, sizeof(gs_occ) * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  if (busy_hist)
    CU(cudaMemcpy2DAsync(busy_hist, 8 * (size_t)busy_pitch, h->d_occ_busy + (size_t)first * 2 * (size_t)h->occ_pitch, 8 * (size_t)h->occ_pitch,
                         8 * (size_t)std::min(width, h->occ_pitch), 2 * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  const size_t E1 = (size_t)h->occ.nedges + 1;
  if (queue_hist) CU(cudaMemcpyAsync(queue_hist, h->d_occ_q + (size_t)first * E1, 8 * E1 * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  CU(wait_stream(h));
  return GS_OK;
}

extern "C" int gs_compare(gs_handle h, int32_t npairs, const int32_t *a, const int32_t *b, int32_t nclasses, const int32_t *bounds,
                          int32_t nedges, const int32_t *edges, gs_jpair *out, uint32_t *hist_out, double *kernel_ms) {
  if (!h) return GS_ERR_ARG;
  if (npairs < 0 || (npairs > 0 && (!a || !b || !out))) return fail(h, GS_ERR_ARG, "gs_compare: bad arguments");
  GsJdCfg cfg;
  const char *why = nullptr;
  if (!gs_jd_make_cfg(nclasses, bounds, nedges, edges, cfg, &why)) return fail(h, GS_ERR_ARG, std::string("gs_compare: ") + why);
  if (nclasses == 0) return fail(h, GS_ERR_ARG, "gs_compare: nclasses must be in 1..8");
  int64_t nmax = 1;
  for (int i = 0; i < npairs; ++i)
    if (a[i] < 0 || a[i] >= h->nsims || b[i] < 0 || b[i] >= h->nsims) return fail(h, GS_ERR_ARG, "gs_compare: a replica index is out of range");
  for (int i = 0; i < npairs; ++i) {
    const SimHost &sa = h->sims[(size_t)a[i]], &sb = h->sims[(size_t)b[i]];
    if (!sa.prepared || !sb.prepared) return fail(h, GS_ERR_STATE, "gs_compare: a replica has not run yet");
    if (sa.dev.n != sb.dev.n) return fail(h, GS_ERR_ARG, "gs_compare: pair " + std::to_string(i) + " holds traces of different lengths");
    nmax = std::max(nmax, (int64_t)sa.dev.n);
  }
  if (kernel_ms) *kernel_ms = 0.0;
  if (npairs == 0) return GS_OK;
  CU(cudaSetDevice(h->device));
  int per_sm = 1, sms = 132;
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gs_cmp_pairs_kernel<GsSumEngineJobs>, GS_SUM_THREADS, 0));
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
  const int grid = std::min(npairs, std::max(1, per_sm) * sms);
  const size_t pitch = align_up((size_t)nmax, 64), P = (size_t)npairs, C = (size_t)cfg.nclasses, nb = (size_t)cfg.nedges + 1;
  // scratch: pair indices, trace-differ flags, records, CDF counts, per-block work
  const size_t o_a = 0, o_b = align_up(4 * P), o_flag = align_up(o_b + 4 * P), o_rec = align_up(o_flag + 4 * P);
  const size_t o_hist = align_up(o_rec + sizeof(gs_jpair) * P * C), o_work = align_up(o_hist + 4 * P * C * 3 * nb);
  int rc = ensure_scratch(h, o_work + 4 * sizeof(int) * pitch * (size_t)grid);
  if (rc) return rc;
  unsigned char *d = (unsigned char *)h->d_scratch;
  CU(cudaMemcpyAsync(d + o_a, a, 4 * P, cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(d + o_b, b, 4 * P, cudaMemcpyHostToDevice, h->stream));
  CU(cudaEventRecord(h->e0, h->stream));
  gs_cmp_pairs_kernel<GsSumEngineJobs><<<(unsigned)grid, GS_SUM_THREADS, 0, h->stream>>>(
      GsSumEngineJobs{h->d_sims}, npairs, (const int *)(d + o_a), (const int *)(d + o_b), cfg, (gs_jpair *)(d + o_rec),
      (unsigned *)(d + o_hist), (int *)(d + o_flag), (int *)(d + o_work), (long long)pitch);
  CU(cudaGetLastError());
  h->launches += 1;
  CU(cudaEventRecord(h->e1, h->stream));
  std::vector<int> flags(P);
  std::vector<gs_jpair> recs(P * C);
  std::vector<uint32_t> hist(hist_out ? P * C * 3 * nb : 0);
  CU(cudaMemcpyAsync(flags.data(), d + o_flag, 4 * P, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaMemcpyAsync(recs.data(), d + o_rec, sizeof(gs_jpair) * P * C, cudaMemcpyDeviceToHost, h->stream));
  if (hist_out) CU(cudaMemcpyAsync(hist.data(), d + o_hist, 4 * hist.size(), cudaMemcpyDeviceToHost, h->stream));
  CU(wait_stream(h));
  for (size_t i = 0; i < P; ++i)
    if (flags[i]) return fail(h, GS_ERR_ARG, "gs_compare: pair " + std::to_string(i) + " (replicas " + std::to_string(a[i]) + ", " +
                                             std::to_string(b[i]) + ") holds different traces");
  memcpy(out, recs.data(), sizeof(gs_jpair) * recs.size());
  if (hist_out) memcpy(hist_out, hist.data(), 4 * hist.size());
  float ms = 0; cudaEventElapsedTime(&ms, h->e0, h->e1);
  if (kernel_ms) *kernel_ms = ms;
  return GS_OK;
}

// ------------------------------------------------------------------ bootstrap replicas (gs_boot.cuh)
extern "C" int gs_boot_population(gs_handle h, const gs_jobin *trace, int64_t k) {
  if (!h) return GS_ERR_ARG;
  if (!trace || k < 1 || k >= (1ll << 31) - 64) return fail(h, GS_ERR_ARG, "gs_boot_population: bad arguments (1 <= k < 2^31 - 64)");
  const JobIn *ji = reinterpret_cast<const JobIn *>(trace);
  SimHost probe;                                        // the load rules do not depend on the cluster without network costs
  memset(&probe.cl, 0, sizeof(probe.cl));
  probe.cl.num_switch = probe.cl.num_node_p_switch = 1;
  int64_t spans = 0;
  double max_need = 1.0;
  int rc = scan_trace(h, probe, k, ji, false, nullptr, nullptr, &spans, &max_need);
  if (rc) return rc;
  if (max_need > (double)(1 << 26)) return fail(h, GS_ERR_ARG, "gs_boot_population: job duration exceeds 2^26 ticks");
  std::vector<int32_t> gaps((size_t)(k > 1 ? k - 1 : 1), 0);
  int64_t max_gap = 0;
  for (int64_t i = 0; i + 1 < k; ++i) {
    gaps[(size_t)i] = ji[i + 1].arrive - ji[i].arrive;
    max_gap = std::max(max_gap, (int64_t)gaps[(size_t)i]);
  }
  CU(cudaSetDevice(h->device));
  const size_t off_gaps = align_up(sizeof(JobIn) * (size_t)k);
  void *d = nullptr;
  CU(cudaMalloc(&d, off_gaps + 4 * gaps.size()));
  cudaError_t e1 = cudaMemcpy(d, ji, sizeof(JobIn) * (size_t)k, cudaMemcpyHostToDevice);
  cudaError_t e2 = cudaMemcpy((unsigned char *)d + off_gaps, gaps.data(), 4 * gaps.size(), cudaMemcpyHostToDevice);
  if (e1 != cudaSuccess || e2 != cudaSuccess) { cudaFree(d); return fail(h, GS_ERR_CUDA, "gs_boot_population: upload failed"); }
  if (h->d_pop || h->d_mix) CU(cudaStreamSynchronize(h->stream));
  if (h->d_pop) cudaFree(h->d_pop);
  if (h->d_mix) cudaFree(h->d_mix);                     // the tables belong to the previous population
  h->d_pop = d; h->pop_k = k; h->pop_max_gap = max_gap; h->pop_max_need = max_need;
  h->d_mix = nullptr; h->nmix = 0; h->mix_T.clear();
  return GS_OK;
}

extern "C" int gs_boot_mixes(gs_handle h, int32_t nmix, const uint32_t *weights) {
  if (!h) return GS_ERR_ARG;
  if (nmix < 0) return fail(h, GS_ERR_ARG, "gs_boot_mixes: nmix must be >= 0");
  if (nmix > 0 && !weights) return fail(h, GS_ERR_ARG, "gs_boot_mixes: weights is NULL");
  if (!h->d_pop) return fail(h, GS_ERR_STATE, "gs_boot_mixes: call gs_boot_population first");
  // every check before anything changes: a refused call leaves the tables as they were
  const int64_t K = h->pop_k;
  for (int32_t m = 0; m < nmix; ++m) {
    const uint32_t *w = weights + (size_t)m * (size_t)K;
    bool any = false;
    for (int64_t i = 0; i < K && !any; ++i) any = w[i] != 0;
    if (!any) return fail(h, GS_ERR_ARG, "gs_boot_mixes: mix " + std::to_string(m) + " has weight sum 0");
  }
  CU(cudaSetDevice(h->device));
  GsBootAlias *d = nullptr;
  std::vector<uint64_t> T((size_t)nmix);
  if (nmix > 0) {
    if ((uint64_t)nmix * (uint64_t)K > (uint64_t)(SIZE_MAX / 2) / sizeof(GsBootAlias))
      return fail(h, GS_ERR_CUDA, "gs_boot_mixes: the tables do not fit in memory");
    if (cudaMalloc(&d, sizeof(GsBootAlias) * (size_t)nmix * (size_t)K) != cudaSuccess) {
      cudaGetLastError();
      return fail(h, GS_ERR_CUDA, "gs_boot_mixes: allocation of the alias tables failed");
    }
    std::vector<GsBootAlias> tab((size_t)K);              // one mix at a time: host memory stays at one table
    for (int32_t m = 0; m < nmix; ++m) {
      T[(size_t)m] = gs_boot_alias_build(weights + (size_t)m * (size_t)K, K, tab.data());
      if (cudaMemcpy(d + (size_t)m * (size_t)K, tab.data(), sizeof(GsBootAlias) * (size_t)K, cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaFree(d);
        return fail(h, GS_ERR_CUDA, "gs_boot_mixes: upload failed");
      }
    }
  }
  if (h->d_mix) { CU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_mix); }
  h->d_mix = d; h->nmix = nmix; h->mix_T.swap(T);
  return GS_OK;
}

extern "C" int gs_boot_traces(gs_handle h, const gs_boot_params *params, double *kernel_ms) {
  return gs_boot_traces_blocked(h, params, nullptr, kernel_ms);
}

extern "C" int gs_boot_traces_blocked(gs_handle h, const gs_boot_params *params, const uint32_t *block_len, double *kernel_ms) {
  return gs_boot_traces_mixed(h, params, block_len, nullptr, kernel_ms);
}

extern "C" int gs_boot_traces_mixed(gs_handle h, const gs_boot_params *params, const uint32_t *block_len, const int32_t *mix,
                                    double *kernel_ms) {
  return gs_boot_traces_profiled(h, params, block_len, mix, nullptr, kernel_ms);
}

extern "C" int gs_boot_profiles(gs_handle h, int32_t nprof, const int32_t *nseg, const int32_t *period, const gs_boot_seg *segs) {
  if (!h) return GS_ERR_ARG;
  if (nprof < 0) return fail(h, GS_ERR_ARG, "gs_boot_profiles: nprof must be >= 0");
  if (nprof > 0 && (!nseg || !period || !segs)) return fail(h, GS_ERR_ARG, "gs_boot_profiles: NULL array");
  // every check before anything changes: a refused call leaves the profiles as they were
  std::vector<int32_t> off((size_t)nprof);
  size_t total = 0;
  for (int32_t p = 0; p < nprof; ++p) {
    const char *why = gs_boot_profile_invalid(segs + total, nseg[p], period[p]);
    if (why) return fail(h, GS_ERR_ARG, "gs_boot_profiles: profile " + std::to_string(p) + ": " + why);
    off[(size_t)p] = (int32_t)total;
    total += (size_t)nseg[p];
  }
  std::vector<GsBootProfSeg> dev(total);
  std::vector<long long> B((size_t)nprof);
  for (int32_t p = 0; p < nprof; ++p)
    B[(size_t)p] = gs_boot_profile_base(segs + off[(size_t)p], nseg[p], period[p], dev.data() + off[(size_t)p]);
  CU(cudaSetDevice(h->device));
  GsBootProfSeg *d = nullptr;
  if (total > 0) {
    if (cudaMalloc(&d, sizeof(GsBootProfSeg) * total) != cudaSuccess) {
      cudaGetLastError();
      return fail(h, GS_ERR_CUDA, "gs_boot_profiles: allocation of the profiles failed");
    }
    if (cudaMemcpy(d, dev.data(), sizeof(GsBootProfSeg) * total, cudaMemcpyHostToDevice) != cudaSuccess) {
      cudaFree(d);
      return fail(h, GS_ERR_CUDA, "gs_boot_profiles: upload failed");
    }
  }
  if (h->d_prof) { CU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_prof); }
  h->d_prof = d; h->nprof = nprof; h->prof_seg.swap(dev); h->prof_off.swap(off); h->prof_B.swap(B);
  h->prof_nseg.assign(nseg, nseg + nprof); h->prof_period.assign(period, period + nprof);
  return GS_OK;
}

extern "C" int gs_boot_traces_profiled(gs_handle h, const gs_boot_params *params, const uint32_t *block_len, const int32_t *mix,
                                       const int32_t *profile, double *kernel_ms) {
  if (!h) return GS_ERR_ARG;
  if (!params) return fail(h, GS_ERR_ARG, "gs_boot_traces: params is NULL");
  if (!h->d_pop) return fail(h, GS_ERR_STATE, "gs_boot_traces: call gs_boot_population first");
  // every check before anything changes: a refused call leaves the replicas' traces as they were
  std::vector<GsBootRep> reps((size_t)h->nsims);
  int64_t nmax = 1;
  bool blocked = false;                                 // some replica has L > 1: the blocked instantiation
  bool mixed = false;                                   // some replica has a mix >= 0: the mixed instantiation
  bool profiled = false;                                // some replica has a profile >= 0: the profiled instantiation
  for (int i = 0; i < h->nsims; ++i) {
    const SimHost &s = h->sims[(size_t)i];
    const gs_boot_params &p = params[i];
    if (!s.configured) return fail(h, GS_ERR_STATE, "gs_boot_traces: call gs_config_sim for every replica first");
    if (s.cl.enable_network_costs) return fail(h, GS_ERR_ARG, "gs_boot_traces: traces with network columns go through gs_load_trace");
    if (p.n < 0 || p.n >= (1ll << 31) - 64) return fail(h, GS_ERR_ARG, "gs_boot_traces: n out of range");
    if (p.gap_num < 0 || p.gap_den < 1) return fail(h, GS_ERR_ARG, "gs_boot_traces: the gap scale needs gap_num >= 0 and gap_den >= 1");
    const bool prof = profile && profile[i] >= 0;      // a profiled replica's bound is checked through its profile
    if (!prof && gs_boot_arrive_bound(p.n, h->pop_max_gap, p.gap_num, p.gap_den) >= 0x7fffffffll)
      return fail(h, GS_ERR_ARG, "gs_boot_traces: the last arrival tick can reach 2^31 - 1 (fewer jobs or a smaller gap scale)");
    if (block_len && block_len[i] == 0) return fail(h, GS_ERR_ARG, "gs_boot_traces_blocked: block_len must be >= 1");
    if (mix && (mix[i] < -1 || mix[i] >= h->nmix))
      return fail(h, GS_ERR_ARG, "gs_boot_traces_mixed: mix index out of range [-1, nmix) for replica " + std::to_string(i));
    if (profile && (profile[i] < -1 || profile[i] >= h->nprof))
      return fail(h, GS_ERR_ARG, "gs_boot_traces_profiled: profile index out of range [-1, nprof) for replica " + std::to_string(i));
    if (prof && (p.gap_num != 1 || p.gap_den != 1))
      return fail(h, GS_ERR_ARG, "gs_boot_traces_profiled: a profiled replica needs the gap scale 1 / 1 (replica " + std::to_string(i) + ")");
    if (prof) {
      const size_t q = (size_t)profile[i];
      if (gs_boot_profile_bound(h->prof_seg.data() + h->prof_off[q], h->prof_nseg[q], h->prof_period[q], h->prof_B[q], p.n,
                                h->pop_max_gap) >= 0x7fffffffll)
        return fail(h, GS_ERR_ARG, "gs_boot_traces_profiled: the last arrival tick of replica " + std::to_string(i) +
                                       " can reach 2^31 - 1 under its profile (fewer jobs or a lighter profile)");
    }
    GsBootRep &r = reps[(size_t)i];
    r.seed = p.seed; r.stream = p.stream; r.n = p.n; r.gap_num = p.gap_num; r.gap_den = p.gap_den;
    r.M = s.cl.num_switch * s.cl.num_node_p_switch; r.block_len = block_len ? block_len[i] : 1u;
    blocked = blocked || r.block_len > 1;
    mixed = mixed || (mix && mix[i] >= 0);
    profiled = profiled || prof;
    nmax = std::max(nmax, p.n);
  }
  std::vector<GsBootMix> mixes(mixed ? (size_t)h->nsims : 0);
  for (size_t i = 0; i < mixes.size(); ++i) {
    mixes[i].T = mix[i] >= 0 ? h->mix_T[(size_t)mix[i]] : 0;
    mixes[i].off = mix[i] >= 0 ? (long long)mix[i] * (long long)h->pop_k : 0;
  }
  std::vector<GsBootProf> profs(profiled ? (size_t)h->nsims : 0);
  for (size_t i = 0; i < profs.size(); ++i) {
    GsBootProf &r = profs[i];
    const int32_t q = profile[i];
    r.B = q >= 0 ? h->prof_B[(size_t)q] : 0;
    r.period = q >= 0 ? h->prof_period[(size_t)q] : 0;
    r.off = q >= 0 ? h->prof_off[(size_t)q] : 0;
    r.nseg = q >= 0 ? h->prof_nseg[(size_t)q] : 0;
    r.reserved = 0;
  }
  CU(cudaSetDevice(h->device));
  int rc = reserve_trace_arena(h, nmax);
  if (rc) return rc;
  const size_t off_out = align_up(sizeof(GsBootRep) * reps.size()), off_mix = align_up(off_out + 16 * reps.size());
  const size_t off_prof = align_up(off_mix + sizeof(GsBootMix) * mixes.size());
  rc = ensure_scratch(h, profiled ? off_prof + sizeof(GsBootProf) * profs.size()
                                  : mixed ? off_mix + sizeof(GsBootMix) * mixes.size() : off_out + 16 * reps.size());
  if (rc) return rc;
  unsigned char *d = (unsigned char *)h->d_scratch;
  std::vector<long long> res(2 * reps.size());
  const JobIn *pop = (const JobIn *)h->d_pop;
  const int *gaps = (const int *)((unsigned char *)h->d_pop + align_up(sizeof(JobIn) * (size_t)h->pop_k));
  CU(cudaMemcpyAsync(d, reps.data(), sizeof(GsBootRep) * reps.size(), cudaMemcpyHostToDevice, h->stream));
  if (mixed) CU(cudaMemcpyAsync(d + off_mix, mixes.data(), sizeof(GsBootMix) * mixes.size(), cudaMemcpyHostToDevice, h->stream));
  if (profiled) CU(cudaMemcpyAsync(d + off_prof, profs.data(), sizeof(GsBootProf) * profs.size(), cudaMemcpyHostToDevice, h->stream));
  CU(cudaEventRecord(h->e0, h->stream));
  const long long stride = (long long)(h->tarena_stride / sizeof(JobIn));
  using MixT = const GsBootMix *;
  using TabT = const GsBootAlias *;
  using ProfT = const GsBootProf *;
  using SegT = const GsBootProfSeg *;
  if (profiled && mixed)
    (blocked ? gs_boot_kernel<true, true, MixT, TabT, ProfT, SegT> : gs_boot_kernel<false, true, MixT, TabT, ProfT, SegT>)
        <<<(unsigned)h->nsims, GS_BOOT_THREADS, 0, h->stream>>>((const GsBootRep *)d, pop, gaps, (long long)h->pop_k, (JobIn *)h->tarena, stride,
                                                               (long long *)(d + off_out), (MixT)(d + off_mix), h->d_mix,
                                                               (ProfT)(d + off_prof), h->d_prof);
  else if (profiled)
    (blocked ? gs_boot_kernel<true, false, ProfT, SegT> : gs_boot_kernel<false, false, ProfT, SegT>)
        <<<(unsigned)h->nsims, GS_BOOT_THREADS, 0, h->stream>>>((const GsBootRep *)d, pop, gaps, (long long)h->pop_k, (JobIn *)h->tarena, stride,
                                                               (long long *)(d + off_out), (ProfT)(d + off_prof), h->d_prof);
  else if (mixed)
    (blocked ? gs_boot_kernel<true, true, const GsBootMix *, const GsBootAlias *> : gs_boot_kernel<false, true, const GsBootMix *, const GsBootAlias *>)
        <<<(unsigned)h->nsims, GS_BOOT_THREADS, 0, h->stream>>>((const GsBootRep *)d, pop, gaps, (long long)h->pop_k, (JobIn *)h->tarena, stride,
                                                               (long long *)(d + off_out), (const GsBootMix *)(d + off_mix), h->d_mix);
  else
    (blocked ? gs_boot_kernel<true, false> : gs_boot_kernel<false, false>)<<<(unsigned)h->nsims, GS_BOOT_THREADS, 0, h->stream>>>(
        (const GsBootRep *)d, pop, gaps, (long long)h->pop_k, (JobIn *)h->tarena, stride, (long long *)(d + off_out));
  CU(cudaGetLastError());
  h->launches += 1;
  CU(cudaEventRecord(h->e1, h->stream));
  CU(cudaMemcpyAsync(res.data(), d + off_out, 16 * reps.size(), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  float ms = 0; cudaEventElapsedTime(&ms, h->e0, h->e1);
  if (kernel_ms) *kernel_ms = ms;
  for (int i = 0; i < h->nsims; ++i) bind_arena_trace(h, i, params[i].n, res[2 * (size_t)i], h->pop_max_need, res[2 * (size_t)i + 1]);
  h->dirty = true;
  return GS_OK;
}

extern "C" int gs_fetch_trace(gs_handle h, int sim, gs_jobin *out) {
  if (!h) return GS_ERR_ARG;
  if (sim < 0 || sim >= h->nsims) return fail(h, GS_ERR_ARG, "gs_fetch_trace: sim index out of range");
  const SimHost &s = h->sims[(size_t)sim];
  if (!s.loaded) return fail(h, GS_ERR_STATE, "gs_fetch_trace: the replica holds no trace");
  if (s.n > 0 && !out) return fail(h, GS_ERR_ARG, "gs_fetch_trace: NULL output");
  CU(cudaSetDevice(h->device));
  return timed_d2h(h, out, s.dev.jobs, sizeof(JobIn) * (size_t)s.n);
}

extern "C" int gs_place_batch(gs_handle h, const gs_cluster *cluster, const gs_node *nodes, int32_t m,
                              const gs_jobreq *jobs, int64_t b, int32_t *first_node, int32_t *nodes_used,
                              const int64_t *task_off, int32_t *task_node, double *kernel_ms) {
  if (!h) return GS_ERR_ARG;
  int rc = check_cluster(h, cluster);
  if (rc) return rc;
  if (!nodes || m <= 0 || m > 16384 || b < 0 || (b > 0 && (!jobs || !first_node)))
    return fail(h, GS_ERR_ARG, "gs_place_batch: bad arguments (1 <= m <= 16384)");
  if ((task_node != nullptr) != (task_off != nullptr))
    return fail(h, GS_ERR_ARG, "gs_place_batch: task_off and task_node go together");
  for (int64_t j = 0; j < b; ++j)
    if (jobs[j].gpu_per_task <= 0 || jobs[j].gpus < jobs[j].gpu_per_task || jobs[j].gpus % jobs[j].gpu_per_task)
      return fail(h, GS_ERR_ARG, "gs_place_batch: gpus must be a positive multiple of gpu_per_task");
  if (b == 0) return GS_OK;
  CU(cudaSetDevice(h->device));
  const int64_t ntask = task_off ? task_off[b] : 0;
  size_t o_nodes = 0, o_jobs = align_up(o_nodes + 16 * (size_t)m), o_first = align_up(o_jobs + 16 * (size_t)b);
  size_t o_used = align_up(o_first + 4 * (size_t)b), o_toff = align_up(o_used + 4 * (size_t)b);
  size_t o_tn = align_up(o_toff + 8 * (size_t)(b + 1)), total = align_up(o_tn + 4 * (size_t)(ntask > 0 ? ntask : 1));
  rc = ensure_scratch(h, total);
  if (rc) return rc;
  unsigned char *d = (unsigned char *)h->d_scratch;
  CU(cudaEventRecord(h->e0, h->stream));
  CU(cudaMemcpyAsync(d + o_nodes, nodes, 16 * (size_t)m, cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(d + o_jobs, jobs, 16 * (size_t)b, cudaMemcpyHostToDevice, h->stream));
  if (task_off) CU(cudaMemcpyAsync(d + o_toff, task_off, 8 * (size_t)(b + 1), cudaMemcpyHostToDevice, h->stream));
  CU(cudaEventRecord(h->e1, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  float ms = 0; cudaEventElapsedTime(&ms, h->e0, h->e1); h->h2d_ms += ms;
  int dev_sms = 132;
  cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, h->device);
  long long want = (b + 255) / 256;
  int grid = (int)(want < (long long)dev_sms * 8 ? want : (long long)dev_sms * 8);
  const long long fit_limit = ((long long)cluster->gpu_mem_cap_mib << 20) - ((long long)500 << 20);
  CU(cudaEventRecord(h->e0, h->stream));
  const size_t place_smem = 12 * (size_t)m + 4 * (GS_MAX_GPUS_PER_NODE + 1);
  if (place_smem > 48 * 1024)
    CU(cudaFuncSetAttribute(gs_place_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)place_smem));
  gs_place_kernel<<<grid, 256, place_smem, h->stream>>>(
      (const uint4 *)(d + o_nodes), m, cluster->num_gpu_p_node, cluster->num_cpu_p_node, cluster->mem_p_node,
      cluster->cpu_per_task, cluster->mem_per_task, fit_limit, (const uint4 *)(d + o_jobs), (long long)b,
      (int *)(d + o_first), (int *)(d + o_used), task_off ? (const long long *)(d + o_toff) : nullptr,
      task_node ? (int *)(d + o_tn) : nullptr);
  CU(cudaGetLastError());
  h->launches += 1;
  CU(cudaEventRecord(h->e1, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  cudaEventElapsedTime(&ms, h->e0, h->e1);
  h->kernel_ms += ms;
  if (kernel_ms) *kernel_ms = ms;
  rc = timed_d2h(h, first_node, d + o_first, 4 * (size_t)b);
  if (rc == GS_OK && nodes_used) rc = timed_d2h(h, nodes_used, d + o_used, 4 * (size_t)b);
  if (rc == GS_OK && task_node && ntask > 0) rc = timed_d2h(h, task_node, d + o_tn, 4 * (size_t)ntask);
  return rc;
}

extern "C" int gs_net_cost(gs_handle h, const gs_cluster *cluster, int64_t b, const int64_t *task_off,
                           const int32_t *task_node, const uint8_t *is_ps, const int32_t *ps_count,
                           const double *model_mb, const double *iterations, double *extra_out) {
  if (!h) return GS_ERR_ARG;
  if (!cluster || b < 0 || (b > 0 && (!task_off || !task_node || !ps_count || !model_mb || !iterations || !extra_out)))
    return fail(h, GS_ERR_ARG, "gs_net_cost: bad arguments");
  if (b == 0) return GS_OK;
  CU(cudaSetDevice(h->device));
  const int64_t nt = task_off[b];
  size_t o_off = 0, o_tn = align_up(o_off + 8 * (size_t)(b + 1)), o_ps = align_up(o_tn + 4 * (size_t)(nt > 0 ? nt : 1));
  size_t o_cnt = align_up(o_ps + (size_t)(nt > 0 ? nt : 1)), o_mm = align_up(o_cnt + 4 * (size_t)b);
  size_t o_it = align_up(o_mm + 8 * (size_t)b), o_out = align_up(o_it + 8 * (size_t)b), total = align_up(o_out + 8 * (size_t)b);
  int rc = ensure_scratch(h, total);
  if (rc) return rc;
  unsigned char *d = (unsigned char *)h->d_scratch;
  CU(cudaMemcpyAsync(d + o_off, task_off, 8 * (size_t)(b + 1), cudaMemcpyHostToDevice, h->stream));
  if (nt > 0) CU(cudaMemcpyAsync(d + o_tn, task_node, 4 * (size_t)nt, cudaMemcpyHostToDevice, h->stream));
  if (is_ps && nt > 0) CU(cudaMemcpyAsync(d + o_ps, is_ps, (size_t)nt, cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(d + o_cnt, ps_count, 4 * (size_t)b, cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(d + o_mm, model_mb, 8 * (size_t)b, cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(d + o_it, iterations, 8 * (size_t)b, cudaMemcpyHostToDevice, h->stream));
  int dev_sms = 132;
  cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, h->device);
  long long want = (b + 3) / 4;
  int grid = (int)(want < (long long)dev_sms * 16 ? want : (long long)dev_sms * 16);
  gs_netcost_kernel<<<grid, 128, 0, h->stream>>>((long long)b, (const long long *)(d + o_off), (const int *)(d + o_tn),
                                                 is_ps ? (const unsigned char *)(d + o_ps) : nullptr,
                                                 (const int *)(d + o_cnt), (const double *)(d + o_mm),
                                                 (const double *)(d + o_it), cluster->bandwidth,
                                                 cluster->internode_latency, (double *)(d + o_out));
  CU(cudaGetLastError());
  h->launches += 1;
  return timed_d2h(h, extra_out, d + o_out, 8 * (size_t)b);
}

extern "C" int gs_switch_yarn(gs_handle h, int32_t ncl, const gs_switch_cluster *clusters, gs_switch_node *nodes, int64_t n_nodes,
                              const gs_switch_job *jobs, int64_t n_jobs, const double *ps_network, int64_t n_ps,
                              double worker_mem, double ps_mem, double p_w_mem,
                              gs_switch_ans *ans, gs_switch_span *spans, int64_t n_spans) {
  if (!h) return GS_ERR_ARG;
  if (ncl < 0 || n_nodes < 0 || n_jobs < 0 || n_ps < 0 || n_spans < 0 ||
      (ncl > 0 && (!clusters || !nodes)) || (n_jobs > 0 && (!jobs || !ans || !spans)) || (n_ps > 0 && !ps_network))
    return fail(h, GS_ERR_ARG, "gs_switch_yarn: bad arguments");
  static_assert(sizeof(gs_switch_cluster) == 40 && sizeof(gs_switch_node) == 24 && sizeof(gs_switch_job) == 32 &&
                sizeof(gs_switch_ans) == 8 && sizeof(gs_switch_span) == 32, "switch record layout");
  for (int32_t c = 0; c < ncl; ++c) {
    const gs_switch_cluster &cl = clusters[c];
    const int64_t m = (int64_t)cl.num_switch * cl.num_node_p_switch;
    if (cl.num_switch <= 0 || cl.num_node_p_switch <= 0 || cl.num_gpu_p_node <= 0 || cl.node_off < 0 || cl.node_off + m > n_nodes ||
        cl.job_off < 0 || cl.job_cnt < 0 || cl.job_off + cl.job_cnt > n_jobs)
      return fail(h, GS_ERR_ARG, "gs_switch_yarn: a cluster record points outside the tables");
    for (int64_t j = cl.job_off; j < cl.job_off + cl.job_cnt; ++j) {
      const gs_switch_job &jb = jobs[j];
      const int64_t slots = jb.num_gpu / cl.num_gpu_p_node + 1;
      if (jb.num_gpu <= 0 || jb.n_ps < 0 || jb.ps_off < 0 || jb.ps_off + jb.n_ps > n_ps || jb.span_off < 0 || jb.span_off + slots > n_spans)
        return fail(h, GS_ERR_ARG, "gs_switch_yarn: a job record points outside the tables (spans need num_gpu / G + 1 slots)");
    }
  }
  if (ncl == 0 || n_jobs == 0) return GS_OK;
  CU(cudaSetDevice(h->device));
  size_t total = 0;
  auto take = [&](size_t bytes) { const size_t o = total; total = align_up(total + (bytes ? bytes : 1)); return o; };
  const size_t o_cl = take(sizeof(gs_switch_cluster) * (size_t)ncl), o_nd = take(sizeof(gs_switch_node) * (size_t)n_nodes);
  const size_t o_jb = take(sizeof(gs_switch_job) * (size_t)n_jobs), o_ps = take(8 * (size_t)n_ps);
  const size_t o_an = take(sizeof(gs_switch_ans) * (size_t)n_jobs), o_sp = take(sizeof(gs_switch_span) * (size_t)n_spans);
  int rc = ensure_scratch(h, total);
  if (rc) return rc;
  unsigned char *d = (unsigned char *)h->d_scratch;
  CU(cudaMemcpyAsync(d + o_cl, clusters, sizeof(gs_switch_cluster) * (size_t)ncl, cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(d + o_nd, nodes, sizeof(gs_switch_node) * (size_t)n_nodes, cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(d + o_jb, jobs, sizeof(gs_switch_job) * (size_t)n_jobs, cudaMemcpyHostToDevice, h->stream));
  if (n_ps > 0) CU(cudaMemcpyAsync(d + o_ps, ps_network, 8 * (size_t)n_ps, cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemsetAsync(d + o_sp, 0, sizeof(gs_switch_span) * (size_t)n_spans, h->stream));
  CU(cudaEventRecord(h->e0, h->stream));
  gs_switch_yarn_kernel<<<(unsigned)ncl, 32, 0, h->stream>>>(ncl, (const gs_switch_cluster *)(d + o_cl), (gs_switch_node *)(d + o_nd),
                                                            (const gs_switch_job *)(d + o_jb), (const double *)(d + o_ps),
                                                            worker_mem, ps_mem, p_w_mem, (gs_switch_ans *)(d + o_an), (gs_switch_span *)(d + o_sp));
  CU(cudaGetLastError());
  h->launches += 1;
  CU(cudaEventRecord(h->e1, h->stream));
  CU(cudaMemcpyAsync(nodes, d + o_nd, sizeof(gs_switch_node) * (size_t)n_nodes, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaMemcpyAsync(ans, d + o_an, sizeof(gs_switch_ans) * (size_t)n_jobs, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaMemcpyAsync(spans, d + o_sp, sizeof(gs_switch_span) * (size_t)n_spans, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  float ms = 0; cudaEventElapsedTime(&ms, h->e0, h->e1);
  h->kernel_ms += ms;
  return GS_OK;
}

// Restart every replica from tick 0 on the traces already resident in HBM.
extern "C" int gs_reset(gs_handle h) {
  if (!h) return GS_ERR_ARG;
  for (auto &s : h->sims) s.prepared = false;
  h->dirty = true;
  h->kernel_ms = h->h2d_ms = h->d2h_ms = 0;
  return GS_OK;
}

extern "C" int64_t gs_launch_count(gs_handle h) { return h ? h->launches : 0; }

// Span-pool sizing.  Default (0): the worst case sum(min(tasks, nodes)) per replica, which can
// never overflow.  budget > 0: min(worst case, budget * n + 4096) records -- less HBM per replica;
// a replica that would overflow stops with GS_ERR_CAPACITY instead of writing out of bounds.
extern "C" int gs_set_span_budget(gs_handle h, double spans_per_job) {
  if (!h) return GS_ERR_ARG;
  if (!(spans_per_job >= 0)) return fail(h, GS_ERR_ARG, "gs_set_span_budget: must be >= 0");
  h->span_budget = spans_per_job;
  return GS_OK;
}

// event-driven policies: 0 (or 1) = one warp per replica, 2 = one thread per replica; the fifo engine has one mapping
extern "C" int gs_set_engine(gs_handle h, int mode) {
  if (!h) return GS_ERR_ARG;
  if (mode < 0 || mode > 2) return fail(h, GS_ERR_ARG, "gs_set_engine: mode must be 0, 1 or 2");
  h->engine_mode = mode;
  return GS_OK;
}

// Pinned host buffers for callers that want DMA-speed gs_load_trace / gs_fetch_* copies.
extern "C" int gs_host_alloc(size_t bytes, void **out) {
  gs_handle h = nullptr;
  if (!out) return GS_ERR_ARG;
  *out = nullptr;
  CU(cudaMallocHost(out, bytes > 0 ? bytes : 1));
  return GS_OK;
}

extern "C" int gs_host_free(void *p) {
  gs_handle h = nullptr;
  if (p) CU(cudaFreeHost(p));
  return GS_OK;
}

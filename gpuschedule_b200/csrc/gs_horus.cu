// gs_horus.cu -- C ABI (include/gsched_horus.h) and kernel of the utilisation-aware placement engine.
// One simulation per thread (see gs_horus_core.cuh for the semantics and the reference citations).
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#define GS_HD __host__ __device__ __forceinline__
#include "gs_horus_core.cuh"
#include "gs_horus_host.h"
#include "gs_summary.cuh"

#ifdef __CUDACC__
// lanes = simulations per warp: 32 (every lane drives one) or 1 (lane 0 only: no divergence inside the warp,
// more warps in flight for the same number of replicas).
#ifndef GS_HORUS_MINBLOCKS
#define GS_HORUS_MINBLOCKS 16      // resident warps per SM the register budget is cut for (one active lane each when lanes == 1):
                                   // 128 registers, no spills
#endif
__global__ void __launch_bounds__(32, GS_HORUS_MINBLOCKS) gs_horus_kernel(HSim *sims, int nsims, long long max_ticks, int lanes) {
  const int i = lanes == 32 ? blockIdx.x * 32 + threadIdx.x : (threadIdx.x == 0 ? (int)blockIdx.x : nsims);
  if (i >= nsims) return;
  HSim s = sims[i];                 // pointers + scalars in registers / local memory
  if (s.n < 0 || s.done || s.status != 0) return;
  h_run(s, max_ticks);
  sims[i] = s;
}

// One simulation per WARP: lane 0 runs the simulation, all lanes score a candidate job's devices together
// (see "Warp-cooperative driver" in gs_horus_core.cuh).  The per-warp copy of the state lives in shared memory.
__global__ void __launch_bounds__(32) gs_horus_coop_kernel(HSim *sims, int nsims, long long max_ticks) {
  __shared__ HSim s;
  __shared__ int req;
  const int b = blockIdx.x, lane = threadIdx.x;
  if (b >= nsims) return;
  if (lane == 0) { s = sims[b]; s.budget = max_ticks > 0 ? max_ticks : 0x7fffffffffffffffLL; }
  __syncwarp();
  if (s.n < 0 || s.done || s.status != 0) return;          // uniform: every lane reads the same shared words
  for (;;) {
    if (lane == 0) req = h_coop_advance(s);
    __syncwarp();                                           // lane 0's state (shared and global) is visible to the warp
    const int r = req;
    if (r == H_REQ_DONE) break;
    if (r == H_REQ_PREP) h_coop_prep(s); else if (r == H_REQ_SCORE) h_coop_score(s); else h_coop_stats(s);
    __syncwarp();                                           // the lanes' counts / costs are visible to lane 0
  }
  if (lane == 0) { h_write_records(s); sims[b] = s; }
}

// gs_horus_summarize: every row the replica holds, [0, ticks), one block per replica (gs_summary.cuh).
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_hsum_rows_kernel(const HSim *sims, int first, gs_summary *acc) {
  const int r = first + blockIdx.x;
  const HSim &S = sims[r];
  GsSumPart p;
  gs_sum_zero(p);
  for (long long i = threadIdx.x; i < S.ticks; i += blockDim.x) gs_sum_row(p, S.rows[i], S.util[i]);
  gs_sum_block_reduce(p);
  if (threadIdx.x == 0) {
    gs_summary &A = acc[r];
    A.n = S.n; A.done = S.done; A.status = S.status;
    gs_sum_add_rows(A, p);
    if (S.ticks > 0) A.makespan = S.rows[S.ticks - 1].now;
  }
}

// Timeline of gs_horus_summarize: the same rows [0, ticks) with the sampled utilisation, into zeroed bins.
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_htl_rows_kernel(const HSim *sims, int first, gs_tbin *bins, long long W, int B) {
  const int r = first + blockIdx.x;
  const HSim &S = sims[r];
  gs_tl_fold_rows(bins + (size_t)r * (size_t)B, B, W, S.rows, S.util, 0, 0, S.ticks);
}

// Occupancy of gs_horus_summarize: the same rows [0, ticks), one tick each, into zeroed records and histograms.  The
// shared counters are static here: a dynamic shared array in this file would round every kernel's static shared memory
// up to 16 bytes.
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_occ_hsum(const HSim *sims, int first, GsOccCfg cfg, gs_occ *occ,
                                                              unsigned long long *busy, long long pitch, unsigned long long *queue) {
  __shared__ unsigned long long occ_sh[GS_OCC_SMEM_COUNTERS];
  const int r = first + blockIdx.x;
  const HSim &S = sims[r];
  unsigned long long *hall = busy + (size_t)r * 2 * (size_t)pitch, *hq = queue + (size_t)r * (size_t)(cfg.nedges + 1);
  gs_occ_fold(GS_OCC_PER_TICK, occ_sh, occ + r, nullptr, hall, hall + pitch, hq, cfg, S.M * S.G, nullptr, 0, 0, 0, S.rows, 0, 0, S.ticks, S.done);
}

#endif  // __CUDACC__

// The trace fields gs_horus_load_trace takes of job j are equal in both jobs (doubles compared bit for bit).
static __host__ __device__ inline long long gs_hjob_bits(double v) { long long u; memcpy(&u, &v, 8); return u; }
static __host__ __device__ inline bool gs_hjob_same(const HJob &x, const HJob &y) {
  return x.arrive == y.arrive && x.gpus == y.gpus && x.gpc == y.gpc && x.mem_b == y.mem_b &&
         gs_hjob_bits(x.duration) == gs_hjob_bits(y.duration) && gs_hjob_bits(x.util_avg) == gs_hjob_bits(y.util_avg) &&
         gs_hjob_bits(x.util_max) == gs_hjob_bits(y.util_max) && gs_hjob_bits(x.mem_avg_mib) == gs_hjob_bits(y.mem_avg_mib);
}

#ifdef __CUDACC__
// job(r, i) is the i-th job of the finish order, job_at(r, j) job j of the trace (meaningful once it has finished).
struct GsSumHorusJobs {
  const HSim *sims;
  __device__ long long finished(int r) const { return sims[r].nfin; }
  __device__ long long n(int r) const { return sims[r].n; }
  __device__ int order(int r, long long i) const { return sims[r].fin[i]; }
  __device__ GsSumJob job(int r, long long i) const { return job_at(r, sims[r].fin[i]); }
  __device__ int arrive_at(int r, int j) const { return sims[r].jobs[j].arrive; }
  __device__ bool same_job(int ra, int rb, int j) const { return gs_hjob_same(sims[ra].jobs[j], sims[rb].jobs[j]); }
  __device__ GsSumJob job_at(int r, int j) const {
    const HSim &S = sims[r];
    const gs_horus_job_rec rec = S.recs[j];
    return gs_sum_job(S.jobs[j].arrive, rec.start, rec.end, rec.jct, rec.preempt, S.jobs[j].gpus);
  }
  __device__ GsIfDur if_at(int r, int j) const {
    const HSim &S = sims[r];
    return GsIfDur{S.jobs[j].gpus, S.recs[j].original, S.recs[j].actual};
  }
};

#endif  // __CUDACC__

namespace {
struct WordStream {                 // raw MT19937 words + the per-position sample tables (gs_horus_host.h)
  std::vector<uint32_t> words;
  unsigned char *dev = nullptr; size_t cap = 0; bool dirty = false;
  const unsigned int *d_words = nullptr; const double *d_ret = nullptr, *d_keep = nullptr; const int *d_next = nullptr;
  const int *d_acc = nullptr, *d_rank = nullptr; int cls_off[5] = {0, 0, 0, 0, 0};
};
struct HorusSimHost {
  bool configured = false, loaded = false, prepared = false;
  bool tl_done = false;             // summarised with the timeline on since it was prepared
  bool jd_done = false;             // summarised with the current jobdist setting since it was prepared
  bool sd_done = false;             // summarised with the current slowdown setting since it was prepared
  bool arr_done = false;            // summarised with the current arrivals setting since it was prepared
  bool occ_done = false;            // summarised with the occupancy on since it was prepared
  bool if_done = false;             // summarised with the current interference setting since it was prepared
  gs_cluster cl{};
  gs_horus_params par{};
  std::vector<HJob> jobs;
  std::vector<double> stream;
  void *slab = nullptr; size_t slab_bytes = 0;
  double *d_stream = nullptr; size_t stream_cap = 0;
  HSim dev{};                       // host mirror of the device struct
  long long rows_cap = 0;
  bool use_shared = false;          // consume the handle-wide stream (gs_horus_load_stream with sim = -1)
  WordStream ws; int word_mode = 0; // 0: standard-normal values, 1: own words, 2: the handle-wide words
  std::vector<double> mem_avg;
};
}  // namespace

struct gs_horus_handle_s {
  int device = 0;
  std::vector<HorusSimHost> sims;
  HSim *d_sims = nullptr;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  float last_ms = 0.f;
  long long launches = 0;
  gs_summary *d_sum = nullptr;      // gs_horus_summarize: one record per replica
  int *d_sum_scratch = nullptr; size_t sum_scratch_bytes = 0;
  gs_tbin *d_tl = nullptr; size_t tl_bytes = 0;   // gs_horus_set_timeline: nsims x tl_nbins bins
  int64_t tl_width = 0; int tl_nbins = 0;
  gs_jclass *d_jd = nullptr; size_t jd_bytes = 0;       // gs_horus_set_jobdist: nsims x C class records
  unsigned *d_jd_hist = nullptr; size_t jd_hist_bytes = 0;   // and nsims x C x 3 x (E + 1) CDF counts
  GsJdCfg jd{};                                          // jd.nclasses = 0: off
  gs_sdclass *d_sd = nullptr; size_t sd_bytes = 0;      // gs_horus_set_slowdown: nsims x C class records
  unsigned *d_sd_hist = nullptr; size_t sd_hist_bytes = 0;   // and nsims x C x (3 (E + 1) + Esd + 1) CDF counts
  GsSdCfg sd{};                                          // sd.nclasses = 0: off
  gs_abin *d_arr = nullptr; size_t arr_bytes = 0;       // gs_horus_set_arrivals: nsims x B bin records, only while on
  GsArrCfg arr{};                                        // arr.nbins = 0: off
  bool occ_on = false; GsOccCfg occ{};                   // gs_horus_set_occupancy
  gs_occ *d_occ = nullptr;                               // nsims records
  unsigned long long *d_occ_busy = nullptr; int64_t occ_pitch = 0;   // nsims x [H_all, H_wait] x occ_pitch counters
  unsigned long long *d_occ_q = nullptr; size_t occ_q_bytes = 0;     // nsims x (E + 1) queue counters
  gs_ifclass *d_if = nullptr; size_t if_bytes = 0;      // gs_horus_set_interference: nsims x C class records
  GsJdCfg ifc{};                                         // ifc.nclasses = 0: off (bounds only)
  std::string err;
  std::vector<double> shared;       // one stream consumed by every replica that did not get its own
  double *d_shared = nullptr; size_t shared_cap = 0; bool shared_dirty = false;
  int lanes = 1;                    // simulations per warp (gs_horus_set_lanes)
  WordStream shared_ws;
};

static std::string g_horus_create_err;
static int hfail(gs_horus_handle h, int code, const std::string &msg) { if (h) h->err = msg; else g_horus_create_err = msg; return code; }
#define HCU(call)                                                                              \
  do {                                                                                         \
    cudaError_t e_ = (call);                                                                   \
    if (e_ != cudaSuccess) return hfail(h, GS_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
  } while (0)

static size_t up(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" int gs_horus_create(int device, int nsims, gs_horus_handle *out) {
  gs_horus_handle h = nullptr;
  if (!out || nsims <= 0) return hfail(nullptr, GS_ERR_ARG, "gs_horus_create: bad arguments");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev <= 0) return hfail(nullptr, GS_ERR_CUDA, "gs_horus_create: no CUDA device (this library has no CPU path)");
  if (device < 0 || device >= ndev) return hfail(nullptr, GS_ERR_ARG, "gs_horus_create: device out of range");
  h = new gs_horus_handle_s();
  h->device = device;
  h->sims.resize((size_t)nsims);
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreate(&h->ev0) != cudaSuccess || cudaEventCreate(&h->ev1) != cudaSuccess ||
      cudaMalloc(&h->d_sims, sizeof(HSim) * (size_t)nsims) != cudaSuccess) {
    delete h;
    return hfail(nullptr, GS_ERR_CUDA, "gs_horus_create: CUDA initialisation failed");
  }
  size_t stack = 0;                 // the scalar kernel keeps ~1.5 KB of per-thread state on its stack frame
  if (cudaDeviceGetLimit(&stack, cudaLimitStackSize) == cudaSuccess && stack < 4096) (void)cudaDeviceSetLimit(cudaLimitStackSize, 4096);
  *out = h;
  return GS_OK;
}

extern "C" int gs_horus_destroy(gs_horus_handle h) {
  if (!h) return GS_ERR_ARG;
  cudaSetDevice(h->device);
  for (auto &s : h->sims) { if (s.slab) cudaFree(s.slab); if (s.d_stream) cudaFree(s.d_stream); if (s.ws.dev) cudaFree(s.ws.dev); }
  if (h->d_shared) cudaFree(h->d_shared);
  if (h->shared_ws.dev) cudaFree(h->shared_ws.dev);
  if (h->d_sims) cudaFree(h->d_sims);
  if (h->d_sum) cudaFree(h->d_sum);
  if (h->d_sum_scratch) cudaFree(h->d_sum_scratch);
  if (h->d_tl) cudaFree(h->d_tl);
  if (h->d_jd) cudaFree(h->d_jd);
  if (h->d_jd_hist) cudaFree(h->d_jd_hist);
  if (h->d_sd) cudaFree(h->d_sd);
  if (h->d_sd_hist) cudaFree(h->d_sd_hist);
  if (h->d_arr) cudaFree(h->d_arr);
  if (h->d_occ) cudaFree(h->d_occ);
  if (h->d_occ_busy) cudaFree(h->d_occ_busy);
  if (h->d_occ_q) cudaFree(h->d_occ_q);
  if (h->d_if) cudaFree(h->d_if);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return GS_OK;
}

extern "C" const char *gs_horus_build_tag(void) {
#ifdef __CUDACC__
  return "cuda:sm_90a";
#else
  return "host-emulation";
#endif
}
extern "C" const char *gs_horus_last_error(gs_horus_handle h) { return h ? h->err.c_str() : g_horus_create_err.c_str(); }
extern "C" int64_t gs_horus_launch_count(gs_horus_handle h) { return h ? h->launches : 0; }
extern "C" int gs_horus_set_lanes(gs_horus_handle h, int lanes) {
  if (!h || (lanes != 0 && lanes != 1 && lanes != 32)) return hfail(h, GS_ERR_ARG, "gs_horus_set_lanes: 0 (cooperative warp), 1 or 32");
  h->lanes = lanes;
  return GS_OK;
}

extern "C" int gs_horus_config(gs_horus_handle h, int32_t sim, const gs_cluster *c, const gs_horus_params *p) {
  if (!h || !c || !p || sim < 0 || sim >= (int)h->sims.size()) return hfail(h, GS_ERR_ARG, "gs_horus_config: bad arguments");
  if (c->num_switch <= 0 || c->num_node_p_switch <= 0 || c->num_gpu_p_node <= 0 || c->num_gpu_p_node > 64)
    return hfail(h, GS_ERR_ARG, "gs_horus_config: bad cluster shape");
  if (p->score != GS_HSCORE_HORUS && p->score != GS_HSCORE_GANDIVA) return hfail(h, GS_ERR_ARG, "gs_horus_config: unknown score function");
  if (p->schedule != GS_HSCHED_HORUS && p->schedule != GS_HSCHED_HORUS_PLUS && p->schedule != GS_HSCHED_GANDIVA)
    return hfail(h, GS_ERR_ARG, "gs_horus_config: schedule must be horus, horus+ or gandiva (with fifo the reference raises KeyError in score_fn, algorithm.py:58)");
  if ((p->schedule == GS_HSCHED_GANDIVA) != (p->score == GS_HSCORE_GANDIVA))
    return hfail(h, GS_ERR_ARG, "gs_horus_config: the score function follows the schedule name (gandiva_score <=> schedule gandiva)");
  if (p->schedule == GS_HSCHED_HORUS_PLUS && (p->num_queue < 1 || p->num_queue > H_MAXQ))
    return hfail(h, GS_ERR_ARG, "gs_horus_config: horus+ needs 1..8 queues");
  if (p->placement != GS_HPLACE_HORUS && p->placement != GS_HPLACE_YARN) return hfail(h, GS_ERR_ARG, "gs_horus_config: unknown placement");
  if (c->enable_network_costs) return hfail(h, GS_ERR_ARG, "gs_horus_config: network costs are not part of this path");
  auto &s = h->sims[(size_t)sim];
  s.cl = *c; s.par = *p; s.configured = true; s.prepared = false;
  return GS_OK;
}

extern "C" int gs_horus_load_trace(gs_horus_handle h, int32_t sim, int64_t n, const int32_t *arrive, const int32_t *gpus,
                                   const int32_t *gpc, const double *duration, const int64_t *mem_bytes,
                                   const double *util_avg, const double *util_max, const double *mem_avg_mib) {
  if (!h || sim < 0 || sim >= (int)h->sims.size() || n < 0 || n > 0x3fffffff) return hfail(h, GS_ERR_ARG, "gs_horus_load_trace: bad arguments");
  if (n > 0 && (!arrive || !gpus || !gpc || !duration || !mem_bytes || !util_avg || !util_max)) return hfail(h, GS_ERR_ARG, "gs_horus_load_trace: null column");
  auto &s = h->sims[(size_t)sim];
  std::vector<HJob> jobs((size_t)n);     // validated into a temporary: a rejected trace leaves the replica as it was
  long long first = 0;
  for (int64_t j = 0; j < n; ++j) {
    if (gpc[j] <= 0 || gpus[j] < gpc[j] || gpus[j] % gpc[j] != 0) return hfail(h, GS_ERR_ARG, "gs_horus_load_trace: used_gpus must be a positive multiple of gpu_per_container");
    if (j > 0 && arrive[j] < arrive[j - 1]) return hfail(h, GS_ERR_ARG, "gs_horus_load_trace: rows must be in admission order");
    if (util_max[j] < util_avg[j]) return hfail(h, GS_ERR_ARG, "gs_horus_load_trace: gpu_utilization_max < avg (numpy raises on a negative scale)");
    HJob &o = jobs[(size_t)j];
    o.arrive = arrive[j]; o.gpus = gpus[j]; o.gpc = gpc[j]; o.ntasks = gpus[j] / gpc[j]; o.first_task = (int)first; o.pad = 0;
    o.mem_b = mem_bytes[j]; o.util_avg = util_avg[j]; o.util_max = util_max[j]; o.duration = duration[j];
    o.mem_avg_mib = mem_avg_mib ? mem_avg_mib[j] : 0.0;
    first += o.ntasks;
    if (first > 0x3fffffff) return hfail(h, GS_ERR_ARG, "gs_horus_load_trace: too many tasks");
  }
  s.jobs.swap(jobs);
  s.loaded = true; s.prepared = false;
  return GS_OK;
}

extern "C" int gs_horus_load_stream(gs_horus_handle h, int32_t sim, const double *g, int64_t count) {
  if (!h || sim < -1 || sim >= (int)h->sims.size() || count < 0 || (count > 0 && !g)) return hfail(h, GS_ERR_ARG, "gs_horus_load_stream: bad arguments");
  if (sim == -1) {                  // every replica reads the same samples (each from position 0)
    h->shared.assign(g, g + count); h->shared_dirty = true;
    for (auto &s : h->sims) { s.use_shared = true; s.stream.clear(); s.prepared = false; s.word_mode = 0; }
    return GS_OK;
  }
  auto &s = h->sims[(size_t)sim];
  s.stream.assign(g, g + count);
  s.use_shared = false; s.prepared = false; s.word_mode = 0;
  return GS_OK;
}

extern "C" int gs_horus_load_words(gs_horus_handle h, int32_t sim, const uint32_t *w, int64_t count) {
  if (!h || sim < -1 || sim >= (int)h->sims.size() || count < 0 || count > 0x7ffffff0 || (count > 0 && !w)) return hfail(h, GS_ERR_ARG, "gs_horus_load_words: bad arguments");
  if (sim == -1) {
    h->shared_ws.words.assign(w, w + count); h->shared_ws.dirty = true;
    for (auto &s : h->sims) { s.word_mode = 2; s.prepared = false; }
    return GS_OK;
  }
  auto &s = h->sims[(size_t)sim];
  s.ws.words.assign(w, w + count); s.ws.dirty = true;
  s.word_mode = 1; s.prepared = false;
  return GS_OK;
}

static int upload_words(gs_horus_handle h, WordStream &ws) {
  if (!ws.dirty) return GS_OK;
  const size_t n = ws.words.size(), N = n ? n : 1;
  const size_t o_w = 0, o_ret = up(4 * N), o_keep = up(o_ret + 8 * N), o_next = up(o_keep + 8 * N), o_acc = up(o_next + 4 * N);
  const size_t o_rank = up(o_acc + 4 * N), total = up(o_rank + 4 * N);
  if (ws.dev && ws.cap < total) { cudaFree(ws.dev); ws.dev = nullptr; }
  if (!ws.dev) { HCU(cudaMalloc(&ws.dev, total)); ws.cap = total; }
  std::vector<double> ret(N), keep(N); std::vector<int> next(N);
  std::vector<int> acc(N), rank(N);
  gs_horus_build_gauss_tables(ws.words.data(), (long long)n, ret.data(), keep.data(), next.data());
  gs_horus_build_gauss_index(next.data(), (long long)n, acc.data(), rank.data(), ws.cls_off);
  if (n) {
    HCU(cudaMemcpyAsync(ws.dev + o_acc, acc.data(), 4 * n, cudaMemcpyHostToDevice, h->stream));
    HCU(cudaMemcpyAsync(ws.dev + o_rank, rank.data(), 4 * n, cudaMemcpyHostToDevice, h->stream));
    HCU(cudaMemcpyAsync(ws.dev + o_w, ws.words.data(), 4 * n, cudaMemcpyHostToDevice, h->stream));
    HCU(cudaMemcpyAsync(ws.dev + o_ret, ret.data(), 8 * n, cudaMemcpyHostToDevice, h->stream));
    HCU(cudaMemcpyAsync(ws.dev + o_keep, keep.data(), 8 * n, cudaMemcpyHostToDevice, h->stream));
    HCU(cudaMemcpyAsync(ws.dev + o_next, next.data(), 4 * n, cudaMemcpyHostToDevice, h->stream));
  }
  HCU(cudaStreamSynchronize(h->stream));
  ws.d_words = (const unsigned int *)(ws.dev + o_w); ws.d_ret = (const double *)(ws.dev + o_ret);
  ws.d_keep = (const double *)(ws.dev + o_keep); ws.d_next = (const int *)(ws.dev + o_next);
  ws.d_acc = (const int *)(ws.dev + o_acc); ws.d_rank = (const int *)(ws.dev + o_rank);
  ws.dirty = false;
  return GS_OK;
}

static int prepare(gs_horus_handle h, HorusSimHost &s, long long rows_cap) {
  const gs_cluster &c = s.cl;
  const int M = c.num_switch * c.num_node_p_switch, G = c.num_gpu_p_node;
  const size_t n = s.jobs.size(), N = n ? n : 1;
  long long ntask = 0; int maxg = 1;
  for (auto &j : s.jobs) { ntask += j.ntasks; maxg = std::max(maxg, j.gpus); }
  const size_t NT = ntask ? (size_t)ntask : 1;
  const int pjw = (M + 63) / 64;
  const int nb = std::max(1, s.par.num_buffer);
  const int nq = s.par.schedule == GS_HSCHED_HORUS_PLUS ? std::max(1, s.par.num_queue) : 1;
  if (s.par.schedule == GS_HSCHED_HORUS_PLUS && s.word_mode == 0)
    return hfail(h, GS_ERR_STATE, "gs_horus_run: horus+ draws integers too: load the raw stream with gs_horus_load_words");
  if (s.word_mode == 1) { int rc = upload_words(h, s.ws); if (rc) return rc; }
  if (rows_cap <= 0) return hfail(h, GS_ERR_ARG, "gs_horus_run: rows_cap must be positive");
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = up(off + bytes); return o; };
  const size_t o_jobs = take(sizeof(HJob) * N), o_js = take(sizeof(HJobState) * N), o_tasks = take(sizeof(HTask) * NT);
  const size_t o_tron = take(4 * NT), o_troo = take(4 * NT), o_nodes = take(sizeof(HNode) * (size_t)M), o_devs = take(sizeof(HDev) * (size_t)M * G);
  const size_t o_pj = take(8 * N * (size_t)pjw), o_q = take(4 * (N + 1) * (size_t)nq), o_run = take(4 * N), o_fin = take(4 * N);
  const size_t o_look = take(4 * (size_t)nb), o_lookq = take(4 * (size_t)nb), o_work = take(4 * N), o_res = take(4 * (size_t)M);
  const size_t o_kall = take(4 * N), o_kas = take(4 * N), o_kold = take(4 * N), o_ksc = take(8 * N);
  const size_t o_sccnt = take(4 * (size_t)M * G), o_scoff = take(4 * (size_t)M * G), o_sccost = take(8 * (size_t)M * G);
  const size_t o_mn = take(4 * (size_t)maxg * maxg), o_mo = take(4 * (size_t)maxg * maxg), o_mc = take(4 * (size_t)maxg);
  const size_t o_ok = take(4 * (size_t)maxg), o_di = take(4 * (size_t)maxg), o_heap = take(sizeof(HCand) * ((size_t)maxg + 2));
  const size_t o_mskip = take(8 * (size_t)maxg);
  const size_t o_rows = take(sizeof(gs_tick_row) * (size_t)rows_cap), o_util = take(8 * (size_t)rows_cap), o_ua = take((size_t)rows_cap);
  const size_t o_recs = take(sizeof(gs_horus_job_rec) * N);
  const size_t total = off;
  if (s.slab && s.slab_bytes < total) { cudaFree(s.slab); s.slab = nullptr; }
  if (!s.slab) { HCU(cudaMalloc(&s.slab, total)); s.slab_bytes = total; }
  HCU(cudaMemsetAsync(s.slab, 0, total, h->stream));
  unsigned char *d = (unsigned char *)s.slab;
  if (n) HCU(cudaMemcpyAsync(d + o_jobs, s.jobs.data(), sizeof(HJob) * n, cudaMemcpyHostToDevice, h->stream));
  std::vector<HTask> tasks(NT);
  std::vector<int> tron(NT, -1);
  gs_horus_init_tasks(s.jobs.data(), (long long)n, (long long)c.gpu_mem_cap_mib << 20, tasks.data());
  HCU(cudaMemcpyAsync(d + o_tasks, tasks.data(), sizeof(HTask) * NT, cudaMemcpyHostToDevice, h->stream));
  HCU(cudaMemcpyAsync(d + o_tron, tron.data(), 4 * NT, cudaMemcpyHostToDevice, h->stream));
  if (s.stream.size() > s.stream_cap) {
    if (s.d_stream) cudaFree(s.d_stream);
    s.d_stream = nullptr;
    HCU(cudaMalloc(&s.d_stream, 8 * s.stream.size()));
    s.stream_cap = s.stream.size();
  }
  if (!s.stream.empty()) HCU(cudaMemcpyAsync(s.d_stream, s.stream.data(), 8 * s.stream.size(), cudaMemcpyHostToDevice, h->stream));
  HCU(cudaStreamSynchronize(h->stream));            // the staging vectors go out of scope below
  HSim &D = s.dev;
  D = HSim{};
  D.M = M; D.G = G; D.S = c.num_switch; D.P = c.num_node_p_switch; D.cpu_cap = c.num_cpu_p_node; D.mem_cap = c.mem_p_node;
  D.placement = s.par.placement;
  D.scheme = s.par.score; D.schedule = s.par.schedule; D.num_buffer = s.par.num_buffer; D.n = (int)n; D.maxg = maxg; D.pjw = pjw;
  D.cap_b = (long long)c.gpu_mem_cap_mib << 20;
  D.jobs = (const HJob *)(d + o_jobs); D.js = (HJobState *)(d + o_js); D.tasks = (HTask *)(d + o_tasks);
  D.tro_node = (int *)(d + o_tron); D.tro_order = (int *)(d + o_troo); D.nodes = (HNode *)(d + o_nodes); D.devs = (HDev *)(d + o_devs);
  D.pj_bits = (unsigned long long *)(d + o_pj); D.queue = (int *)(d + o_q); D.running = (int *)(d + o_run); D.fin = (int *)(d + o_fin);
  D.look = (int *)(d + o_look); D.look_q = (int *)(d + o_lookq); D.work = (int *)(d + o_work); D.res_nodes = (int *)(d + o_res);
  D.km_all = (int *)(d + o_kall); D.km_assign = (int *)(d + o_kas); D.km_old = (int *)(d + o_kold); D.km_score = (double *)(d + o_ksc);
  D.nq = nq;
  D.sc_cnt = (int *)(d + o_sccnt); D.sc_off = (int *)(d + o_scoff); D.sc_cost = (double *)(d + o_sccost);
  if (s.word_mode) {
    const WordStream &ws = s.word_mode == 1 ? s.ws : h->shared_ws;
    D.words = ws.d_words; D.gv_ret = ws.d_ret; D.gv_keep = ws.d_keep; D.gv_next = ws.d_next; D.words_n = (long long)ws.words.size();
    D.gv_acc = ws.d_acc; D.gv_rank = ws.d_rank; for (int c = 0; c < 5; ++c) D.gv_cls_off[c] = ws.cls_off[c];
  }
  D.map_node = (int *)(d + o_mn); D.map_order = (int *)(d + o_mo); D.map_n = (int *)(d + o_mc); D.ok = (int *)(d + o_ok); D.distinct = (int *)(d + o_di);
  D.heap = (HCand *)(d + o_heap); D.map_skip = (long long *)(d + o_mskip);
  D.gauss = s.use_shared ? h->d_shared : s.d_stream;
  D.gauss_n = (long long)(s.use_shared ? h->shared.size() : s.stream.size()); D.gauss_pos = 0;
  D.rows = (gs_tick_row *)(d + o_rows); D.util = (double *)(d + o_util); D.util_arr = d + o_ua; D.recs = (gs_horus_job_rec *)(d + o_recs);
  D.rows_cap = rows_cap;
  D.current_remaining = (long long)n; D.running_jobs = 0;
  s.rows_cap = rows_cap;
  s.prepared = true; s.tl_done = false; s.jd_done = false; s.sd_done = false; s.arr_done = false; s.occ_done = false; s.if_done = false;
  return GS_OK;
}

extern "C" int gs_horus_run(gs_horus_handle h, int64_t max_ticks, int64_t rows_cap) {
  if (!h) return GS_ERR_ARG;
  HCU(cudaSetDevice(h->device));
  const int nsims = (int)h->sims.size();
  std::vector<HSim> host((size_t)nsims);
  if (h->shared_dirty) {
    if (h->shared.size() > h->shared_cap) {
      if (h->d_shared) cudaFree(h->d_shared);
      h->d_shared = nullptr;
      HCU(cudaMalloc(&h->d_shared, 8 * h->shared.size()));
      h->shared_cap = h->shared.size();
    }
    if (!h->shared.empty()) HCU(cudaMemcpyAsync(h->d_shared, h->shared.data(), 8 * h->shared.size(), cudaMemcpyHostToDevice, h->stream));
    HCU(cudaStreamSynchronize(h->stream));
    h->shared_dirty = false;
    for (auto &s : h->sims) if (s.use_shared) s.prepared = false;          // the buffer may have moved
  }
  if (h->shared_ws.dirty) {
    int rc = upload_words(h, h->shared_ws); if (rc) return rc;
    for (auto &s : h->sims) if (s.word_mode == 2) s.prepared = false;
  }
  for (int i = 0; i < nsims; ++i) {
    auto &s = h->sims[(size_t)i];
    if (!s.configured || !s.loaded) return hfail(h, GS_ERR_STATE, "gs_horus_run: every replica needs gs_horus_config + gs_horus_load_trace");
    if (!s.prepared) { int rc = prepare(h, s, rows_cap); if (rc) return rc; }
    host[(size_t)i] = s.dev;
  }
  HCU(cudaMemcpyAsync(h->d_sims, host.data(), sizeof(HSim) * (size_t)nsims, cudaMemcpyHostToDevice, h->stream));
  HCU(cudaEventRecord(h->ev0, h->stream));
#ifdef __CUDACC__
  if (h->lanes == 32) gs_horus_kernel<<<(nsims + 31) / 32, 32, 0, h->stream>>>(h->d_sims, nsims, (long long)max_ticks, 32);
  else if (h->lanes == 1) gs_horus_kernel<<<nsims, 32, 0, h->stream>>>(h->d_sims, nsims, (long long)max_ticks, 1);
  else gs_horus_coop_kernel<<<nsims, 32, 0, h->stream>>>(h->d_sims, nsims, (long long)max_ticks);
#else   // host build for tests/emu (fake_cuda/cuda_runtime.h): what the kernels do, one simulation after the other
  for (int i = 0; i < nsims; ++i) {
    HSim &sm = h->d_sims[i];
    if (sm.n < 0 || sm.done || sm.status != 0) continue;
    if (h->lanes == 0) h_run_coop(sm, (long long)max_ticks); else h_run(sm, (long long)max_ticks);
  }
#endif
  h->launches += 1;
  HCU(cudaGetLastError());
  HCU(cudaEventRecord(h->ev1, h->stream));
  HCU(cudaMemcpyAsync(host.data(), h->d_sims, sizeof(HSim) * (size_t)nsims, cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaStreamSynchronize(h->stream));
  HCU(cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1));
  int worst = GS_OK;
  for (int i = 0; i < nsims; ++i) {
    h->sims[(size_t)i].dev = host[(size_t)i];
    if (host[(size_t)i].status != 0 && worst == GS_OK) worst = host[(size_t)i].status;
  }
  if (worst == GS_ERR_CAPACITY) return hfail(h, worst, "gs_horus_run: a replica ran out of rows or of random samples (raise rows_cap / load a longer stream)");
  if (worst != GS_OK) return hfail(h, worst, "gs_horus_run: a replica reached an inconsistent state");
  return GS_OK;
}

extern "C" int gs_horus_stats(gs_horus_handle h, int32_t sim, gs_horus_run_stats *out) {
  if (!h || !out || sim < 0 || sim >= (int)h->sims.size()) return hfail(h, GS_ERR_ARG, "gs_horus_stats: bad arguments");
  const HSim &D = h->sims[(size_t)sim].dev;
  out->ticks = D.ticks; out->events = D.events; out->draws = D.draws;
  int queued = 0;
  for (int q = 0; q < D.nq; ++q) queued += D.qn[q];
  out->finished = D.nfin; out->queued = queued; out->running = D.nrun; out->done = D.done; out->status = D.status; out->reserved = 0;
  out->kernel_ms = h->last_ms; out->reserved2 = 0.f;
  return GS_OK;
}

extern "C" int gs_horus_fetch(gs_horus_handle h, int32_t sim, gs_tick_row *rows, double *util, uint8_t *util_is_array,
                              int64_t rows_cap, gs_horus_job_rec *recs, int32_t *finish_order, int64_t *n_rows, int64_t *n_finished) {
  if (!h || sim < 0 || sim >= (int)h->sims.size()) return hfail(h, GS_ERR_ARG, "gs_horus_fetch: bad arguments");
  auto &s = h->sims[(size_t)sim];
  if (!s.prepared) return hfail(h, GS_ERR_STATE, "gs_horus_fetch: nothing has run");
  HCU(cudaSetDevice(h->device));
  const HSim &D = s.dev;
  if (D.ticks > rows_cap) return hfail(h, GS_ERR_CAPACITY, "gs_horus_fetch: row buffer too small");
  if (rows && D.ticks) HCU(cudaMemcpyAsync(rows, D.rows, sizeof(gs_tick_row) * (size_t)D.ticks, cudaMemcpyDeviceToHost, h->stream));
  if (util && D.ticks) HCU(cudaMemcpyAsync(util, D.util, 8 * (size_t)D.ticks, cudaMemcpyDeviceToHost, h->stream));
  if (util_is_array && D.ticks) HCU(cudaMemcpyAsync(util_is_array, D.util_arr, (size_t)D.ticks, cudaMemcpyDeviceToHost, h->stream));
  if (recs && D.n) HCU(cudaMemcpyAsync(recs, D.recs, sizeof(gs_horus_job_rec) * (size_t)D.n, cudaMemcpyDeviceToHost, h->stream));
  if (finish_order && D.nfin) HCU(cudaMemcpyAsync(finish_order, D.fin, 4 * (size_t)D.nfin, cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaStreamSynchronize(h->stream));
  if (n_rows) *n_rows = D.ticks;
  if (n_finished) *n_finished = D.nfin;
  return GS_OK;
}

extern "C" int gs_horus_summarize(gs_horus_handle h, int32_t first, int32_t count, gs_summary *out, double *kernel_ms) {
  if (!h) return GS_ERR_ARG;
  const int nsims = (int)h->sims.size();
  if (first < 0 || count < 0 || first > nsims - count || (count > 0 && !out)) return hfail(h, GS_ERR_ARG, "gs_horus_summarize: bad arguments");
  if (kernel_ms) *kernel_ms = 0.0;
  if (count == 0) return GS_OK;
  long long kmax = 1;
  for (int i = first; i < first + count; ++i) {
    if (!h->sims[(size_t)i].prepared) return hfail(h, GS_ERR_STATE, "gs_horus_summarize: a replica has not run yet");
    kmax = std::max(kmax, (long long)h->sims[(size_t)i].dev.nfin);
    if (h->occ_on && (int64_t)h->sims[(size_t)i].dev.M * h->sims[(size_t)i].dev.G > GS_OCC_MAX_GPUS)
      return hfail(h, GS_ERR_ARG, "gs_horus_summarize: the occupancy statistics take clusters of at most 65535 GPUs");
  }
  HCU(cudaSetDevice(h->device));
  if (h->occ_on) {        // the pitch of the busy histograms
    int64_t need = 1;
    for (int i = first; i < first + count; ++i) need = std::max(need, (int64_t)h->sims[(size_t)i].dev.M * h->sims[(size_t)i].dev.G + 1);
    if (need > h->occ_pitch) {                             // every replica is folded again from zero: nothing to move
      HCU(cudaStreamSynchronize(h->stream));
      if (h->d_occ_busy) cudaFree(h->d_occ_busy);
      h->d_occ_busy = nullptr; h->occ_pitch = 0;
      for (auto &s : h->sims) s.occ_done = false;
      HCU(cudaMalloc(&h->d_occ_busy, 16 * (size_t)need * h->sims.size()));
      h->occ_pitch = need;
    }
    const size_t E1 = (size_t)h->occ.nedges + 1;
    HCU(cudaMemsetAsync(h->d_occ + first, 0, sizeof(gs_occ) * (size_t)count, h->stream));
    HCU(cudaMemsetAsync(h->d_occ_busy + (size_t)first * 2 * (size_t)h->occ_pitch, 0, 16 * (size_t)h->occ_pitch * (size_t)count, h->stream));
    HCU(cudaMemsetAsync(h->d_occ_q + (size_t)first * E1, 0, 8 * E1 * (size_t)count, h->stream));
  }
  if (!h->d_sum) HCU(cudaMalloc(&h->d_sum, sizeof(gs_summary) * (size_t)nsims));
  HCU(cudaMemsetAsync(h->d_sum + first, 0, sizeof(gs_summary) * (size_t)count, h->stream));
  const int B = h->tl_nbins;
  if (B > 0) HCU(cudaMemsetAsync(h->d_tl + (size_t)first * B, 0, sizeof(gs_tbin) * (size_t)B * (size_t)count, h->stream));
  const int C = h->jd.nclasses, Csd = h->sd.nclasses, Cif = h->ifc.nclasses, Barr = h->arr.nbins;
#ifdef __CUDACC__
  int per_sm = 1, sms = 132;
  HCU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gs_sum_jobs_kernel<GsSumHorusJobs>, GS_SUM_THREADS, 0));
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
  const int grid = std::min(count, std::max(1, per_sm) * sms);
  int grid_arr = 0;
  if (Barr > 0) {
    int per_arr = 1;
    HCU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_arr, gs_arr_jobs_kernel<GsSumHorusJobs>, GS_SUM_THREADS, 0));
    grid_arr = std::min(grid, std::max(1, per_arr) * sms);
  }
  const size_t pitch = (size_t)(kmax + 63) / 64 * 64;
  const size_t need = std::max((Cif > 0 ? GS_IF_ROWS : Csd > 0 ? 4 : 3) * sizeof(int) * pitch * (size_t)grid,
                               GS_ARR_ROWS * sizeof(int) * pitch * (size_t)grid_arr);   // gs_arr_jobs_kernel: its own rows
  if (h->sum_scratch_bytes < need) {
    if (h->d_sum_scratch) { HCU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_sum_scratch); }
    h->d_sum_scratch = nullptr; h->sum_scratch_bytes = 0;
    HCU(cudaMalloc(&h->d_sum_scratch, need));
    h->sum_scratch_bytes = need;
  }
  HCU(cudaEventRecord(h->ev0, h->stream));
  gs_hsum_rows_kernel<<<(unsigned)count, GS_SUM_THREADS, 0, h->stream>>>(h->d_sims, first, h->d_sum);
  HCU(cudaGetLastError());
  gs_sum_jobs_kernel<GsSumHorusJobs><<<(unsigned)grid, GS_SUM_THREADS, 0, h->stream>>>(GsSumHorusJobs{h->d_sims}, first, count, h->d_sum,
                                                                                      h->d_sum_scratch, (long long)pitch);
  HCU(cudaGetLastError());
  h->launches += 2;
  if (C > 0) {            // after gs_sum_jobs_kernel, on the same scratch
    int per_jd = 1;
    HCU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_jd, gs_jd_jobs_kernel<GsSumHorusJobs>, GS_SUM_THREADS, 0));
    const int grid_jd = std::min(grid, std::max(1, per_jd) * sms);
    gs_jd_jobs_kernel<GsSumHorusJobs><<<(unsigned)grid_jd, GS_SUM_THREADS, 0, h->stream>>>(GsSumHorusJobs{h->d_sims}, first, count, h->jd,
                                                                                          h->d_jd, h->d_jd_hist, h->d_sum_scratch, (long long)pitch);
    HCU(cudaGetLastError());
    h->launches += 1;
  }
  if (Csd > 0) {          // after gs_sum_jobs_kernel, on the same scratch with a fourth row
    int per_sd = 1;
    HCU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sd, gs_sd_jobs_kernel<GsSumHorusJobs>, GS_SUM_THREADS, 0));
    const int grid_sd = std::min(grid, std::max(1, per_sd) * sms);
    gs_sd_jobs_kernel<GsSumHorusJobs><<<(unsigned)grid_sd, GS_SUM_THREADS, 0, h->stream>>>(GsSumHorusJobs{h->d_sims}, first, count, h->sd,
                                                                                          h->d_sd, h->d_sd_hist, h->d_sum_scratch, (long long)pitch);
    HCU(cudaGetLastError());
    h->launches += 1;
  }
  if (Cif > 0) {          // after gs_sum_jobs_kernel, on the same scratch with GS_IF_ROWS rows
    int per_if = 1;
    HCU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_if, gs_if_jobs_kernel<GsSumHorusJobs>, GS_SUM_THREADS, 0));
    const int grid_if = std::min(grid, std::max(1, per_if) * sms);
    gs_if_jobs_kernel<GsSumHorusJobs><<<(unsigned)grid_if, GS_SUM_THREADS, 0, h->stream>>>(GsSumHorusJobs{h->d_sims}, first, count, h->ifc,
                                                                                          h->d_if, h->d_sum_scratch, (long long)pitch);
    HCU(cudaGetLastError());
    h->launches += 1;
  }
  if (Barr > 0) {         // after the other job kernels, on the same scratch with GS_ARR_ROWS rows
    gs_arr_jobs_kernel<GsSumHorusJobs><<<(unsigned)grid_arr, GS_SUM_THREADS, 0, h->stream>>>(GsSumHorusJobs{h->d_sims}, first, count, h->arr,
                                                                                            h->d_arr, h->d_sum_scratch, (long long)pitch);
    HCU(cudaGetLastError());
    h->launches += 1;
  }
  if (B > 0) {
    gs_htl_rows_kernel<<<(unsigned)count, GS_SUM_THREADS, 0, h->stream>>>(h->d_sims, first, h->d_tl, (long long)h->tl_width, B);
    HCU(cudaGetLastError());
    h->launches += 1;
  }
  if (h->occ_on) {
    gs_occ_hsum<<<(unsigned)count, GS_SUM_THREADS, 0, h->stream>>>(h->d_sims, first, h->occ, h->d_occ, h->d_occ_busy,
                                                                                         (long long)h->occ_pitch, h->d_occ_q);
    HCU(cudaGetLastError());
    h->launches += 1;
  }
  HCU(cudaEventRecord(h->ev1, h->stream));
#else   // host build for tests/emu: the same folds, one replica after the other
  for (int r = first; r < first + count; ++r) {
    const HSim &S = h->d_sims[r];
    gs_summary &A = h->d_sum[r];
    GsSumPart p;
    gs_sum_zero(p);
    for (long long i = 0; i < S.ticks; ++i) gs_sum_row(p, S.rows[i], S.util[i]);
    A.n = S.n; A.done = S.done; A.status = S.status;
    gs_sum_add_rows(A, p);
    if (S.ticks > 0) A.makespan = S.rows[S.ticks - 1].now;
    std::vector<GsSumJob> jobs((size_t)S.nfin);
    for (int i = 0; i < S.nfin; ++i) {
      const int j = S.fin[i];
      jobs[(size_t)i] = gs_sum_job(S.jobs[j].arrive, S.recs[j].start, S.recs[j].end, S.recs[j].jct, S.recs[j].preempt, S.jobs[j].gpus);
    }
    gs_sum_jobs_serial(jobs.data(), S.nfin, A);
    if (C > 0) gs_jd_jobs_serial(jobs.data(), S.nfin, h->jd, h->d_jd + (size_t)r * C, h->d_jd_hist + (size_t)r * C * 3 * (h->jd.nedges + 1));
    if (Csd > 0) gs_sd_serial(jobs.data(), S.nfin, h->sd, h->d_sd + (size_t)r * Csd, h->d_sd_hist + (size_t)r * Csd * gs_sd_row_len(h->sd));
    if (Cif > 0) {
      std::vector<GsIfDur> durs((size_t)S.nfin);
      for (int i = 0; i < S.nfin; ++i) {
        const int j = S.fin[i];
        durs[(size_t)i] = GsIfDur{S.jobs[j].gpus, S.recs[j].original, S.recs[j].actual};
      }
      gs_if_serial(jobs.data(), durs.data(), S.nfin, h->ifc, h->d_if + (size_t)r * Cif);
    }
    if (Barr > 0) {
      const int n = std::max(S.n, 0);
      std::vector<int> fin_arrive((size_t)S.nfin), trace_arrive((size_t)n);
      for (int i = 0; i < S.nfin; ++i) fin_arrive[(size_t)i] = S.jobs[S.fin[i]].arrive;
      for (int j = 0; j < n; ++j) trace_arrive[(size_t)j] = S.jobs[j].arrive;
      gs_arr_serial(jobs.data(), fin_arrive.data(), S.nfin, trace_arrive.data(), n, h->arr, h->d_arr + (size_t)r * Barr);
    }
    if (B > 0) gs_tl_fold_rows_serial(h->d_tl + (size_t)r * B, B, (long long)h->tl_width, S.rows, S.util, 0, 0, S.ticks);
    if (h->occ_on) {
      gs_occ &o = h->d_occ[r];
      o.total_gpus = S.M * S.G;
      unsigned long long *hall = h->d_occ_busy + (size_t)r * 2 * (size_t)h->occ_pitch;
      const GsOccHist H{hall, hall + h->occ_pitch, h->d_occ_q + (size_t)r * (size_t)(h->occ.nedges + 1)};
      GsOccCarry c{0, 0, 0, 0, 0};
      gs_occ_serial(o, c, H, h->occ, S.rows, 0, 0, S.ticks, S.done, 1);
    }
  }
  (void)kmax;
#endif
  HCU(cudaMemcpyAsync(out, h->d_sum + first, sizeof(gs_summary) * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaStreamSynchronize(h->stream));
#ifdef __CUDACC__
  float ms = 0.f;
  HCU(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  if (kernel_ms) *kernel_ms = ms;
#endif
  for (int i = first; i < first + count; ++i) {
    if (B > 0) h->sims[(size_t)i].tl_done = true;
    if (C > 0) h->sims[(size_t)i].jd_done = true;
    if (Csd > 0) h->sims[(size_t)i].sd_done = true;
    if (Barr > 0) h->sims[(size_t)i].arr_done = true;
    if (h->occ_on) h->sims[(size_t)i].occ_done = true;
    if (Cif > 0) h->sims[(size_t)i].if_done = true;
  }
  return GS_OK;
}

extern "C" int gs_horus_set_timeline(gs_horus_handle h, int64_t bin_width, int32_t nbins) {
  if (!h) return GS_ERR_ARG;
  if (nbins < 0 || nbins > GS_TIMELINE_MAX_BINS || (nbins > 0 && (bin_width < 1 || bin_width > (1ll << 40))))
    return hfail(h, GS_ERR_ARG, "gs_horus_set_timeline: nbins must be in 0..1024 and, when it is not 0, bin_width in 1..2^40");
  const size_t need = sizeof(gs_tbin) * h->sims.size() * (size_t)nbins;
  if (need > h->tl_bytes) {
    HCU(cudaSetDevice(h->device));
    gs_tbin *d = nullptr;
    HCU(cudaMalloc(&d, need));
    if (h->d_tl) { HCU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_tl); }
    h->d_tl = d; h->tl_bytes = need;
  }
  h->tl_width = nbins > 0 ? bin_width : 0;
  h->tl_nbins = nbins;
  for (auto &s : h->sims) s.tl_done = false;
  return GS_OK;
}

extern "C" int gs_horus_fetch_timeline(gs_horus_handle h, int32_t first, int32_t count, gs_tbin *out) {
  if (!h) return GS_ERR_ARG;
  const int nsims = (int)h->sims.size();
  if (first < 0 || count < 0 || first > nsims - count || (count > 0 && !out)) return hfail(h, GS_ERR_ARG, "gs_horus_fetch_timeline: bad arguments");
  if (h->tl_nbins == 0) return hfail(h, GS_ERR_STATE, "gs_horus_fetch_timeline: the timeline is off (gs_horus_set_timeline)");
  for (int i = first; i < first + count; ++i)
    if (!h->sims[(size_t)i].prepared || !h->sims[(size_t)i].tl_done)
      return hfail(h, GS_ERR_STATE, "gs_horus_fetch_timeline: a replica has not been summarised with the timeline on since it was prepared");
  if (count == 0) return GS_OK;
  HCU(cudaSetDevice(h->device));
  const size_t B = (size_t)h->tl_nbins;
  HCU(cudaMemcpyAsync(out, h->d_tl + (size_t)first * B, sizeof(gs_tbin) * B * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaStreamSynchronize(h->stream));
  return GS_OK;
}

extern "C" int gs_horus_set_jobdist(gs_horus_handle h, int32_t nclasses, const int32_t *bounds, int32_t nedges, const int32_t *edges) {
  if (!h) return GS_ERR_ARG;
  GsJdCfg cfg;
  const char *why = nullptr;
  if (!gs_jd_make_cfg(nclasses, bounds, nedges, edges, cfg, &why)) return hfail(h, GS_ERR_ARG, std::string("gs_horus_set_jobdist: ") + why);
  const size_t need = sizeof(gs_jclass) * h->sims.size() * (size_t)cfg.nclasses;
  const size_t need_hist = sizeof(unsigned) * h->sims.size() * (size_t)cfg.nclasses * 3 * (size_t)(cfg.nedges + 1);
  if (need > h->jd_bytes || need_hist > h->jd_hist_bytes) {
    HCU(cudaSetDevice(h->device));
    gs_jclass *d = nullptr;
    unsigned *dh = nullptr;
    HCU(cudaMalloc(&d, std::max(need, h->jd_bytes)));
    if (cudaMalloc(&dh, std::max(need_hist, h->jd_hist_bytes)) != cudaSuccess) {
      cudaFree(d);
      return hfail(h, GS_ERR_CUDA, "gs_horus_set_jobdist: cudaMalloc failed");
    }
    HCU(cudaStreamSynchronize(h->stream));
    if (h->d_jd) cudaFree(h->d_jd);
    if (h->d_jd_hist) cudaFree(h->d_jd_hist);
    h->d_jd = d; h->jd_bytes = std::max(need, h->jd_bytes);
    h->d_jd_hist = dh; h->jd_hist_bytes = std::max(need_hist, h->jd_hist_bytes);
  }
  h->jd = cfg;
  for (auto &s : h->sims) s.jd_done = false;
  return GS_OK;
}

extern "C" int gs_horus_fetch_jobdist(gs_horus_handle h, int32_t first, int32_t count, gs_jclass *classes_out, uint32_t *hist_out) {
  if (!h) return GS_ERR_ARG;
  const int nsims = (int)h->sims.size();
  if (first < 0 || count < 0 || first > nsims - count) return hfail(h, GS_ERR_ARG, "gs_horus_fetch_jobdist: bad arguments");
  if (h->jd.nclasses == 0) return hfail(h, GS_ERR_STATE, "gs_horus_fetch_jobdist: the job statistics are off (gs_horus_set_jobdist)");
  for (int i = first; i < first + count; ++i)
    if (!h->sims[(size_t)i].prepared || !h->sims[(size_t)i].jd_done)
      return hfail(h, GS_ERR_STATE, "gs_horus_fetch_jobdist: a replica has not been summarised with this setting since it was prepared");
  if (count == 0) return GS_OK;
  HCU(cudaSetDevice(h->device));
  const size_t C = (size_t)h->jd.nclasses, per = C * 3 * (size_t)(h->jd.nedges + 1);
  if (classes_out)
    HCU(cudaMemcpyAsync(classes_out, h->d_jd + (size_t)first * C, sizeof(gs_jclass) * C * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  if (hist_out)
    HCU(cudaMemcpyAsync(hist_out, h->d_jd_hist + (size_t)first * per, sizeof(unsigned) * per * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaStreamSynchronize(h->stream));
  return GS_OK;
}

extern "C" int gs_horus_set_slowdown(gs_horus_handle h, const gs_slowdown_cfg *in) {
  if (!h) return GS_ERR_ARG;
  GsSdCfg cfg;
  const char *why = nullptr;
  if (!gs_sd_make_cfg(in, cfg, &why)) return hfail(h, GS_ERR_ARG, std::string("gs_horus_set_slowdown: ") + why);
  const size_t need = sizeof(gs_sdclass) * h->sims.size() * (size_t)cfg.nclasses;
  const size_t need_hist = sizeof(unsigned) * h->sims.size() * (size_t)cfg.nclasses * (size_t)gs_sd_row_len(cfg);
  if (need > h->sd_bytes || need_hist > h->sd_hist_bytes) {
    HCU(cudaSetDevice(h->device));
    gs_sdclass *d = nullptr;
    unsigned *dh = nullptr;
    HCU(cudaMalloc(&d, std::max(need, h->sd_bytes)));
    if (cudaMalloc(&dh, std::max(need_hist, h->sd_hist_bytes)) != cudaSuccess) {
      cudaFree(d);
      return hfail(h, GS_ERR_CUDA, "gs_horus_set_slowdown: cudaMalloc failed");
    }
    HCU(cudaStreamSynchronize(h->stream));
    if (h->d_sd) cudaFree(h->d_sd);
    if (h->d_sd_hist) cudaFree(h->d_sd_hist);
    h->d_sd = d; h->sd_bytes = std::max(need, h->sd_bytes);
    h->d_sd_hist = dh; h->sd_hist_bytes = std::max(need_hist, h->sd_hist_bytes);
  }
  h->sd = cfg;
  for (auto &s : h->sims) s.sd_done = false;
  return GS_OK;
}

extern "C" int gs_horus_fetch_slowdown(gs_horus_handle h, int32_t first, int32_t count, gs_sdclass *out, uint32_t *hist_out) {
  if (!h) return GS_ERR_ARG;
  const int nsims = (int)h->sims.size();
  if (first < 0 || count < 0 || first > nsims - count) return hfail(h, GS_ERR_ARG, "gs_horus_fetch_slowdown: bad arguments");
  if (h->sd.nclasses == 0) return hfail(h, GS_ERR_STATE, "gs_horus_fetch_slowdown: the slowdown statistics are off (gs_horus_set_slowdown)");
  for (int i = first; i < first + count; ++i)
    if (!h->sims[(size_t)i].prepared || !h->sims[(size_t)i].sd_done)
      return hfail(h, GS_ERR_STATE, "gs_horus_fetch_slowdown: a replica has not been summarised with this setting since it was prepared");
  if (count == 0) return GS_OK;
  HCU(cudaSetDevice(h->device));
  const size_t C = (size_t)h->sd.nclasses, per = C * (size_t)gs_sd_row_len(h->sd);
  if (out)
    HCU(cudaMemcpyAsync(out, h->d_sd + (size_t)first * C, sizeof(gs_sdclass) * C * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  if (hist_out)
    HCU(cudaMemcpyAsync(hist_out, h->d_sd_hist + (size_t)first * per, sizeof(unsigned) * per * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaStreamSynchronize(h->stream));
  return GS_OK;
}

extern "C" int gs_horus_set_arrivals(gs_horus_handle h, int64_t bin_width, int32_t nbins, int64_t tau) {
  if (!h) return GS_ERR_ARG;
  GsArrCfg cfg;
  const char *why = nullptr;
  if (!gs_arr_make_cfg(bin_width, nbins, tau, cfg, &why)) return hfail(h, GS_ERR_ARG, std::string("gs_horus_set_arrivals: ") + why);
  HCU(cudaSetDevice(h->device));
  const size_t need = sizeof(gs_abin) * h->sims.size() * (size_t)cfg.nbins;
  if (need > h->arr_bytes) {
    bool fits = true;
#ifdef __CUDACC__
    size_t free_b = 0, total_b = 0;
    HCU(cudaMemGetInfo(&free_b, &total_b));
    fits = need <= free_b;
#endif
    gs_abin *d = nullptr;
    if (!fits || cudaMalloc(&d, need) != cudaSuccess) {
      (void)cudaGetLastError();
      return hfail(h, GS_ERR_CAPACITY, "gs_horus_set_arrivals: the bin records (" + std::to_string(need) + " bytes) do not fit the device's free memory");
    }
    if (h->d_arr) { HCU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_arr); }
    h->d_arr = d; h->arr_bytes = need;
  } else if (cfg.nbins == 0 && h->d_arr) {           // off: the records are not kept
    HCU(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_arr);
    h->d_arr = nullptr; h->arr_bytes = 0;
  }
  h->arr = cfg;
  for (auto &s : h->sims) s.arr_done = false;
  return GS_OK;
}

extern "C" int gs_horus_fetch_arrivals(gs_horus_handle h, int32_t first, int32_t count, gs_abin *out) {
  if (!h) return GS_ERR_ARG;
  const int nsims = (int)h->sims.size();
  if (first < 0 || count < 0 || first > nsims - count || (count > 0 && !out)) return hfail(h, GS_ERR_ARG, "gs_horus_fetch_arrivals: bad arguments");
  if (h->arr.nbins == 0) return hfail(h, GS_ERR_STATE, "gs_horus_fetch_arrivals: the arrival statistics are off (gs_horus_set_arrivals)");
  for (int i = first; i < first + count; ++i)
    if (!h->sims[(size_t)i].prepared || !h->sims[(size_t)i].arr_done)
      return hfail(h, GS_ERR_STATE, "gs_horus_fetch_arrivals: a replica has not been summarised with this setting since it was prepared");
  if (count == 0) return GS_OK;
  HCU(cudaSetDevice(h->device));
  const size_t B = (size_t)h->arr.nbins;
  HCU(cudaMemcpyAsync(out, h->d_arr + (size_t)first * B, sizeof(gs_abin) * B * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaStreamSynchronize(h->stream));
  return GS_OK;
}

extern "C" int gs_horus_set_occupancy(gs_horus_handle h, int32_t on, int32_t nedges, const int32_t *edges) {
  if (!h) return GS_ERR_ARG;
  GsOccCfg cfg{};
  const char *why = nullptr;
  if (on && !gs_occ_make_cfg(nedges, edges, cfg, &why)) return hfail(h, GS_ERR_ARG, std::string("gs_horus_set_occupancy: ") + why);
  if (on) {
    HCU(cudaSetDevice(h->device));
    if (!h->d_occ) HCU(cudaMalloc(&h->d_occ, sizeof(gs_occ) * h->sims.size()));
    const size_t need_q = 8 * h->sims.size() * (size_t)(cfg.nedges + 1);
    if (need_q > h->occ_q_bytes) {
      unsigned long long *d = nullptr;
      HCU(cudaMalloc(&d, need_q));
      if (h->d_occ_q) { HCU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_occ_q); }
      h->d_occ_q = d; h->occ_q_bytes = need_q;
    }
  }
  h->occ_on = on != 0;
  h->occ = cfg;
  for (auto &s : h->sims) s.occ_done = false;
  return GS_OK;
}

extern "C" int gs_horus_fetch_occupancy(gs_horus_handle h, int32_t first, int32_t count, gs_occ *out, uint64_t *busy_hist, int32_t busy_pitch,
                                        uint64_t *queue_hist) {
  if (!h) return GS_ERR_ARG;
  const int nsims = (int)h->sims.size();
  if (first < 0 || count < 0 || first > nsims - count) return hfail(h, GS_ERR_ARG, "gs_horus_fetch_occupancy: bad arguments");
  if (!h->occ_on) return hfail(h, GS_ERR_STATE, "gs_horus_fetch_occupancy: the occupancy statistics are off (gs_horus_set_occupancy)");
  int64_t width = 1;
  for (int i = first; i < first + count; ++i) {
    const HorusSimHost &s = h->sims[(size_t)i];
    if (!s.prepared || !s.occ_done)
      return hfail(h, GS_ERR_STATE, "gs_horus_fetch_occupancy: a replica has not been summarised with the occupancy on since it was prepared");
    width = std::max(width, (int64_t)s.dev.M * s.dev.G + 1);
  }
  if (busy_hist && count > 0 && busy_pitch < width)
    return hfail(h, GS_ERR_CAPACITY, "gs_horus_fetch_occupancy: busy_pitch is smaller than total_gpus + 1 of a fetched replica");
  if (count == 0) return GS_OK;
  HCU(cudaSetDevice(h->device));
  if (out) HCU(cudaMemcpyAsync(out, h->d_occ + first, sizeof(gs_occ) * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  if (busy_hist) {
    const unsigned long long *src = h->d_occ_busy + (size_t)first * 2 * (size_t)h->occ_pitch;
    const size_t w = 8 * (size_t)std::min(width, h->occ_pitch);
#ifdef __CUDACC__
    HCU(cudaMemcpy2DAsync(busy_hist, 8 * (size_t)busy_pitch, src, 8 * (size_t)h->occ_pitch, w, 2 * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
#else
    for (size_t k = 0; k < 2 * (size_t)count; ++k)
      HCU(cudaMemcpyAsync(busy_hist + k * (size_t)busy_pitch, src + k * (size_t)h->occ_pitch, w, cudaMemcpyDeviceToHost, h->stream));
#endif
  }
  const size_t E1 = (size_t)h->occ.nedges + 1;
  if (queue_hist) HCU(cudaMemcpyAsync(queue_hist, h->d_occ_q + (size_t)first * E1, 8 * E1 * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaStreamSynchronize(h->stream));
  return GS_OK;
}

extern "C" int gs_horus_set_interference(gs_horus_handle h, int32_t nclasses, const int32_t *bounds) {
  if (!h) return GS_ERR_ARG;
  GsJdCfg cfg;
  const char *why = "nclasses must be in 0..8";
  if (nclasses < 0 || nclasses > GS_JOBDIST_MAX_CLASSES || !gs_jd_make_cfg(nclasses, bounds, 0, nullptr, cfg, &why))
    return hfail(h, GS_ERR_ARG, std::string("gs_horus_set_interference: ") + why);
  const size_t need = sizeof(gs_ifclass) * h->sims.size() * (size_t)cfg.nclasses;
  if (need > h->if_bytes) {
    HCU(cudaSetDevice(h->device));
    gs_ifclass *d = nullptr;
    HCU(cudaMalloc(&d, need));
    if (h->d_if) { HCU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_if); }
    h->d_if = d; h->if_bytes = need;
  }
  h->ifc = cfg;
  for (auto &s : h->sims) s.if_done = false;
  return GS_OK;
}

extern "C" int gs_horus_fetch_interference(gs_horus_handle h, int32_t first, int32_t count, gs_ifclass *out) {
  if (!h) return GS_ERR_ARG;
  const int nsims = (int)h->sims.size();
  if (first < 0 || count < 0 || first > nsims - count || (count > 0 && !out)) return hfail(h, GS_ERR_ARG, "gs_horus_fetch_interference: bad arguments");
  if (h->ifc.nclasses == 0) return hfail(h, GS_ERR_STATE, "gs_horus_fetch_interference: the interference statistics are off (gs_horus_set_interference)");
  for (int i = first; i < first + count; ++i)
    if (!h->sims[(size_t)i].prepared || !h->sims[(size_t)i].if_done)
      return hfail(h, GS_ERR_STATE, "gs_horus_fetch_interference: a replica has not been summarised with this setting since it was prepared");
  if (count == 0) return GS_OK;
  HCU(cudaSetDevice(h->device));
  const size_t C = (size_t)h->ifc.nclasses;
  HCU(cudaMemcpyAsync(out, h->d_if + (size_t)first * C, sizeof(gs_ifclass) * C * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaStreamSynchronize(h->stream));
  return GS_OK;
}

extern "C" int gs_horus_compare(gs_horus_handle h, int32_t npairs, const int32_t *a, const int32_t *b, int32_t nclasses, const int32_t *bounds,
                                int32_t nedges, const int32_t *edges, gs_jpair *out, uint32_t *hist_out, double *kernel_ms) {
  if (!h) return GS_ERR_ARG;
  if (npairs < 0 || (npairs > 0 && (!a || !b || !out))) return hfail(h, GS_ERR_ARG, "gs_horus_compare: bad arguments");
  GsJdCfg cfg;
  const char *why = nullptr;
  if (!gs_jd_make_cfg(nclasses, bounds, nedges, edges, cfg, &why)) return hfail(h, GS_ERR_ARG, std::string("gs_horus_compare: ") + why);
  if (nclasses == 0) return hfail(h, GS_ERR_ARG, "gs_horus_compare: nclasses must be in 1..8");
  const int nsims = (int)h->sims.size();
  for (int i = 0; i < npairs; ++i)
    if (a[i] < 0 || a[i] >= nsims || b[i] < 0 || b[i] >= nsims) return hfail(h, GS_ERR_ARG, "gs_horus_compare: a replica index is out of range");
  long long nmax = 1;
  for (int i = 0; i < npairs; ++i) {
    const HorusSimHost &sa = h->sims[(size_t)a[i]], &sb = h->sims[(size_t)b[i]];
    if (!sa.prepared || !sb.prepared) return hfail(h, GS_ERR_STATE, "gs_horus_compare: a replica has not run yet");
    if (sa.dev.n != sb.dev.n) return hfail(h, GS_ERR_ARG, "gs_horus_compare: pair " + std::to_string(i) + " holds traces of different lengths");
    nmax = std::max(nmax, (long long)sa.dev.n);
  }
  if (kernel_ms) *kernel_ms = 0.0;
  if (npairs == 0) return GS_OK;
  HCU(cudaSetDevice(h->device));
  const size_t P = (size_t)npairs, C = (size_t)cfg.nclasses, nb = (size_t)cfg.nedges + 1;
  std::vector<int> flags(P, 0);
  std::vector<gs_jpair> recs(P * C);
  std::vector<uint32_t> hist(P * C * 3 * nb);
#ifdef __CUDACC__
  int per_sm = 1, sms = 132;
  HCU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gs_cmp_pairs_kernel<GsSumHorusJobs>, GS_SUM_THREADS, 0));
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
  const int grid = std::min(npairs, std::max(1, per_sm) * sms);
  const size_t pitch = (size_t)(nmax + 63) / 64 * 64;
  // scratch: pair indices, trace-differ flags, records, CDF counts, per-block work
  const size_t o_a = 0, o_b = up(4 * P), o_flag = up(o_b + 4 * P), o_rec = up(o_flag + 4 * P);
  const size_t o_hist = up(o_rec + sizeof(gs_jpair) * P * C), o_work = up(o_hist + 4 * P * C * 3 * nb);
  const size_t need = o_work + 4 * sizeof(int) * pitch * (size_t)grid;
  if (h->sum_scratch_bytes < need) {
    if (h->d_sum_scratch) { HCU(cudaStreamSynchronize(h->stream)); cudaFree(h->d_sum_scratch); }
    h->d_sum_scratch = nullptr; h->sum_scratch_bytes = 0;
    HCU(cudaMalloc(&h->d_sum_scratch, need));
    h->sum_scratch_bytes = need;
  }
  unsigned char *d = (unsigned char *)h->d_sum_scratch;
  HCU(cudaMemcpyAsync(d + o_a, a, 4 * P, cudaMemcpyHostToDevice, h->stream));
  HCU(cudaMemcpyAsync(d + o_b, b, 4 * P, cudaMemcpyHostToDevice, h->stream));
  HCU(cudaEventRecord(h->ev0, h->stream));
  gs_cmp_pairs_kernel<GsSumHorusJobs><<<(unsigned)grid, GS_SUM_THREADS, 0, h->stream>>>(
      GsSumHorusJobs{h->d_sims}, npairs, (const int *)(d + o_a), (const int *)(d + o_b), cfg, (gs_jpair *)(d + o_rec),
      (unsigned *)(d + o_hist), (int *)(d + o_flag), (int *)(d + o_work), (long long)pitch);
  HCU(cudaGetLastError());
  HCU(cudaEventRecord(h->ev1, h->stream));
  HCU(cudaMemcpyAsync(flags.data(), d + o_flag, 4 * P, cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaMemcpyAsync(recs.data(), d + o_rec, sizeof(gs_jpair) * P * C, cudaMemcpyDeviceToHost, h->stream));
  if (hist_out) HCU(cudaMemcpyAsync(hist.data(), d + o_hist, 4 * hist.size(), cudaMemcpyDeviceToHost, h->stream));
  HCU(cudaStreamSynchronize(h->stream));
#else   // host build for tests/emu: the same steps, one pair after the other
  for (size_t p = 0; p < P; ++p) {
    const HSim &A = h->d_sims[a[p]], &B = h->d_sims[b[p]];
    for (int j = 0; j < A.n && !flags[p]; ++j) flags[p] = !gs_hjob_same(A.jobs[j], B.jobs[j]);
    if (flags[p]) continue;
    std::vector<GsSumJob> ja((size_t)A.n), jb((size_t)B.n);
    for (int j = 0; j < A.n; ++j) {
      ja[(size_t)j] = gs_sum_job(A.jobs[j].arrive, A.recs[j].start, A.recs[j].end, A.recs[j].jct, A.recs[j].preempt, A.jobs[j].gpus);
      jb[(size_t)j] = gs_sum_job(B.jobs[j].arrive, B.recs[j].start, B.recs[j].end, B.recs[j].jct, B.recs[j].preempt, B.jobs[j].gpus);
    }
    gs_cmp_pair_serial(ja.data(), jb.data(), A.n, A.fin, A.nfin, B.fin, B.nfin, cfg, recs.data() + p * C, hist.data() + p * C * 3 * nb);
  }
  (void)nmax;
#endif
  h->launches += 1;
  for (size_t i = 0; i < P; ++i)
    if (flags[i]) return hfail(h, GS_ERR_ARG, "gs_horus_compare: pair " + std::to_string(i) + " (replicas " + std::to_string(a[i]) + ", " +
                                              std::to_string(b[i]) + ") holds different traces");
  memcpy(out, recs.data(), sizeof(gs_jpair) * recs.size());
  if (hist_out) memcpy(hist_out, hist.data(), 4 * hist.size());
#ifdef __CUDACC__
  float ms = 0.f;
  HCU(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  if (kernel_ms) *kernel_ms = ms;
#endif
  return GS_OK;
}

/*
 * gsched.h -- C ABI of libgsched.so, the sm_90a discrete-event engine that
 * replaces the per-tick hot path of matthewygf/GPUSchedule.
 *
 * The reference has no FFI: its "operator API" is the Python loop object and
 * three dict registries.  Every entry point below names the reference
 * interface it replaces (paths relative to the reference root):
 *
 *   gs_run            Scheduler.start()            core/scheduling/schedule.py:178-215
 *                     (gen_jobs jobs_manager.py:228-241, _schedule schedule.py:40-60,
 *                      schedule_fifo algorithm.py:189-202, ms_yarn_placement :28-32,
 *                      step jobs_manager.py:143-148, release_finished_jobs
 *                      schedule.py:141-162, _construct_info schedule.py:95-133)
 *   gs_place_batch    placement_algorithms['yarn'](infrastructure, job, scheme)
 *                     core/scheduling/algorithm.py:28-32,301-393,396-417
 *   gs_net_cost       calculate_network_costs(infrastructure, job)
 *                     core/network/network_service.py:3-39
 *   gs_load_trace     JobsManager.gen_jobs' per-row Job(...) construction
 *                     core/jobs/jobs_manager.py:233-239 (rows arrive pre-sorted by
 *                     the host ingest, job_generator.py:181-193)
 *   gs_config_sim     Infrastructure(FLAGS)        infra/infrastructure.py:26-58
 *
 * Conventions: every function returns 0 on success and a negative gs_status
 * on failure (message via gs_last_error); nothing throws or exits across the
 * boundary.  The caller owns every host buffer and passes sizes explicitly;
 * the library owns all device memory and its CUDA stream.  One handle is
 * bound to one CUDA device and must be driven by one host thread at a time;
 * handles are independent.  There is NO CPU fallback: without a usable CUDA
 * device gs_create fails with GS_ERR_CUDA.
 */
#ifndef GSCHED_H_
#define GSCHED_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GS_ABI_VERSION 4
#define GS_MAX_QUEUES 8
#define GS_MAX_GPUS_PER_NODE 64
#define GS_MAX_RANKS 8          /* GPUs of one box that may share one simulation (gs_comm_init) */

typedef enum {
  GS_OK = 0,
  GS_ERR_ARG = -1,      /* bad argument / unsupported configuration          */
  GS_ERR_CUDA = -2,     /* CUDA runtime or driver error                      */
  GS_ERR_STATE = -3,    /* call order (e.g. gs_run before gs_load_trace)     */
  GS_ERR_CAPACITY = -4, /* an output buffer is too small                     */
  GS_ERR_COMM = -5      /* sharded multi-GPU path: a peer did not answer in time / IPC error */
} gs_status;

/* scheduling policies (run_sim.py:37-49 names) and placement schemes (:25-36) */
enum { GS_SCHED_FIFO = 0, GS_SCHED_SJF = 1, GS_SCHED_DLAS = 2,
       GS_SCHED_DLAS_GPU = 3, GS_SCHED_GITTINS = 4 };
enum { GS_SCHEME_YARN = 0, GS_SCHEME_COUNT = 1 };

/* Cluster description == the flags Infrastructure reads (infrastructure.py:26-43). */
typedef struct gs_cluster {
  int32_t num_switch;
  int32_t num_node_p_switch;
  int32_t num_gpu_p_node;        /* G <= GS_MAX_GPUS_PER_NODE                  */
  int32_t num_cpu_p_node;
  int32_t mem_p_node;
  int32_t gpu_mem_cap_mib;       /* gpu_memory_capacity * 1024 (infrastructure.py:36) */
  int32_t enable_network_costs;  /* schedule.py:49                             */
  int32_t cpu_per_task;          /* 12 in the reference (job.py:105)           */
  int32_t mem_per_task;          /* 60 in the reference (job.py:106)           */
  int32_t reserved0;
  double bandwidth;              /* MB/s   (run_sim.py:59)                     */
  double internode_latency;      /* s      (run_sim.py:65)                     */
} gs_cluster;

typedef struct gs_policy {
  int32_t schedule;              /* GS_SCHED_*                                 */
  int32_t scheme;                /* GS_SCHEME_*                                */
  int32_t num_queue;             /* dlas MLFQ depth (<= GS_MAX_QUEUES)          */
  int32_t gittins_n;             /* entries in the gittins tables              */
  double queue_limit[GS_MAX_QUEUES]; /* dlas thresholds (README.md:57-62)      */
  double gittins_delta;          /* service quantum for the index (3250)       */
  const double *gittins_data;    /* host ptr, sorted sample + sentinel         */
  const double *gittins_index;   /* host ptr, index per sample + 0.0           */
} gs_policy;

/* One row of integer aggregates per simulated tick: everything LogInfo
 * (log_manager.py:5-30) carries except the RNG column, as integers so that the
 * host can apply the reference's own float expressions.  64 bytes.            */
typedef struct gs_tick_row {
  int32_t now;            /* 'delta' column (already incremented, schedule.py:193) */
  int32_t idle_nodes;     /* nodes that never hosted a placement (node.py:93-97)  */
  int32_t busy_nodes;
  int32_t busy_gpus;
  int32_t idle_gpus;
  int32_t running;
  int32_t queued;
  int32_t finished;
  int64_t mem_busy_bytes; /* sum over busy devices of min(cap, task memory_max)   */
  int64_t pend_sum;       /* sum of pending ticks over the queue                  */
  int32_t pend_max;       /* 0 when the queue is empty                            */
  int32_t pend_med_lo;    /* the two middle pending values (equal when odd)       */
  int32_t pend_med_hi;
  int32_t reserved;
} gs_tick_row;

/* Compact form of the same information, as the fifo engine writes it.  On a tick where nothing arrives,
 * starts or finishes no LogInfo counter changes except `delta` and the pending times, which move linearly
 * with the tick, so the engine writes one gs_evrow per tick on which a counter DID change (and for the first
 * tick of every gs_run window), beside it one gs_qrow while the queue is non-empty, and one gs_nodeev whenever
 * the number of nodes that ever hosted a job grows (and for the first record of a window); the row of any tick
 * v in [now_k, now_k+1) follows from record k:
 *   delta = v, pending sum = queued*v - arrive_sum, max/median pending = v - oldest / middle arrivals
 * (jobs_manager.py:72-87), busy nodes = the last gs_nodeev at or before v, queue statistics = the gs_qrow with
 * the same `now` (both streams are ordered by `now`).  gs_fetch_rows does this expansion on the device;
 * gs_fetch_compact / gs_fetch_results hand out the records themselves (about a quarter of the bytes of the rows
 * on the BASELINE trace).  24 + 24 + 8 bytes.                                                              */
typedef struct gs_evrow {
  int32_t now;              /* 'delta' of the first row this record describes                          */
  int32_t queued;
  int32_t finished;
  uint16_t busy_gpus;       /* (the engine requires M*G <= 65535)                                      */
  uint16_t running;
  int64_t mem_busy_bytes;
} gs_evrow;

typedef struct gs_qrow {
  int32_t now;              /* the gs_evrow this record belongs to                                     */
  int32_t oldest_arrive;    /* arrival tick of the job that has waited longest                         */
  int32_t med_lo_arrive;    /* arrival ticks of the two middle jobs of the queue (equal when odd)      */
  int32_t med_hi_arrive;
  int64_t arrive_sum;       /* sum of the arrival ticks of the queued jobs                             */
} gs_qrow;

typedef struct gs_nodeev {
  int32_t now;              /* from this row on ...                                                    */
  int32_t busy_nodes;       /* ... this many nodes have hosted a placement (node.py:93-97, never decreases) */
} gs_nodeev;

/* Compact per-job result of the fifo engine: the start tick (-1: the job never started).  fifo never preempts,
 * so the rest of job.csv follows from the trace: run length = max(1, ceil(job.duration)) ticks (quirk Q11; with
 * network costs job.duration is the value gs_fetch_compact returns in duration_out), end = start + run length,
 * jct = run length, preempt = 1 (quirk Q12).  4 bytes per job.                                          */
typedef int32_t gs_job_start;

/* Compact (job, node) record of the fifo engine for clusters with at most 32 GPUs per node (every BASELINE
 * cluster); wider nodes keep the 16-byte gs_span with GS_SPAN_FIRST in ntasks.  8 bytes.                  */
typedef struct gs_cspan {
  uint32_t where;           /* node (bits 0-19) | (ntasks - 1) << 20 | first record of a job << 31           */
  uint32_t devmask;         /* devices of that node held by the job                                          */
} gs_cspan;
#define GS_CSPAN_NODE(w) ((w) & 0xfffffu)
#define GS_CSPAN_NTASKS(w) ((((w) >> 20) & 0x3fu) + 1u)
#define GS_CSPAN_FIRST(w) ((w) >> 31)

/* What the last gs_run window of one replica holds (sizes for gs_fetch_compact).                        */
typedef struct gs_window_info {
  int64_t row_first;        /* tick index of the window's first row                                    */
  int64_t ticks;            /* rows produced so far (the window is [row_first, ticks))                 */
  int64_t ev_rows, q_rows;  /* records of the window                                                   */
  int64_t node_events;      /* gs_nodeev records of the window (at least 1 once a tick has run)         */
  int64_t spans_used;       /* (job, node) records so far, start order                                 */
  int64_t admitted;         /* trace rows consumed so far: gs_job_start is defined for jobs below this  */
  int64_t finished;
  int64_t n;
} gs_window_info;

/* Per-job result, 24 bytes: what LogManager.jcts prints (log_manager.py:143-153). */
typedef struct gs_job_rec {
  int32_t start;          /* start_time; -1 if the job never started             */
  int32_t end;            /* end_time;   -1 if it never finished                 */
  int32_t jct;            /* time_processed() at completion                      */
  int32_t preempt;        /* migration_count (1 for a never-preempted job)       */
  double duration;        /* job.duration after network cost (job.py:196-197)    */
} gs_job_rec;

/* Where a job's tasks ran: one record per (job, node).  16 bytes.               */
#define GS_SPAN_FIRST 0x80000000u  /* gs_fetch_compact only: set in ntasks on the first record of every job */
typedef struct gs_span {
  int32_t node;           /* 0-based node index (reference node_id = node + 1)   */
  int32_t ntasks;
  uint64_t devmask;       /* devices of that node held by the job                */
} gs_span;

typedef struct gs_run_stats {
  int64_t ticks;          /* rows produced so far                                */
  int64_t events;         /* arrivals + starts + completions (+preempt/resume)   */
  int64_t finished;       /* jobs completed                                      */
  int64_t started;
  int64_t placement_evals;/* (job,node) candidate evaluations                    */
  int32_t done;           /* 1 when the loop's exit condition was reached        */
  int32_t status;         /* 0 or a gs_status raised inside the kernel           */
  double kernel_ms;       /* CUDA-event time of the engine kernel(s)             */
  double h2d_ms, d2h_ms;  /* CUDA-event time of the copies of the last calls     */
} gs_run_stats;

/* cluster state record for the stateless placement entry point. 16 bytes.       */
typedef struct gs_node {
  uint64_t busy_mask;     /* bit d set <=> device d has a task                   */
  int32_t cpu_used;
  int32_t mem_used;
} gs_node;

typedef struct gs_jobreq {
  int32_t gpus;           /* Job.gpus                                            */
  int32_t gpu_per_task;   /* Job.gpu_per_worker                                  */
  int64_t mem_bytes;      /* memory_max                                          */
} gs_jobreq;

/* One trace row as the device stores it (32 bytes, one DRAM sector).               */
typedef struct gs_jobin {
  int32_t arrive_tick;    /* first tick with normalized_time <= tick             */
  int32_t gpus;
  int32_t gpu_per_task;
  int32_t ps_count;       /* 0 when the trace has no network columns             */
  int64_t mem_bytes;
  double duration;        /* minutes * scale_factor                              */
} gs_jobin;

/* One replica's run reduced to the numbers the reference's notebooks compute from its cluster.csv and job.csv
 * (makespan, mean utilisation, mean pending time, job-level means / medians / spreads).  256 bytes.
 * "Rows" are the lines of cluster.csv: one per tick for the fifo and horus engines, one per event for the
 * event-driven policies.  "Jobs" are the lines of job.csv, i.e. the finished jobs.  A job's `arrive` is its
 * arrival tick gs_jobin.arrive_tick = ceil(normalized_time); job.csv's submit_time is int(normalized_time) and
 * can be one less.  fifo's start / end / jct / preempt are what job.csv prints: end = start + max(1, ceil(duration))
 * (duration after the network cost when network costs are on), jct = that run length, preempt = 1.
 * A summary of a replica that is not done yet covers the rows and finished jobs so far.                        */
typedef struct gs_summary {
  int64_t n;                /* jobs in the trace                                                               */
  int64_t rows;             /* rows folded so far                                                              */
  int32_t done, status;     /* the replica's done flag and in-kernel status (gs_run_stats)                     */
  int64_t makespan;         /* `delta` of the last row folded (df.delta.max())                                 */
  int64_t busy_gpus_sum, running_sum, queued_sum;   /* sums over rows of num_busy_gpus / num_running_jobs / num_queuing_jobs */
  int32_t busy_gpus_max, running_max, queued_max;   /* their maxima over rows                                            */
  int32_t pend_max_max;     /* max over rows of max_pending_time                                               */
  uint64_t pend_sum_lo, pend_sum_hi;   /* sum over rows of the row's pending-time sum (gs_tick_row.pend_sum), 128-bit */
  uint64_t mem_busy_lo, mem_busy_hi;   /* sum over rows of mem_busy_bytes, 128-bit; mean avg_gpu_memory_allocated =
                                          this / 2^20 / (M * G * gpu_mem_cap_mib) / rows                              */
  int64_t pending_rows;     /* rows with avg_pending_time != 0                                                 */
  double avg_pending_sum;   /* sum of avg_pending_time over those rows, each term pend_sum / (queued + 1e-9)
                               (log_manager.pending_columns); the mean the notebooks take is this / pending_rows    */
  double util_sum;          /* horus engine: sum over rows of the sampled avg_gpu_utilization, NaN counted as 0
                               (the notebooks' fillna(0)); NaN from gs_summarize (that column is sampled on the host) */
  int64_t finished;         /* lines of job.csv                                                                */
  int64_t wait_sum, turnaround_sum, jct_sum, preempt_sum, gpu_ticks_sum;  /* sums over finished jobs of start - arrive,
                               end - arrive, jct, preempt, num_gpu * jct                                          */
  int32_t wait_q[5], turnaround_q[5], jct_q[5];   /* nearest-rank order statistics at 50 / 90 / 95 / 99 / 100 %: of k
                               values sorted ascending, rank q (per mille) is element ceil(q * k / 1000) - 1; 0 when k = 0 */
  int32_t reserved[5];
} gs_summary;

typedef struct gs_engine *gs_handle;

int gs_abi_version(void);
const char *gs_build_tag(void);          /* "cuda:sm_90a": the package refuses any other build of these entry points */
const char *gs_last_error(gs_handle h);  /* h may be NULL: last creation error    */

/* A handle simulates `nsims` independent replicas on CUDA device `device`.      */
int gs_create(int device, int nsims, gs_handle *out);
void gs_destroy(gs_handle h);

int gs_config_sim(gs_handle h, int sim, const gs_cluster *cluster, const gs_policy *policy);

/* Trace of one replica, rows in admission order (arrive_tick non-decreasing).
 * model_mb / iterations / ps_count may be NULL (no network term).               */
int gs_load_trace(gs_handle h, int sim, int64_t n,
                  const int32_t *arrive_tick, const int32_t *gpus,
                  const int32_t *gpu_per_task, const double *duration,
                  const int64_t *mem_bytes, const double *model_mb,
                  const double *iterations, const int32_t *ps_count);

/* The same trace already packed as gs_jobin records (no column gather on the host). */
int gs_load_trace_packed(gs_handle h, int sim, int64_t n, const gs_jobin *jobs,
                         const double *model_mb, const double *iterations);

/* Advance every replica by at most max_ticks ticks (<=0: until done).  Record
 * storage on the device is sized by rows_cap per replica at the first call (fifo: that many gs_evrow
 * and gs_qrow records; event-driven policies: that many rows); a launch also ends when it is full,
 * so any value >= 1 is safe -- drain with the fetch calls and call again.                            */
int gs_run(gs_handle h, int64_t max_ticks, int64_t rows_cap);
/* Separate capacity for the gs_qrow stream of replicas prepared afterwards (0 = same as rows_cap).   */
int gs_set_queue_rows_cap(gs_handle h, int64_t qrows_cap);

int gs_stats(gs_handle h, int sim, gs_run_stats *out);

/* Restart every replica at tick 0 on the traces already resident in device
 * memory (sweeps, benchmarking); also clears the accumulated timers.           */
int gs_reset(gs_handle h);

/* Kernel mapping of the event-driven policies: 0 = warp-cooperative kernels (default), 2 = one thread
 * per replica (first version, kept as a cross-check).  The fifo engine has one mapping (a warp per replica). */
int gs_set_engine(gs_handle h, int mode);

/* Span-pool sizing for traces loaded afterwards: 0 (default) = worst case, never overflows;
 * x > 0 = min(worst case, x * n + 4096) records per replica (overflow -> GS_ERR_CAPACITY). */
int gs_set_span_budget(gs_handle h, double spans_per_job);

/* Number of CUDA kernels this handle has launched so far.                       */
int64_t gs_launch_count(gs_handle h);

/* Page-locked host memory for DMA-speed gs_load_trace / gs_fetch_* transfers.  */
int gs_host_alloc(size_t bytes, void **out);
int gs_host_free(void *p);

/* Copy results of one replica to caller-owned host buffers (any may be NULL).  */
int gs_fetch_rows(gs_handle h, int sim, int64_t first, int64_t count, gs_tick_row *rows_out);
int gs_fetch_jobs(gs_handle h, int sim, gs_job_rec *jobs_out /* n */,
                  int32_t *finish_order_out /* n, first `finished` valid */);
int gs_fetch_spans(gs_handle h, int sim, int64_t *span_off_out /* n+1 */,
                   gs_span *spans_out, int64_t spans_cap, int64_t *spans_used);

/* All results of one replica in one call (any output may be NULL); rows [first, first+count)
 * must lie in the last gs_run window.                                           */
int gs_fetch_all(gs_handle h, int sim, int64_t first, int64_t count, gs_tick_row *rows_out,
                 gs_job_rec *jobs_out, int32_t *finish_order_out, int64_t *span_off_out,
                 gs_span *spans_out, int64_t spans_cap, int64_t *spans_used);

/* ---- compact, asynchronous result path (fifo engine) ------------------------------------------------
 * gs_window_info: sizes of what the last gs_run left.  gs_fetch_compact enqueues the copies of every
 * non-NULL output on the handle's stream and returns; gs_sync waits for them.  Buffers from
 * gs_host_alloc make the copies true DMA.  Sizes: ev_out ev_rows, q_out q_rows, nodeev_out node_events, jobs_out n,
 * duration_out n (only with network costs, else left untouched), finish_order_out finished,
 * spans_out spans_used records of gs_result_layout's span_bytes each (8: gs_cspan, 16: gs_span; start order,
 * the first-of-job flag marks job boundaries; jobs in start order = jobs_out sorted by start, start ticks are
 * unique -- one start per tick, schedule.py:188-190).                                                   */
int gs_window(gs_handle h, int sim, gs_window_info *out);
int gs_fetch_compact(gs_handle h, int sim, gs_evrow *ev_out, gs_qrow *q_out, gs_nodeev *nodeev_out, gs_job_start *jobs_out,
                     double *duration_out, int32_t *finish_order_out, void *spans_out /* gs_cspan[] or gs_span[], see gs_result_layout */);
int gs_sync(gs_handle h);
/* The same, for many replicas with ONE copy each way (what bench.py's end-to-end path uses).  The replicas of a
 * handle keep their results in blocks of one layout, side by side on the device:
 *   gs_load_traces_packed  all traces of the handle from one host block, trace i at jobs + i * pitch_bytes
 *                          (n_each[i] records): one strided upload
 *   gs_result_layout       byte offsets of the arrays inside a replica's result block, their capacities, and
 *                          block_bytes, the length of the block
 *   gs_fetch_results       the blocks of replicas [first, first + count) into out + i * out_pitch: one strided
 *                          copy, asynchronous (gs_sync waits); gs_window tells how many entries of each array are valid */
typedef struct gs_result_layout_t {
  int64_t block_bytes;
  int64_t off_ev, off_q, off_nodeev, off_jobs, off_duration /* -1 without network costs */, off_finish_order, off_spans;
  int64_t cap_ev, cap_q, cap_nodeev, cap_spans, n;
  int64_t span_bytes;       /* 8: gs_cspan records (at most 32 GPUs per node), 16: gs_span records               */
} gs_result_layout_t;
int gs_load_traces_packed(gs_handle h, const gs_jobin *jobs, size_t pitch_bytes, const int64_t *n_each);
int gs_result_layout(gs_handle h, int sim, gs_result_layout_t *out);
int gs_fetch_results(gs_handle h, int first, int count, void *out, size_t out_pitch);
/* 1: gs_load_trace_packed from a page-locked buffer enqueues the upload without staging and returns
 * before it completes -- the caller keeps the buffer unchanged until the next gs_run / gs_sync on
 * this handle returns.  0 (default): every call copies and completes before returning.              */
int gs_set_async(gs_handle h, int on);

/* ---- one simulation on several GPUs of one box (BASELINE config C4; SURVEY 8(e)) ----------------------
 * The north-star sketches "the trace sharded across the 8 GPUs with one allreduce per tick".  What is worth
 * sharding in this path is the per-event work that is O(runnable jobs): for the gittins policy that is the index
 * evaluation (run_sim.py:1040-1078 -> get_gittins_index :949-954, a table search per runnable job per event).
 * Every rank holds the (small) cluster / queue state and the trace; rank r evaluates the chunks c of the
 * runnable list with c mod nranks == r and STORES the results straight into every peer's receive buffer over
 * NVLink (peer memory opened with CUDA IPC), then publishes an event counter in the peers' flag words and waits
 * for theirs -- one exchange per event, inside the persistent kernel, no host round trip and no NCCL call on the
 * data path (torch.distributed only carries the 64-byte IPC handles at start-up).  Order, admission and the
 * statistics are then computed redundantly and identically on every rank: results are bit-identical to one GPU.
 *
 *   gs_comm_prepare  allocates this handle's exchange buffer (for traces of up to max_jobs jobs) and returns its IPC handle
 *   gs_comm_init     receives the handles of ALL ranks (own at [rank]), opens the peers', arms the sharded mode for
 *                    gittins replicas prepared afterwards; the handle must hold exactly one replica
 *   gs_comm_stats    exchanges done and their mean cost in microseconds (publish -> all peers seen, incl. skew)
 * A peer that does not answer within ~5 s ends the run with GS_ERR_COMM on every waiting rank.            */
typedef struct gs_comm_handle { unsigned char bytes[64]; } gs_comm_handle;
int gs_comm_prepare(gs_handle h, int64_t max_jobs, gs_comm_handle *out);
int gs_comm_init(gs_handle h, int rank, int nranks, const gs_comm_handle *all_ranks);
int gs_comm_stats(gs_handle h, int64_t *exchanges, double *mean_us);
/* Events with at most k runnable jobs are evaluated by every rank itself -- the replicated state guarantees identical
 * results without sending anything -- and only longer lists are split and exchanged.  k = 0: always exchange.
 * DEFAULT: no list is long enough (k = INT32_MAX).  An exchange costs 2-4 us, and since the index of a job is one table
 * load (the direct table of gs_config_sim) no list we measured -- up to ~7000 runnable jobs -- is evaluated slower by
 * one GPU than an exchange takes (DESIGN section 7 has the numbers); the call is how a caller opts in. */
int gs_comm_set_min_runnable(gs_handle h, int k);

/* ---- on-device run summaries -------------------------------------------------------------------------
 * gs_summarize folds, for replicas [first, first + count), the rows of the last gs_run window not folded yet into
 * per-replica accumulators the handle keeps on the device (gs_result_layout and the result blocks are untouched),
 * recomputes the job part from the finish order and the per-job results, and copies `count` gs_summary records
 * to `out` (one copy, synchronous).  Call it after every gs_run to summarise a run of several windows; calling it
 * twice folds nothing twice.  A replica prepared afresh (first gs_run, gs_reset, a new trace) starts from zero.
 * kernel_ms (may be NULL) receives the device time of its kernels; gs_run_stats.kernel_ms does not include it.
 * Errors: GS_ERR_ARG for a bad range, GS_ERR_STATE for a replica that has not run or whose earlier window was
 * not summarised (nothing is changed then).  util_sum is NaN here.                                        */
int gs_summarize(gs_handle h, int first, int count, gs_summary *out, double *kernel_ms);

/* ---- binned time series of a run's rows (timeline) -----------------------------------------------------
 * A timeline of bin width W >= 1 (ticks of `delta`) and B bins (1 <= B <= GS_TIMELINE_MAX_BINS) puts a row into bin
 * min(floor(delta / W), B - 1) (a negative `delta` into bin 0): the last bin is open-ended, so the bins of a replica
 * together hold exactly the rows its gs_summary holds.  A bin holds the row part of gs_summary restricted to its
 * rows, the smallest and largest `delta` folded into it and the `finished` counter of its last row in row order.
 * The fields of a bin without rows are 0 (util_sum: NaN from gs_summarize).  128 bytes.                    */
#define GS_TIMELINE_MAX_BINS 1024
typedef struct gs_tbin {
  int64_t rows;
  int64_t busy_gpus_sum, running_sum, queued_sum;
  int32_t busy_gpus_max, running_max, queued_max, pend_max_max;
  uint64_t pend_sum_lo, pend_sum_hi;   /* 128-bit, as in gs_summary */
  uint64_t mem_busy_lo, mem_busy_hi;
  int64_t pending_rows;
  double avg_pending_sum;
  double util_sum;
  int64_t delta_min, delta_max;        /* the smallest / largest `delta` of the bin's rows                          */
  int64_t finished_last;               /* `finished` of the bin's last row in row order                              */
} gs_tbin;
/* gs_set_timeline: while nbins > 0, every gs_summarize also folds the rows it folds (the same rows past the same
 * watermark) into per-replica bins on the device; nbins = 0 (the default) turns the timeline off, and bin_width is
 * then ignored.  Every replica starts again from zero bins.  GS_ERR_ARG for a bad width or count, GS_ERR_STATE when a
 * replica has folded rows since it was last prepared (set the timeline before the first gs_summarize of a run, or
 * after gs_reset); nothing changes on an error.
 * gs_fetch_timeline copies count * nbins records (replica-major) as of the last gs_summarize (synchronous).
 * GS_ERR_ARG for a bad range, GS_ERR_STATE when the timeline is off or a replica has not been summarised since it was
 * prepared with the timeline on.  A replica prepared afresh (first gs_run, gs_reset, a new trace, gs_boot_traces)
 * starts from zero bins.                                                                                   */
int gs_set_timeline(gs_handle h, int64_t bin_width, int32_t nbins);
int gs_fetch_timeline(gs_handle h, int first, int count, gs_tbin *out);

/* ---- job statistics by job size (jobdist) ---------------------------------------------------------------
 * The jobs are the finished jobs of gs_summary's job part, with the same wait = start - arrive, turnaround =
 * end - arrive, jct, preempt and gpus (num_gpu).  C classes (1 <= C <= GS_JOBDIST_MAX_CLASSES) are given by C - 1
 * strictly increasing bounds b_1 < ... < b_{C-1}, each >= 1: a job's class is the number of bounds <= gpus (bounds
 * {5, 17, 65}: classes 1-4, 5-16, 17-64, 65+; C = 1: all jobs).  Per class, one gs_jclass: the class's part of
 * gs_summary's job fields, exact 128-bit sums of squares, and the order statistics under gs_summary's rank rule
 * (0 for an empty class).  With C = 1 the record equals the summary's job part field for field.
 * CDF histogram: E strictly increasing edges e_0 < ... < e_{E-1} (0 <= E <= GS_JOBDIST_MAX_EDGES), one list for
 * wait, turnaround and jct.  Per (class, quantity) E + 1 uint32 counts: value v goes to bin #{i : e_i < v}, so the
 * count through bin b is #(v <= e_b), the right-continuous CDF at e_b.  Layout per replica [class][wait, turnaround,
 * jct][bin].  Every field is an integer; a repeated call gives the same bytes.                                 */
#define GS_JOBDIST_MAX_CLASSES 8
#define GS_JOBDIST_MAX_EDGES 255
typedef struct gs_jclass {
  int64_t jobs;                                            /* finished jobs in the class                         */
  int64_t wait_sum, turnaround_sum, jct_sum, preempt_sum, gpu_ticks_sum;   /* as in gs_summary                  */
  uint64_t wait_sq_lo, wait_sq_hi;                         /* sums of squares, 128-bit                           */
  uint64_t turnaround_sq_lo, turnaround_sq_hi;
  uint64_t jct_sq_lo, jct_sq_hi;
  int32_t wait_q[5], turnaround_q[5], jct_q[5];            /* 50 / 90 / 95 / 99 / 100 %, gs_summary's rank rule   */
  int32_t reserved;
} gs_jclass;
/* gs_set_jobdist: while nclasses > 0, every gs_summarize also computes the class records and CDF histograms of the
 * replicas it summarises (the job part is recomputed in full on every call, so this may be called at any time);
 * nclasses = 0 (the default) turns it off, and the arrays are then ignored.  Every replica is marked as not
 * summarised with this setting.  GS_ERR_ARG for nclasses outside 0..8, nedges outside 0..255, bounds that are not
 * strictly increasing or below 1, edges that are not strictly increasing, or a NULL array with a positive count;
 * nothing changes on an error.
 * gs_fetch_jobdist copies count * C records and count * C * 3 * (E + 1) counts (replica-major; either output may be
 * NULL) as of the last gs_summarize (synchronous).  GS_ERR_ARG for a bad range, GS_ERR_STATE when the feature is off
 * or a replica has not been summarised since it was prepared (first gs_run, gs_reset, a new trace, gs_boot_traces)
 * or since the last gs_set_jobdist.                                                                          */
int gs_set_jobdist(gs_handle h, int32_t nclasses, const int32_t *bounds, int32_t nedges, const int32_t *edges);
int gs_fetch_jobdist(gs_handle h, int first, int count, gs_jclass *classes_out, uint32_t *hist_out);

/* ---- job statistics by a chosen key, with bounded slowdown (slowdown) ------------------------------------------
 * The jobs are jobdist's: the finished jobs of gs_summary's job part with arrive, start, end, jct and gpus, wait =
 * start - arrive and turnaround = end - arrive.  jct is the job's run length in ticks: max(1, ceil(duration)) in the
 * fifo and policy engines, the largest time_processed of the job's tasks in the horus engine.
 * Key of a job, chosen per setting: GS_JKEY_GPUS: gpus (jobdist's key); GS_JKEY_LENGTH: jct; GS_JKEY_GPU_TIME:
 * gpus * jct (int64).  C classes (1 <= C <= GS_JOBDIST_MAX_CLASSES) from C - 1 strictly increasing int64 bounds, each
 * >= 1: a job's class is the number of bounds <= its key.
 * Bounded slowdown of a job, in fixed point (units of 1/1024), for an integer tau >= 1:
 *     sd = min(2^31 - 1, max(1024, floor(1024 * turnaround / max(jct, tau))))
 * computed in 64-bit integer arithmetic (no floating point).  tau = 1 gives plain slowdown, turnaround / jct.  The
 * value saturates at 2^31 - 1, a slowdown of about 2.1 million; sd_clamped counts the class's jobs whose sd is that
 * value.  Per class one gs_sdclass: `jc` is the class's gs_jclass with jobdist's meaning field for field (with
 * key = gpus and jobdist's bounds it is byte-equal to gs_fetch_jobdist's), then the same statistics of sd, and the
 * exact sum of the class's keys.
 * CDF histograms: wait, turnaround and jct at E strictly increasing int32 edges (0 <= E <= GS_JOBDIST_MAX_EDGES,
 * jobdist's edges and rule: value v in bin #{i : e_i < v}); sd at its own Esd strictly increasing int32 edges
 * (0 <= Esd <= GS_SLOWDOWN_MAX_EDGES, in units of 1/1024, the same rule).  Layout per replica
 * [class][wait, turnaround, jct, sd][bin]: per class 3 * (E + 1) + (Esd + 1) uint32 counts, the rows of wait,
 * turnaround and jct E + 1 long each, then the sd row Esd + 1 long.  Every field is an integer; a repeated call gives
 * the same bytes.                                                                                              */
#define GS_JKEY_GPUS 0
#define GS_JKEY_LENGTH 1
#define GS_JKEY_GPU_TIME 2
#define GS_SLOWDOWN_MAX_EDGES 255
typedef struct gs_sdclass {
  gs_jclass jc;                      /* the class's jobdist record                                                   */
  int64_t sd_sum;                    /* sum of sd (units of 1/1024)                                                  */
  uint64_t sd_sq_lo, sd_sq_hi;       /* exact 128-bit sum of sd^2                                                    */
  int32_t sd_q[5];                   /* 50 / 90 / 95 / 99 / 100 %, gs_summary's rank rule; 0 for an empty class      */
  int32_t sd_min;                    /* smallest sd; 0 for an empty class                                            */
  int64_t sd_clamped;                /* jobs with sd = 2^31 - 1                                                      */
  uint64_t key_sum_lo, key_sum_hi;   /* exact 128-bit sum of the keys (gpus * jct < 2^55 per job)                    */
} gs_sdclass;                        /* 232 bytes */
typedef struct gs_slowdown_cfg {
  int32_t key;                       /* GS_JKEY_*                                                                   */
  int32_t nclasses;                  /* 0: off; 1..GS_JOBDIST_MAX_CLASSES                                           */
  int64_t bounds[GS_JOBDIST_MAX_CLASSES - 1];   /* the first nclasses - 1 are used                                 */
  int64_t tau;                       /* >= 1, ticks                                                                 */
  int32_t nedges, nsd_edges;         /* E, Esd                                                                      */
  const int32_t *edges;              /* E edges of wait, turnaround and jct (may be NULL when E = 0)                */
  const int32_t *sd_edges;           /* Esd edges of sd (may be NULL when Esd = 0)                                  */
} gs_slowdown_cfg;
/* gs_set_slowdown: while cfg->nclasses > 0, every gs_summarize also computes the class records and CDF histograms of
 * the replicas it summarises (the job part is recomputed in full on every call, so this may be called at any time);
 * cfg == NULL or nclasses = 0 (the default) turns it off.  Every replica is marked as not summarised with this
 * setting.  Jobdist and slowdown may both be on; each keeps its own arrays and state.  GS_ERR_ARG for a key other than
 * GS_JKEY_*, nclasses outside 0..8, bounds that are not strictly increasing or below 1, tau < 1, E or Esd outside
 * 0..255, edges that are not strictly increasing, or a NULL array with a positive count; nothing changes on an error.
 * gs_fetch_slowdown copies count * C records and count * C * (3 * (E + 1) + Esd + 1) counts (replica-major; either
 * output may be NULL) as of the last gs_summarize (synchronous).  GS_ERR_ARG for a bad range, GS_ERR_STATE when the
 * feature is off or a replica has not been summarised since it was prepared (first gs_run, gs_reset, a new trace,
 * gs_boot_traces) or since the last gs_set_slowdown.                                                         */
int gs_set_slowdown(gs_handle h, const gs_slowdown_cfg *cfg);
int gs_fetch_slowdown(gs_handle h, int first, int count, gs_sdclass *out, uint32_t *hist_out);

/* ---- job statistics by arrival time (arrivals) -------------------------------------------------------------------
 * The jobs are slowdown's, binned by arrival tick instead of a class key.  A setting is a bin width W >= 1 (ticks),
 * B bins (1 <= B <= GS_ARRIVALS_MAX_BINS) and a slowdown bound tau >= 1.  A job that arrives at tick a falls in bin
 * min(floor(a / W), B - 1), a negative a in bin 0: the last bin is open-ended.  The ticks are the timeline's `delta`
 * ticks, so a timeline and the arrival bins may share W.  Per (replica, bin) one gs_abin: `s` is slowdown's gs_sdclass
 * field for field, restricted to the bin's finished jobs, with the arrival tick as the key (key_sum is the exact sum
 * of their arrival ticks), and `arrived` counts the bin's jobs of the replica's trace, finished or not: arrived -
 * s.jc.jobs of them had not finished (a run of several windows, a job wider than the cluster).  There are no CDF
 * histograms.  Every field is an integer; a repeated call gives the same bytes.                                  */
#define GS_ARRIVALS_MAX_BINS 1024
typedef struct gs_abin {
  gs_sdclass s;                      /* slowdown's record of the bin's finished jobs, key = arrival tick              */
  int64_t arrived;                   /* jobs of the replica's trace in this bin, finished or not                      */
} gs_abin;                           /* 240 bytes */
/* gs_set_arrivals: while nbins > 0, every gs_summarize also computes the bin records of the replicas it summarises
 * (the job part is recomputed in full on every call, so this may be called at any time); nbins = 0 (the default)
 * turns it off, and bin_width and tau are then ignored.  Every replica is marked as not summarised with this setting.
 * Jobdist, slowdown and arrivals may all be on; each keeps its own arrays and state.  The records take nsims * B * 240
 * bytes of device memory, allocated only while the feature is on.  GS_ERR_ARG for nbins outside 0..1024, or, when
 * nbins > 0, bin_width < 1 or tau < 1; GS_ERR_CAPACITY when the records do not fit the device's free memory; nothing
 * changes on an error.
 * gs_fetch_arrivals copies count * B records (replica-major) as of the last gs_summarize (synchronous).  GS_ERR_ARG
 * for a bad range, GS_ERR_STATE when the feature is off or a replica has not been summarised since it was prepared
 * (first gs_run, gs_reset, a new trace, gs_boot_traces) or since the last gs_set_arrivals.                     */
int gs_set_arrivals(gs_handle h, int64_t bin_width, int32_t nbins, int64_t tau);
int gs_fetch_arrivals(gs_handle h, int first, int count, gs_abin *out);

/* ---- time-weighted occupancy (occupancy) -----------------------------------------------------------------------
 * The rows of gs_summary's row part, each weighed by the ticks it stands for.  busy = busy_gpus as the row holds it
 * (horus: devices with at least one task), G = M * G of the replica's cluster (at most 65535).
 * Weights: a row of the fifo or horus engine is one tick (a fifo record k stands for the now_(k+1) - now_k rows up to
 * the next record, the last one for the rows up to `ticks`).  Row i of an event-driven policy weighs
 * max(0, delta_(i+1) - delta_i) ticks: a row whose successor's delta is smaller or equal (dlas can emit such rows)
 * weighs 0.  The last row of a finished run (done) weighs 1; the last row of an unfinished window is kept in a
 * per-replica carry (its delta, busy, running and queued) and weighed when a later gs_summarize sees its successor
 * or the run done.  Rows folded once are not folded again (gs_summarize's watermark).
 * Per replica one gs_occ, all integers (w the weight of a row; T = ticks < 2^31; sums cannot overflow int64):
 *   rows (rows weighed), ticks = T = sum of w, busy_sum / running_sum / queued_sum = sum of w * value,
 *   running_max / queued_max over rows with w > 0, wait_ticks = sum of w over rows with queued > 0,
 *   idle_wait_sum = sum of w * (G - busy) over rows with queued > 0, total_gpus = G.
 * Histograms of ticks (uint64): H_all[b], b = 0..G, ticks with busy == b; H_wait[b], ticks with busy == b and
 * queued > 0; Q[k], k = 0..E, ticks whose queue length v lies in bin #{i : e_i < v} of E strictly increasing edges
 * e_0 < ... < e_{E-1}, each >= 0 (0 <= E <= GS_OCC_MAX_EDGES; jobdist's rule).  Sum of H_all = sum of Q = T,
 * sum of H_wait = wait_ticks.  Integer adds only: a repeated call gives the same bytes.                       */
#define GS_OCC_MAX_EDGES 255
typedef struct gs_occ {
  int64_t rows;                      /* rows weighed so far                                                         */
  int64_t ticks;                     /* T, the sum of the weights                                                   */
  int64_t busy_sum, running_sum, queued_sum;   /* sums of w * busy_gpus / running / queued                         */
  int64_t wait_ticks;                /* sum of w over rows with queued > 0                                          */
  int64_t idle_wait_sum;             /* sum of w * (total_gpus - busy_gpus) over rows with queued > 0               */
  int32_t running_max, queued_max;   /* over rows with w > 0                                                        */
  int32_t total_gpus;                /* M * G                                                                       */
  int32_t reserved;
} gs_occ;                            /* 72 bytes */
/* gs_set_occupancy: while on != 0, every gs_summarize also folds the rows it folds into the replicas' gs_occ records
 * and histograms, with queue edges edges[0 .. nedges); on = 0 (the default) turns it off, and the edges are then
 * ignored.  Every replica starts again from zero.  GS_ERR_ARG for nedges outside 0..255, edges that are negative or
 * not strictly increasing, or a NULL array with a positive count; GS_ERR_STATE when a replica has folded rows since it
 * was last prepared (gs_set_timeline's rule); nothing changes on an error.  While it is on, gs_summarize returns
 * GS_ERR_ARG, before anything changes, for a replica with more than 65535 GPUs.
 * gs_fetch_occupancy copies, as of the last gs_summarize (synchronous; any output may be NULL), count records to out,
 * replica first + i's H_all to busy_hist + i * 2 * busy_pitch and its H_wait busy_pitch entries further (entries past
 * its total_gpus are 0 up to the widest fetched replica's, and not written beyond), and count * (E + 1) queue counts to queue_hist.  GS_ERR_ARG for a bad range,
 * GS_ERR_CAPACITY for busy_hist with busy_pitch < total_gpus + 1 of a fetched replica, GS_ERR_STATE when the feature is
 * off or a replica has not been summarised with it on since it was prepared (first gs_run, gs_reset, a new trace,
 * gs_boot_traces*).                                                                                            */
int gs_set_occupancy(gs_handle h, int32_t on, int32_t nedges, const int32_t *edges);
int gs_fetch_occupancy(gs_handle h, int first, int count, gs_occ *out, uint64_t *busy_hist, int32_t busy_pitch, uint64_t *queue_hist);

/* ---- paired per-job comparison of two replicas on the same trace ------------------------------------------
 * A pair (a, b) is two replicas of one handle that hold the same trace: the same job count n and, for every j < n,
 * a byte-equal gs_jobin record (gs_horus_compare: equal fields as taken by gs_horus_load_trace).  They may differ in
 * anything else (policy, cluster, dlas limits, network cost); (a, a) is a pair too.  Per job j the quantities x are
 * gs_summary's wait, turnaround and jct; job j is finished in a run if it is in that replica's finish order so far,
 * so a pair may be compared after any gs_run window (gs_summarize is not needed first).  Classes are jobdist's
 * (C - 1 strictly increasing bounds >= 1, 1 <= C <= 8); both runs share the trace, so they agree on every class.
 * Every x is a non-negative int32 (start >= arrive, end >= arrive), so d = x_b - x_a has |d| <= 2^31 - 1 and both d
 * and -d fit in int32.  Per (pair, class) one gs_jpair; its order statistics sort the k = `jobs` differences
 * ascending, d_(0) <= ... <= d_(k-1), and with rank_t the nearest rank of gs_summary (50 / 90 / 95 / 99 / 100 %) give
 * q_hi[m][t] = d_(rank_t) and q_lo[m][t] = d_(k-1-rank_t): q_hi[m][4] is the maximum, q_lo[m][4] the minimum, and
 * swapping a pair gives q_hi(b, a) = -q_lo(a, b).  0 when k = 0.
 * Optional CDF of d: E strictly increasing signed int32 edges (0 <= E <= 255), per (pair, class, quantity) E + 1
 * uint32 counts, value d in bin #(edges < d) (jobdist's rule).  Every field is an integer; a repeated call gives the
 * same bytes.                                                                                                 */
typedef struct gs_jpair {
  int64_t jobs;                      /* jobs of the class finished in both runs                                    */
  int64_t only_a, only_b;            /* finished in run a only / in run b only                                     */
  int64_t lt[3], eq[3], gt[3];       /* per quantity (wait, turnaround, jct), d = x_b - x_a: #(d < 0), #(d == 0),
                                        #(d > 0) over the `jobs` jobs                                               */
  int64_t d_sum[3];
  uint64_t d_sq_lo[3], d_sq_hi[3];   /* exact 128-bit sum of d^2                                                   */
  int32_t q_hi[3][5];                /* d ascending, gs_summary's nearest ranks 50 / 90 / 95 / 99 / 100 %          */
  int32_t q_lo[3][5];                /* d descending, the same ranks: 50 % and 10 / 5 / 1 / 0 % from below         */
} gs_jpair;
/* gs_compare: npairs pairs (a[i], b[i]) into out (pair-major, npairs * C records) and, when hist_out is not NULL,
 * npairs * C * 3 * (E + 1) counts ([pair][class][wait, turnaround, jct][bin]).  Synchronous; one kernel launch when
 * npairs > 0, none when npairs == 0.  Uses the handle's summary scratch in stream order and touches no summary
 * accumulator, watermark, timeline or jobdist state.  kernel_ms (may be NULL) receives the kernel's device time.
 * Errors leave out, hist_out and the handle unchanged: GS_ERR_ARG for npairs < 0, a NULL a, b or out with npairs > 0,
 * an index outside [0, nsims), classes or edges gs_set_jobdist refuses or C = 0, pairs with different job counts,
 * and pairs whose traces differ (found on the device; gs_last_error names the first such pair); GS_ERR_STATE for
 * a replica that has not run.                                                                                 */
int gs_compare(gs_handle h, int32_t npairs, const int32_t *a, const int32_t *b, int32_t nclasses, const int32_t *bounds,
               int32_t nedges, const int32_t *edges, gs_jpair *out, uint32_t *hist_out, double *kernel_ms);

/* ---- bootstrap replicas generated on the device ---------------------------------------------------------
 * gs_boot_population gives the handle one base trace P of k >= 1 records (admission order, the gs_load_trace rules;
 * validated once, copied to the device); D holds its k - 1 inter-arrival gaps D[i] = P[i+1].arrive_tick - P[i].arrive_tick.
 * gs_boot_traces then draws a trace for EVERY replica of the handle from params[sim] (nsims entries): job j takes the
 * words w0..w3 of the Philox4x64-10 block with key (seed, stream) and counter (j + 1, 0, 0, 0) -- numpy's
 * Philox(key=[seed, stream], counter=[j, 0, 0, 0]).random_raw(4) -- and becomes
 *   {floor(S_j * gap_num / gap_den), P[r].gpus, P[r].gpu_per_task, 0, P[r].mem_bytes, P[r].duration}
 * with r = floor(w0 * k / 2^64), S_j = g_0 + ... + g_j, g_0 = 0, g_j = D[floor(w1 * (k - 1) / 2^64)] (0 when k = 1).
 * gap_num / gap_den = 1 / 1 keeps the base trace's arrival rate in expectation, 1 / 2 doubles the offered load; the same
 * (seed, stream) draws the same rows and gaps at every load (common random numbers).  w3 is used only by gs_boot_traces_mixed (below),
 * and w2 only by gs_boot_traces_blocked, which draws replica sim as a stationary block bootstrap with mean block length
 * L = block_len[sim] (block_len NULL: L = 1 for all, exactly gs_boot_traces): job 0 starts a block, job j > 0 starts one
 * iff floor(w2 * L / 2^64) == 0; with b the last block start <= j and s_b = floor(w0_b * k / 2^64), job j copies row
 * r = (s_b + j - b) mod k, and its gap is D[r - 1] when j continues a block with r > 0, the iid gap above otherwise.
 * L = 1 is the iid bootstrap, byte for byte; the same (seed, stream) is coupled across loads and values of L.
 * Afterwards every replica is in the state gs_load_traces_packed leaves (loaded, not prepared, span budget applied);
 * kernel_ms (may be NULL) receives the generator's device time.  gs_fetch_trace copies the n records of any resident
 * trace of one replica (synchronous).
 * Errors (nothing changes): GS_ERR_ARG for a NULL argument, k < 1 or a record that breaks the load rules, n outside
 * gs_load_traces_packed's range, gap_num < 0 or gap_den < 1, block_len[sim] == 0, a replica whose cluster has network
 * costs, or a worst-case last arrival floor((n - 1) * max(D) * gap_num / gap_den) of 2^31 - 1 or more; GS_ERR_STATE
 * without a population, for a replica not configured with gs_config_sim, or (gs_fetch_trace) for a replica that holds
 * no trace.                                                                                                  */
typedef struct gs_boot_params {
  uint64_t seed, stream;    /* Philox key                                                                     */
  int64_t n;                /* jobs                                                                           */
  int32_t gap_num, gap_den; /* gap scale: gap_num >= 0, gap_den >= 1                                          */
} gs_boot_params;           /* 32 bytes */
int gs_boot_population(gs_handle h, const gs_jobin *trace, int64_t k);
int gs_boot_traces(gs_handle h, const gs_boot_params *params /* nsims */, double *kernel_ms);
int gs_boot_traces_blocked(gs_handle h, const gs_boot_params *params /* nsims */, const uint32_t *block_len /* nsims; NULL = all 1 */,
                           double *kernel_ms);
int gs_fetch_trace(gs_handle h, int sim, gs_jobin *out /* n records */);

/* ---- mixed bootstrap replicas: another job mix drawn from the same population ----------------------------
 * gs_boot_mixes gives the handle nmix mixes of the current population (weights: nmix * k uint32, mix-major): mix m
 * draws row i with probability w_i / T, T = sum over i of w_i >= 1.  Each mix becomes an exact integer alias table
 * (Walker / Vose) on the host: with q_i = w_i * k (below 2^63, as is T), take FIFO worklists S = {i : q_i < T} and
 * G = {i : q_i >= T} in ascending row order; while both are non-empty, take s from the front of S, let g be the front
 * of G, set U_s = q_s, A_s = g and q_g -= T - q_s, and move g from the front of G to the back of S once q_g < T; every
 * row still in G gets U_i = T, A_i = i.  The tables are uploaded as one device array; nmix = 0 clears them, and so does
 * a new gs_boot_population.
 * gs_boot_traces_mixed is gs_boot_traces_blocked where replica sim with mix[sim] = m >= 0 picks its rows through mix m:
 * with c = floor(w0 * k / 2^64) and u = floor(w3 * T / 2^64), the row is c if u < U_c, else A_c (row m' has
 * probability w_m' / T to within 2^-64 per column).  A blocked replica (L > 1) picks s_b this way at block starts only;
 * a block still continues through the base trace in order, so it can copy rows of weight 0, and the shares of the
 * rows equal the mix only at L = 1.  Gaps, arrivals, the arrival bound and every other field are those of
 * gs_boot_traces_blocked, and the same (seed, stream) stays coupled across mixes, loads and block lengths.  Equal
 * weights give U_i = T for every row: the unweighted replica byte for byte.  mix[sim] = -1 (mix NULL: all -1) is the
 * unweighted replica, and a call without any mix >= 0 is gs_boot_traces_blocked exactly (the same launches).
 * Errors (nothing changes): gs_boot_mixes: GS_ERR_ARG for nmix < 0, NULL weights with nmix > 0 or a mix with T = 0,
 * GS_ERR_STATE without a population, GS_ERR_CUDA if the tables cannot be allocated; gs_boot_traces_mixed: the errors of
 * gs_boot_traces_blocked, checked in the same order, then GS_ERR_ARG for mix[sim] outside [-1, nmix).          */
int gs_boot_mixes(gs_handle h, int32_t nmix, const uint32_t *weights /* nmix * k, mix-major */);
int gs_boot_traces_mixed(gs_handle h, const gs_boot_params *params /* nsims */, const uint32_t *block_len /* NULL = all 1 */,
                         const int32_t *mix /* nsims, -1 = unweighted; NULL = all -1 */, double *kernel_ms);

/* ---- profiled bootstrap replicas: a time-varying offered load ----------------------------------------------
 * gs_boot_profiles gives the handle nprof load profiles (segs: the nseg[p] segments of every profile p in turn).
 * Profile p has m = nseg[p] segments, 1 <= m <= GS_BOOT_MAX_SEGMENTS, and a period P = period[p] >= 0.  Segment k
 * starts at tick t_k = segs[k].start (t_0 = 0, strictly increasing, below 2^31 - 1) and scales the gaps it spans by
 * gap_num / gap_den (both >= 1; reserved is ignored, set it to 0).  P = 0: the last segment never ends; P > 0: the
 * profile repeats with period P, t_(m-1) < P < 2^31 - 1.  The host converts each profile once, exactly, to base-time
 * starts s_0 = 0, s_(k+1) = s_k + ceil((t_(k+1) - t_k) * den_k / num_k), and B = s_m with t_m := P (P > 0), and
 * uploads them as one device array; nprof = 0 clears them.  Profiles do not depend on the population: a new
 * gs_boot_population keeps them.
 * gs_boot_traces_profiled is gs_boot_traces_mixed where replica sim with profile[sim] = p >= 0 takes its arrivals
 * from profile p: with S the job's gap sum (the base time gs_boot_traces scales by gap_num / gap_den),
 *   a(S) = t_k + floor((S - s_k) * num_k / den_k), k the last segment with s_k <= S
 *   arrive = a(S) (P = 0), or (S div B) * P + a(S mod B) (P > 0).
 * Arrivals never decrease, and the first base time that reaches t_k is s_k, which arrives exactly at t_k (in every
 * period).  Rows, gaps, block starts and mix picks are those of the same replica without a profile, so the same
 * (seed, stream) stays coupled across profiles; a profiled replica's params[sim] must have gap_num / gap_den = 1 / 1.
 * One segment {0, num, den} with P = 0 is the unprofiled replica at gap scale num / den, byte for byte, and a
 * periodic {0, 1, 1} is the identity.  profile[sim] = -1 (profile NULL: all -1) keeps the replica unprofiled, and a
 * call without any profile >= 0 is gs_boot_traces_mixed exactly (the same launches).
 * Errors (nothing changes): gs_boot_profiles: GS_ERR_ARG for nprof < 0, NULL arrays with nprof > 0 or a profile
 * that breaks a rule above; GS_ERR_CUDA if the profiles cannot be allocated.  gs_boot_traces_profiled: the errors of
 * gs_boot_traces_mixed, checked in the same order (a profiled replica's arrival bound is its profile's, below), then
 * GS_ERR_ARG for profile[sim] outside [-1, nprof), a profiled replica whose gap scale is not 1 / 1, and a profiled
 * replica whose worst-case last arrival arrive((n - 1) * max(D)), computed exactly, reaches 2^31 - 1.          */
#define GS_BOOT_MAX_SEGMENTS 64
typedef struct gs_boot_seg {
  int32_t start, gap_num, gap_den, reserved;
} gs_boot_seg;              /* 16 bytes */
int gs_boot_profiles(gs_handle h, int32_t nprof, const int32_t *nseg /* nprof */, const int32_t *period /* nprof */,
                     const gs_boot_seg *segs /* sum of nseg, profile-major */);
int gs_boot_traces_profiled(gs_handle h, const gs_boot_params *params /* nsims */, const uint32_t *block_len /* NULL = all 1 */,
                            const int32_t *mix /* NULL = all -1 */, const int32_t *profile /* nsims, -1 = none; NULL = all -1 */,
                            double *kernel_ms);

/* Stateless candidate scoring: evaluate b jobs against ONE cluster state.
 * first_node[i] = node of a single-node first fit, or the first node of a
 * cross-node fill, or -1 if the job cannot be placed; task_node (optional)
 * receives the node of each task at task_off[i] .. task_off[i+1].               */
int gs_place_batch(gs_handle h, const gs_cluster *cluster, const gs_node *nodes, int32_t m,
                   const gs_jobreq *jobs, int64_t b, int32_t *first_node,
                   int32_t *nodes_used, const int64_t *task_off, int32_t *task_node,
                   double *kernel_ms);

/* ---- legacy switch-local yarn placement with parameter-server traffic accounting (SURVEY row a13) --------
 * _Cluster.ms_yarn_placement (infra/cluster.py:888-898) over _Switch.try_cross_node_alloc / try_single_node_alloc
 * (infra/switch.py:38-167,190-206): all gpus of a job come from ONE switch; a job wider than a node takes
 * floor(g/G) completely idle nodes plus one node for the remainder, is charged 6 cpus per gpu and
 * (ps_mem + g*p_w_mem + worker_mem) memory per gpu, and every node's network load grows by
 *   round(model*k, 1), then per PS shard on the node:  += ps*(g-k);  -= ps*k;  round(., 1)     (switch.py:98-108)
 * (Python's round, reproduced exactly).  `ncl` independent clusters per call; the jobs of a cluster are placed in
 * order and change its node table (in/out).  spans: caller-sized, job j writes at span_off (floor(g/G)+1 slots);
 * network is NaN on the single-node path (the reference records none there).                              */
typedef struct gs_switch_cluster {
  int32_t num_switch, num_node_p_switch, num_gpu_p_node, reserved;
  int64_t node_off;        /* first record of this cluster in `nodes` (num_switch * num_node_p_switch records)   */
  int64_t job_off, job_cnt;
} gs_switch_cluster;
typedef struct gs_switch_node { int32_t free_gpus, free_cpus; double free_mem; double net_in; } gs_switch_node;
typedef struct gs_switch_job {
  int32_t num_gpu, n_ps;   /* job['num_gpu'], len(job['ps_network'])                                             */
  int64_t ps_off;          /* first entry of the job's ps_network in `ps_network`                                */
  int64_t span_off;        /* where the job's per-node records go in `spans`                                     */
  double model_size;       /* job['model']['total_size']                                                         */
} gs_switch_job;
typedef struct gs_switch_ans { int32_t n_nodes; int32_t sw; } gs_switch_ans;   /* n_nodes == 0: not placed      */
typedef struct gs_switch_span { int32_t node, num_gpu, num_cpu, reserved; double mem, network; } gs_switch_span;
int gs_switch_yarn(gs_handle h, int32_t ncl, const gs_switch_cluster *clusters, gs_switch_node *nodes, int64_t n_nodes,
                   const gs_switch_job *jobs, int64_t n_jobs, const double *ps_network, int64_t n_ps,
                   double worker_mem, double ps_mem, double p_w_mem,
                   gs_switch_ans *ans, gs_switch_span *spans, int64_t n_spans);

/* ---- host side of the log writer (no device work): the sampled avg_gpu_utilization column of cluster.csv.
 * The reference draws one np.random.normal per busy device and tick, nodes in id order, devices 0..G-1
 * (infra/device.py:48-54, core/scheduling/schedule.py:103-120), from numpy's sequential global stream; the caller draws the
 * standard-normal values from numpy, these entry points consume them in that order.  A holding = one (job, device)
 * pair counted on rows first..last; holdings are passed sorted by `first`, key = node * G + device.                */
typedef struct gs_logcol_s *gs_logcol;
gs_logcol gs_logcol_open(int64_t n_rows, int32_t width, int64_t n_hold, const int64_t *first, const int64_t *last,
                         const int32_t *key, const int32_t *job);
void gs_logcol_close(gs_logcol c);
int gs_logcol_counts(gs_logcol c, int64_t *counts);                  /* values consumed by each row                  */
int gs_logcol_rows(gs_logcol c, int64_t r_end, const double *loc, const double *scale, const double *z, int64_t n_z,
                   double *acc, int32_t *unclipped);                 /* rows [current, r_end): sums in draw order     */

/* PS<->worker transfer time for a batch of placed jobs.  task_node holds the
 * node of every task (segments given by task_off), is_ps marks PS tasks.        */
int gs_net_cost(gs_handle h, const gs_cluster *cluster, int64_t b,
                const int64_t *task_off, const int32_t *task_node, const uint8_t *is_ps,
                const int32_t *ps_count, const double *model_mb, const double *iterations,
                double *extra_out);

#ifdef __cplusplus
}
#endif
#endif /* GSCHED_H_ */

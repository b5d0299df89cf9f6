/*
 * gsched_horus.h -- C ABI of the utilisation-aware placement engine (horus / gandiva).
 *
 * Widening row f1 (SURVEY 8(f) rank 1) of the simulator hot path: the same tick loop as gsched.h,
 * with the reference's score-based placement and its two schedulers in place of yarn + fifo:
 *
 *   placement_algorithms['horus' | 'gandiva'] = horus_placement     core/scheduling/algorithm.py:34-180,182-187
 *   placement_algorithms['yarn'] under the same schedulers          core/scheduling/algorithm.py:28-32,301-417
 *   score_fn['horus' | 'gandiva']                                    core/scheduling/horus.py:6-56, algorithm.py:9-13
 *   scheduling_algorithms['horus'] = schedule_horus (look-ahead)     core/scheduling/algorithm.py:204-240,292-298
 *   scheduling_algorithms['gandiva'] = schedule_fifo + time slicing  core/scheduling/algorithm.py:189-202,420-444
 *   Device / Node packing rules (4 tasks per device, 500 MiB margin) infra/device.py:20-76, infra/node.py:57-232
 *
 * The reference samples numpy's global random stream inside these decisions (device.py:31,52).
 * The caller passes that stream as standard-normal values (numpy.random.standard_normal(count) drawn
 * from the same generator state the reference run would start from); the engine consumes them in the
 * reference's order, so a seeded reference run is reproduced bit for bit.  A stream that is too short
 * ends the run with GS_ERR_CAPACITY (load a longer one and run again).
 *
 * horus+ (credit queues re-clustered by k-means every tick, jobs_manager.py:93-139, algorithm.py:242-290)
 * interleaves integer draws with the normal samples, so it takes the stream as raw generator words instead
 * (gs_horus_load_words); the host side of the library tabulates the normal sampler over them.
 *
 * Conventions as in gsched.h: 0 / negative gs_status, caller-owned host buffers, one handle per
 * device and driving thread, no CPU fallback (gs_horus_create fails without a CUDA device).
 */
#ifndef GSCHED_HORUS_H
#define GSCHED_HORUS_H

#include <stdint.h>

#include "gsched.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Which score_fn runs (algorithm.py:9-13).  NOTE: the reference indexes score_fn with the SCHEDULE name
 * (schedule.py:47 passes self.schedule down as `scheme`; algorithm.py:58,196): horus and horus+ -> horus_score,
 * gandiva -> gandiva_score, fifo -> KeyError.  --scheme horus|horus+|gandiva only selects horus_placement. */
enum { GS_HSCORE_HORUS = 0, GS_HSCORE_GANDIVA = 1 };
enum { GS_HSCHED_FIFO = 0, GS_HSCHED_HORUS = 1, GS_HSCHED_HORUS_PLUS = 2, GS_HSCHED_GANDIVA = 3 };   /* --schedule (algorithm.py:292-298) */

enum { GS_HPLACE_HORUS = 0, GS_HPLACE_YARN = 1 };   /* --scheme: horus | horus+ | gandiva -> horus_placement, yarn -> ms_yarn_placement (algorithm.py:182-187) */

typedef struct gs_horus_params {
  int32_t score;        /* GS_HSCORE_* */
  int32_t schedule;     /* GS_HSCHED_* */
  int32_t num_buffer;   /* look-ahead width k of schedule_horus (--num_buffer, run_sim.py:76) */
  int32_t num_queue;    /* horus+: number of credit queues (--num_queue, run_sim.py:75); 0 or 1 otherwise */
  int32_t placement;    /* GS_HPLACE_* */
  int32_t reserved;
} gs_horus_params;

/* One finished (or unfinished) job: the fields LogManager.jcts prints (log_manager.py:137-153). */
typedef struct gs_horus_job_rec {
  int32_t start, end;   /* Job.start_time (last start), Job.end_time */
  int32_t jct;          /* Job.time_processed() */
  int32_t preempt;      /* Job.migration_count */
  double original;      /* Job.duration */
  double actual;        /* Job.get_duration(): longest task duration incl. interference penalties */
} gs_horus_job_rec;

typedef struct gs_horus_run_stats {
  int64_t ticks, events, draws;     /* rows written; arrivals + starts + completions + preemptions; samples consumed */
  int32_t finished, queued, running, done;
  int32_t status, reserved;
  float kernel_ms, reserved2;
} gs_horus_run_stats;

typedef struct gs_horus_handle_s *gs_horus_handle;

int gs_horus_create(int device, int nsims, gs_horus_handle *out);
int gs_horus_destroy(gs_horus_handle h);
/* Infrastructure(FLAGS) + --scheme / --schedule / --num_buffer   (infra/infrastructure.py:26-58, run_sim.py:25-49,76) */
int gs_horus_config(gs_horus_handle h, int32_t sim, const gs_cluster *cluster, const gs_horus_params *params);
/* Job(idx, minutes*0.5, normalized_time, gpu_per_container, gpu_utilization_avg/max, memory_max, used_gpus)
 * per trace row  (core/jobs/jobs_manager.py:233-239); rows in admission order, arrive = ceil(normalized_time). */
int gs_horus_load_trace(gs_horus_handle h, int32_t sim, int64_t n, const int32_t *arrive, const int32_t *gpus,
                        const int32_t *gpu_per_task, const double *duration, const int64_t *mem_bytes,
                        const double *util_avg, const double *util_max, const double *mem_avg_mib /* horus+ only, may be NULL */);
/* The numpy stream the run consumes (see the header comment).  sim = -1: one stream shared by every replica
 * of the handle, each reading it from position 0 (replicas that differ in trace or parameters only). */
int gs_horus_load_stream(gs_horus_handle h, int32_t sim, const double *standard_normal, int64_t count);
/* The same numpy stream as raw MT19937 output words (numpy.random.randint(0, 2**32, count, dtype=uint32) from the
 * generator state the reference run would start from).  Serves every schedule and is REQUIRED for horus+, whose
 * k-means integer draws (core/jobs/utils.py:39,62) share the stream with the normal samples.  sim = -1: shared. */
int gs_horus_load_words(gs_horus_handle h, int32_t sim, const uint32_t *mt19937_words, int64_t count);
/* Scheduler.start() for every configured replica: runs to completion, or max_ticks ticks (0 = no limit). */
int gs_horus_run(gs_horus_handle h, int64_t max_ticks, int64_t rows_cap);
int gs_horus_stats(gs_horus_handle h, int32_t sim, gs_horus_run_stats *out);
/* cluster.csv rows (LogInfo, schedule.py:95-133) with the sampled utilisation column as value + "is a numpy
 * array" flag (how str() prints it), and the job records in finish order. */
int gs_horus_fetch(gs_horus_handle h, int32_t sim, gs_tick_row *rows, double *util, uint8_t *util_is_array,
                   int64_t rows_cap, gs_horus_job_rec *recs, int32_t *finish_order, int64_t *n_rows, int64_t *n_finished);
/* Run summaries (gs_summary, gsched.h) of replicas [first, first + count), computed on the device from every row the
 * replicas hold -- [0, ticks): a replica that ran out of rows starts over, so there is no window to carry across --
 * and from their finished jobs.  util_sum is the sum of the sampled avg_gpu_utilization values (NaN counted as 0).
 * kernel_ms (may be NULL) receives the device time of the summary kernels.  GS_ERR_ARG for a bad range,
 * GS_ERR_STATE for a replica that has not run. */
int gs_horus_summarize(gs_horus_handle h, int32_t first, int32_t count, gs_summary *out, double *kernel_ms);
/* Timeline (gs_tbin, gsched.h) filled by gs_horus_summarize from the same rows [0, ticks) with the sampled utilisation
 * (util_sum).  gs_horus_summarize folds every row again on every call, so the timeline may be set at any time; setting
 * it marks every replica as not summarised.  Errors as gs_set_timeline / gs_fetch_timeline.                 */
int gs_horus_set_timeline(gs_horus_handle h, int64_t bin_width, int32_t nbins);
int gs_horus_fetch_timeline(gs_horus_handle h, int32_t first, int32_t count, gs_tbin *out);
/* Job statistics by job size (gs_jclass and CDF histograms, gsched.h) filled by gs_horus_summarize from the same
 * finished jobs as its job part.  Same meaning and errors as gs_set_jobdist / gs_fetch_jobdist.                 */
int gs_horus_set_jobdist(gs_horus_handle h, int32_t nclasses, const int32_t *bounds, int32_t nedges, const int32_t *edges);
int gs_horus_fetch_jobdist(gs_horus_handle h, int32_t first, int32_t count, gs_jclass *classes_out, uint32_t *hist_out);
/* Job statistics by a chosen key with bounded slowdown (gs_sdclass and CDF histograms, gsched.h) filled by
 * gs_horus_summarize from the same finished jobs.  Same meaning and errors as gs_set_slowdown / gs_fetch_slowdown. */
int gs_horus_set_slowdown(gs_horus_handle h, const gs_slowdown_cfg *cfg);
int gs_horus_fetch_slowdown(gs_horus_handle h, int32_t first, int32_t count, gs_sdclass *out, uint32_t *hist_out);
/* Job statistics by arrival time (gs_abin, gsched.h) filled by gs_horus_summarize from the same finished jobs and the
 * replica's loaded trace.  Same meaning and errors as gs_set_arrivals / gs_fetch_arrivals.                      */
int gs_horus_set_arrivals(gs_horus_handle h, int64_t bin_width, int32_t nbins, int64_t tau);
int gs_horus_fetch_arrivals(gs_horus_handle h, int32_t first, int32_t count, gs_abin *out);
/* Time-weighted occupancy (gs_occ and histograms, gsched.h) filled by gs_horus_summarize from the same rows [0, ticks),
 * every row one tick.  gs_horus_summarize folds every row again on every call, so no carry is kept and the feature may
 * be set at any time; setting it marks every replica as not summarised.  Otherwise the same meaning and errors as
 * gs_set_occupancy / gs_fetch_occupancy.                                                                      */
int gs_horus_set_occupancy(gs_horus_handle h, int32_t on, int32_t nedges, const int32_t *edges);
int gs_horus_fetch_occupancy(gs_horus_handle h, int32_t first, int32_t count, gs_occ *out, uint64_t *busy_hist, int32_t busy_pitch,
                             uint64_t *queue_hist);
/* ---- interference statistics (interference) -------------------------------------------------------------------
 * The jobs are jobdist's: the finished jobs of gs_summary's job part, classed by jobdist's C - 1 bounds on num_gpu
 * (1 <= C <= GS_JOBDIST_MAX_CLASSES, the same rules).  A job is DEGRADED when actual > original (its gs_horus_job_rec,
 * compared as doubles): co-location stretched its longest task.  Every other finished job is clean.
 * Durations are kept in fixed point, units of 2^-10 tick: fp(x) = min(2^31 - 1, max(0, round(1024 * x))), rounded to
 * nearest with ties to even.  a = fp(actual) and o = fp(original) for every job; e = fp(actual - original), the
 * difference taken in IEEE double, for a degraded job.  The rounding makes the reference's interference penalty of 5
 * ticks, which reaches the records as 4.999999999999998 or 5.0, one value (e = 5120).  `clamped` counts the jobs with a
 * value that saturated (or was NaN).  Per class one gs_ifclass, every field an integer (a repeated call gives the
 * same bytes):
 *   degraded, clean      jobdist's gs_jclass restricted to each group (degraded + clean = gs_horus_fetch_jobdist's
 *                        record under the same bounds, for counts and sums)
 *   degraded_jct_mid     the degraded jobs' jct at ranks floor((k - 1) / 2) and ceil((k - 1) / 2) (the median is
 *                        their mean; [0] equals degraded.jct_q[0])
 *   actual_*             a over the class's finished jobs: sum, 128-bit sum of squares, gs_summary's 50 / 90 / 95 /
 *                        99 / 100 % and the two middle order statistics
 *   original_sum         sum of o
 *   excess_*, lost_gpu_time_*   over the degraded jobs: sum and maximum of e, 128-bit sum of gpus * e
 *   preempted_jobs, preempt_max jobs with preempt > 1 (gandiva's time slicing) and the largest preempt
 * Order statistics and maxima are 0 for an empty group. */
typedef struct gs_ifclass {
  gs_jclass degraded, clean;
  int64_t actual_sum;
  uint64_t actual_sq_lo, actual_sq_hi;
  int64_t original_sum;
  int64_t excess_sum;
  uint64_t lost_gpu_time_lo, lost_gpu_time_hi;
  int64_t preempted_jobs;
  int64_t clamped;
  int32_t degraded_jct_mid[2];
  int32_t actual_q[5];
  int32_t actual_mid[2];
  int32_t excess_max;
  int32_t preempt_max;
  int32_t reserved;
} gs_ifclass;                        /* 440 bytes */
/* gs_horus_set_interference: while nclasses > 0, every gs_horus_summarize also computes the class records of the
 * replicas it summarises; nclasses = 0 (the default) turns it off.  Every replica is marked as not summarised with
 * this setting.  GS_ERR_ARG for nclasses outside 0..8, bounds that are not strictly increasing or below 1, or NULL
 * bounds with nclasses > 1; nothing changes on an error.
 * gs_horus_fetch_interference copies count * C records (replica-major) as of the last gs_horus_summarize.  GS_ERR_ARG
 * for a bad range or a NULL output, GS_ERR_STATE when the feature is off or a replica has not been summarised with
 * this setting since it was prepared.                                                                          */
int gs_horus_set_interference(gs_horus_handle h, int32_t nclasses, const int32_t *bounds);
int gs_horus_fetch_interference(gs_horus_handle h, int32_t first, int32_t count, gs_ifclass *out);
/* Paired per-job comparison (gs_jpair, gsched.h: gs_compare) of replicas of this handle that hold the same trace: equal
 * arrival, gpus, gpu_per_container, duration, memory, utilisation and mean-memory fields for every job.  The same
 * outputs, launches and errors as gs_compare; a replica has run once gs_horus_run has prepared it.           */
int gs_horus_compare(gs_horus_handle h, int32_t npairs, const int32_t *a, const int32_t *b, int32_t nclasses, const int32_t *bounds,
                     int32_t nedges, const int32_t *edges, gs_jpair *out, uint32_t *hist_out, double *kernel_ms);
/* Kernel mapping (no reference counterpart): simulations per warp, 1 (default: lane 0 of each warp) or 32; 0 = one
 * simulation per warp with all 32 lanes scoring a candidate job's devices together (gs_horus_coop_kernel). */
int gs_horus_set_lanes(gs_horus_handle h, int lanes_per_warp);
int64_t gs_horus_launch_count(gs_horus_handle h);
const char *gs_horus_last_error(gs_horus_handle h);
/* "cuda:sm_90a" for the shipped library.  The test suite also compiles this file's host side with g++ against a
 * stand-in CUDA runtime (tests/emu); that build answers "host-emulation" and the package refuses to load it. */
const char *gs_horus_build_tag(void);

#ifdef __cplusplus
}
#endif
#endif

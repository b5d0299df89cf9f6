// gs_summary.cuh -- on-device run summaries (gs_summary, include/gsched.h), included by gsched.cu and gs_horus.cu.
//
// A replica's run is reduced to the few numbers the reference's notebooks compute from its cluster.csv / job.csv.
// Two parts:
//   * rows: one block per replica folds gs_tick_rows (event-driven policies, horus) or, for fifo, the compact
//     records directly -- record k stands for the rows now_k .. now_(k+1) - 1, on which only `delta` and the pending
//     terms move, linearly (gs_expand_rows_kernel), so each record is folded in closed form and no row is rebuilt;
//   * jobs: the three per-job values (wait, turnaround, jct) of every finished job are written once to scratch, and
//     a block-wide radix select over 9-bit digits finds the 15 order statistics (3 values x 5 ranks) in the same
//     passes: ceil(bits / 9) passes, where bits is the width of the largest value range (about 18 on the BASELINE
//     trace: two passes).
// The per-row arithmetic, the record fold and the rank / digit arithmetic are __host__ __device__ functions: the
// host-emulation build of gs_horus.cu (tests/emu) runs them on the CPU, and so can a CPU test.
#pragma once

#include <math.h>
#include <stdint.h>

#include "gsched.h"
#include "gsched_horus.h"

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#endif
#ifndef __device__
#define __device__
#endif
#endif

#define GS_SUM_HD static __host__ __device__ inline
#define GS_SUM_THREADS 256
#define GS_SUM_BINS 512            // 9-bit digits
#define GS_SUM_TARGETS 15          // {wait, turnaround, jct} x {50, 90, 95, 99, 100 %}

static_assert(sizeof(gs_summary) == 256, "gs_summary is 256 bytes");

typedef __int128 gs_i128;
typedef unsigned __int128 gs_u128;

// Partial fold of some rows (one thread's share, then block-reduced).
struct GsSumPart {
  long long rows, busy, running, queued, pending_rows;
  int busy_max, running_max, queued_max, pend_max;
  gs_i128 pend, mem;
  double avg, util;
};

GS_SUM_HD void gs_sum_zero(GsSumPart &p) {
  p.rows = p.busy = p.running = p.queued = p.pending_rows = 0;
  p.busy_max = p.running_max = p.queued_max = p.pend_max = 0;
  p.pend = 0; p.mem = 0; p.avg = 0.0; p.util = 0.0;
}

GS_SUM_HD int gs_sum_imax(int a, int b) { return a > b ? a : b; }

GS_SUM_HD double gs_sum_i128_to_double(gs_i128 x) {
  const long long lo = (long long)x;
  if ((gs_i128)lo == x) return (double)lo;
  return (double)(long long)(x >> 64) * 18446744073709551616.0 + (double)(unsigned long long)x;
}

// One cluster.csv row.  `util`: the sampled avg_gpu_utilization value (horus), NaN counted as 0; 0 when there is none.
GS_SUM_HD void gs_sum_row(GsSumPart &p, const gs_tick_row &r, double util) {
  p.rows += 1;
  p.busy += r.busy_gpus; p.running += r.running; p.queued += r.queued;
  p.busy_max = gs_sum_imax(p.busy_max, r.busy_gpus); p.running_max = gs_sum_imax(p.running_max, r.running);
  p.queued_max = gs_sum_imax(p.queued_max, r.queued); p.pend_max = gs_sum_imax(p.pend_max, r.pend_max);
  p.pend += (gs_i128)r.pend_sum; p.mem += (gs_i128)r.mem_busy_bytes;
  if (r.queued > 0 && r.pend_sum != 0) {      // avg_pending_time != 0 (log_manager.pending_columns)
    p.pending_rows += 1;
    p.avg += (double)r.pend_sum / ((double)r.queued + 1e-9);
  }
  if (util == util) p.util += util;
}

// The rows v_lo .. v_hi (values of `delta`) of one fifo record: every counter is constant there, and the pending sum of
// row v is queued * v - arrive_sum (q = the same-tick gs_qrow; arrive_sum / oldest are unused when queued == 0).
// avg_pending_sum: the denominator queued + 1e-9 is constant within the record, so the record adds
// (sum of its nonzero pending sums) / (queued + 1e-9).
GS_SUM_HD void gs_sum_record(GsSumPart &p, const gs_evrow &e, long long arrive_sum, int oldest, long long v_lo, long long v_hi) {
  const long long L = v_hi - v_lo + 1;
  if (L <= 0) return;
  p.rows += L;
  p.busy += (long long)e.busy_gpus * L; p.running += (long long)e.running * L; p.queued += (long long)e.queued * L;
  p.busy_max = gs_sum_imax(p.busy_max, e.busy_gpus); p.running_max = gs_sum_imax(p.running_max, e.running);
  p.queued_max = gs_sum_imax(p.queued_max, e.queued);
  p.mem += (gs_i128)e.mem_busy_bytes * L;
  if (e.queued > 0) {
    const long long q = e.queued;
    const long long sv = (v_lo + v_hi) * L / 2;                     // sum of v over the record (exact: (v_lo + v_hi) * L is even)
    const gs_i128 x = (gs_i128)q * sv - (gs_i128)L * arrive_sum;
    p.pend += x;
    p.pend_max = gs_sum_imax(p.pend_max, (int)(v_hi - oldest));
    // q * v - arrive_sum grows with v: it is zero on at most one row, v = arrive_sum / q
    const bool zero = arrive_sum % q == 0 && arrive_sum / q >= v_lo && arrive_sum / q <= v_hi;
    const long long nz = L - (zero ? 1 : 0);
    p.pending_rows += nz;
    if (nz > 0) p.avg += gs_sum_i128_to_double(x) / ((double)q + 1e-9);
  }
}

GS_SUM_HD void gs_sum_merge(GsSumPart &a, const GsSumPart &b) {
  a.rows += b.rows; a.busy += b.busy; a.running += b.running; a.queued += b.queued; a.pending_rows += b.pending_rows;
  a.busy_max = gs_sum_imax(a.busy_max, b.busy_max); a.running_max = gs_sum_imax(a.running_max, b.running_max);
  a.queued_max = gs_sum_imax(a.queued_max, b.queued_max); a.pend_max = gs_sum_imax(a.pend_max, b.pend_max);
  a.pend += b.pend; a.mem += b.mem; a.avg += b.avg; a.util += b.util;
}

GS_SUM_HD void gs_sum_add128(uint64_t &lo, uint64_t &hi, gs_i128 v) {
  const gs_u128 s = (((gs_u128)hi << 64) | (gs_u128)lo) + (gs_u128)v;
  lo = (uint64_t)s; hi = (uint64_t)(s >> 64);
}

// Add a fold to a summary's row part (rows, sums, maxima; makespan is set by the caller).
GS_SUM_HD void gs_sum_add_rows(gs_summary &s, const GsSumPart &p) {
  s.rows += p.rows;
  s.busy_gpus_sum += p.busy; s.running_sum += p.running; s.queued_sum += p.queued;
  s.busy_gpus_max = gs_sum_imax(s.busy_gpus_max, p.busy_max); s.running_max = gs_sum_imax(s.running_max, p.running_max);
  s.queued_max = gs_sum_imax(s.queued_max, p.queued_max); s.pend_max_max = gs_sum_imax(s.pend_max_max, p.pend_max);
  gs_sum_add128(s.pend_sum_lo, s.pend_sum_hi, p.pend);
  gs_sum_add128(s.mem_busy_lo, s.mem_busy_hi, p.mem);
  s.pending_rows += p.pending_rows; s.avg_pending_sum += p.avg; s.util_sum += p.util;
}

// ---- timeline (gs_tbin): the row fold above, keyed by bin = min(floor(delta / W), B - 1)
static_assert(sizeof(gs_tbin) == 128, "gs_tbin is 128 bytes");

// Partial fold of some rows of ONE bin.  `last` orders rows (row index, or `delta` for the fifo records, which are
// monotone): `fin` is the `finished` counter of the row with the largest `last`.
struct GsTlPart {
  GsSumPart s;
  long long dmin, dmax, last, fin;
};

GS_SUM_HD int gs_tl_bin(long long delta, long long W, int B) {
  if (delta < 0) return 0;
  const long long b = delta / W;
  return b < B - 1 ? (int)b : B - 1;
}

GS_SUM_HD void gs_tl_zero(GsTlPart &p) {
  gs_sum_zero(p.s);
  p.dmin = 0x7fffffffffffffffll; p.dmax = -0x7fffffffffffffffll - 1; p.last = -1; p.fin = 0;
}

GS_SUM_HD void gs_tl_row(GsTlPart &p, const gs_tick_row &r, double util, long long index) {
  gs_sum_row(p.s, r, util);
  p.dmin = r.now < p.dmin ? r.now : p.dmin; p.dmax = r.now > p.dmax ? r.now : p.dmax;
  if (index > p.last) { p.last = index; p.fin = r.finished; }
}

// The rows v_lo .. v_hi of one fifo record (already clipped to the bin and to the watermark; nothing if empty).
GS_SUM_HD void gs_tl_record(GsTlPart &p, const gs_evrow &e, long long arrive_sum, int oldest, long long v_lo, long long v_hi) {
  if (v_hi < v_lo) return;
  gs_sum_record(p.s, e, arrive_sum, oldest, v_lo, v_hi);
  p.dmin = v_lo < p.dmin ? v_lo : p.dmin; p.dmax = v_hi > p.dmax ? v_hi : p.dmax;
  if (v_hi > p.last) { p.last = v_hi; p.fin = e.finished; }
}

GS_SUM_HD void gs_tl_merge(GsTlPart &a, const GsTlPart &b) {
  gs_sum_merge(a.s, b.s);
  a.dmin = b.dmin < a.dmin ? b.dmin : a.dmin; a.dmax = b.dmax > a.dmax ? b.dmax : a.dmax;
  if (b.last > a.last) { a.last = b.last; a.fin = b.fin; }
}

// Add a partial to a bin.  Partials reach a bin in row order (later windows, later runs of rows), so the newest one
// carries the bin's last row.
GS_SUM_HD void gs_tl_add(gs_tbin &t, const GsTlPart &p) {
  if (p.s.rows == 0) return;
  if (t.rows == 0) { t.delta_min = p.dmin; t.delta_max = p.dmax; }
  else { t.delta_min = p.dmin < t.delta_min ? p.dmin : t.delta_min; t.delta_max = p.dmax > t.delta_max ? p.dmax : t.delta_max; }
  t.finished_last = p.fin;
  t.rows += p.s.rows;
  t.busy_gpus_sum += p.s.busy; t.running_sum += p.s.running; t.queued_sum += p.s.queued;
  t.busy_gpus_max = gs_sum_imax(t.busy_gpus_max, p.s.busy_max); t.running_max = gs_sum_imax(t.running_max, p.s.running_max);
  t.queued_max = gs_sum_imax(t.queued_max, p.s.queued_max); t.pend_max_max = gs_sum_imax(t.pend_max_max, p.s.pend_max);
  gs_sum_add128(t.pend_sum_lo, t.pend_sum_hi, p.s.pend);
  gs_sum_add128(t.mem_busy_lo, t.mem_busy_hi, p.s.mem);
  t.pending_rows += p.s.pending_rows; t.avg_pending_sum += p.s.avg; t.util_sum += p.s.util;
}

// Rows lo .. hi - 1 (rows[i - base]; util may be NULL) in row order, one partial per run of rows that share a bin.
// Any order of `delta` is binned correctly.  The bin kernel's path for rows whose `delta` is not monotone (run by one
// thread) and the host-emulation build's horus timeline.
GS_SUM_HD void gs_tl_fold_rows_serial(gs_tbin *bins, int B, long long W, const gs_tick_row *rows, const double *util,
                                      long long base, long long lo, long long hi) {
  GsTlPart p;
  gs_tl_zero(p);
  int cur = -1;
  for (long long i = lo; i < hi; ++i) {
    const gs_tick_row &r = rows[i - base];
    const int b = gs_tl_bin(r.now, W, B);
    if (b != cur) {
      if (cur >= 0) gs_tl_add(bins[cur], p);
      gs_tl_zero(p);
      cur = b;
    }
    gs_tl_row(p, r, util ? util[i - base] : 0.0, i);
  }
  if (cur >= 0) gs_tl_add(bins[cur], p);
}

// ---- jobs
struct GsSumJob { int wait, turn, jct, preempt, gpus; };

GS_SUM_HD GsSumJob gs_sum_job(int arrive, int start, int end, int jct, int preempt, int gpus) {
  GsSumJob v; v.wait = start - arrive; v.turn = end - arrive; v.jct = jct; v.preempt = preempt; v.gpus = gpus;
  return v;
}

// fifo's run length, max(1, ceil(duration)) ticks (quirk Q11; need_of in gs_tick2.cuh)
GS_SUM_HD int gs_sum_run_length(double dur) {
  const double c = ceil(dur);
  return c < 1.0 ? 1 : (c > 1.0e9 ? 0x7fffffff : (int)c);
}

GS_SUM_HD int gs_sum_permille(int t) { return t == 0 ? 500 : t == 1 ? 900 : t == 2 ? 950 : t == 3 ? 990 : 1000; }

// Nearest rank: of k > 0 values sorted ascending, rank q per mille is element ceil(q * k / 1000) - 1.
GS_SUM_HD long long gs_sum_rank(int permille, long long k) { return (permille * k + 999) / 1000 - 1; }

// Radix passes over 9-bit digits needed for values whose range (max - min) is `span`.
GS_SUM_HD int gs_sum_passes(unsigned long long span) {
  int bits = 1;
  while (bits < 64 && (span >> bits) != 0) ++bits;
  return (bits + 8) / 9;
}

// One radix step: the digit whose bin holds element `rank` of the group the histogram counts; rank becomes the
// element's rank inside that bin.
GS_SUM_HD unsigned gs_sum_pick(const unsigned *hist, long long &rank) {
  long long below = 0;
  unsigned d = 0;
  for (; d + 1 < GS_SUM_BINS; ++d) {
    if (below + (long long)hist[d] > rank) break;
    below += hist[d];
  }
  rank -= below;
  return d;
}

// ---- job statistics by job size (gs_jclass, include/gsched.h)
static_assert(sizeof(gs_jclass) == 160, "gs_jclass is 160 bytes");

// A jobdist setting, passed to the kernel by value (1 KB of parameters; the edges are staged in shared memory).
struct GsJdCfg {
  int nclasses, nedges;
  int bounds[GS_JOBDIST_MAX_CLASSES - 1];
  int edges[GS_JOBDIST_MAX_EDGES];
};

// Class of a job with `gpus` GPUs: the number of the nb = C - 1 increasing bounds that are <= gpus.
GS_SUM_HD int gs_jd_class(const int *bounds, int nb, int gpus) {
  int c = 0;
  while (c < nb && bounds[c] <= gpus) ++c;
  return c;
}

// CDF bin of a value: #{i : edges[i] < v} over E increasing edges (binary search).
GS_SUM_HD int gs_jd_bin(const int *edges, int E, int v) {
  int lo = 0, hi = E;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (edges[mid] < v) lo = mid + 1; else hi = mid; }
  return lo;
}

// A jobdist setting from the C ABI's arrays, or false (the message in *why) when it is not valid.
static inline bool gs_jd_make_cfg(int32_t nclasses, const int32_t *bounds, int32_t nedges, const int32_t *edges, GsJdCfg &cfg, const char **why) {
  *why = "nclasses must be in 0..8 and nedges in 0..255";
  if (nclasses < 0 || nclasses > GS_JOBDIST_MAX_CLASSES || nedges < 0 || nedges > GS_JOBDIST_MAX_EDGES) return false;
  cfg = GsJdCfg{};
  if (nclasses == 0) return true;
  *why = "a NULL array with a positive count";
  if ((nclasses > 1 && !bounds) || (nedges > 0 && !edges)) return false;
  *why = "the class bounds must be >= 1 and strictly increasing";
  for (int i = 0; i < nclasses - 1; ++i)
    if (bounds[i] < 1 || (i > 0 && bounds[i] <= bounds[i - 1])) return false;
  *why = "the edges must be strictly increasing";
  for (int i = 1; i < nedges; ++i)
    if (edges[i] <= edges[i - 1]) return false;
  cfg.nclasses = nclasses; cfg.nedges = nedges;
  for (int i = 0; i < nclasses - 1; ++i) cfg.bounds[i] = bounds[i];
  for (int i = 0; i < nedges; ++i) cfg.edges[i] = edges[i];
  return true;
}

// v * v (< 2^62 for any int32 v) added to a 128-bit sum of squares.
GS_SUM_HD void gs_jd_add_sq(uint64_t &lo, uint64_t &hi, int v) { gs_sum_add128(lo, hi, (gs_i128)((long long)v * v)); }

static_assert(sizeof(gs_jpair) == 288, "gs_jpair is 288 bytes");

// ---- job statistics by a chosen key, with bounded slowdown (gs_sdclass, include/gsched.h)
static_assert(sizeof(gs_sdclass) == 232 && sizeof(gs_sdclass) % 8 == 0, "gs_sdclass is 232 bytes, a multiple of 8");
#define GS_SD_MAX 0x7fffffffll       // the saturated slowdown, 2^31 - 1 (units of 1/1024)

// A slowdown setting, passed to the kernel by value (2.1 KB of parameters; the edges are staged in shared memory).
struct GsSdCfg {
  int key, nclasses, nedges, nsd;
  long long bounds[GS_JOBDIST_MAX_CLASSES - 1];
  long long tau;
  int edges[GS_JOBDIST_MAX_EDGES];
  int sd_edges[GS_SLOWDOWN_MAX_EDGES];
};

// Key of a job (GS_JKEY_*): gpus, jct or gpus * jct.
GS_SUM_HD long long gs_sd_key(int key, int gpus, int jct) {
  return key == GS_JKEY_GPUS ? (long long)gpus : key == GS_JKEY_LENGTH ? (long long)jct : (long long)gpus * jct;
}

// Class of a key: the number of the nb = C - 1 increasing bounds that are <= key.
GS_SUM_HD int gs_sd_class(const long long *bounds, int nb, long long key) {
  int c = 0;
  while (c < nb && bounds[c] <= key) ++c;
  return c;
}

// Bounded slowdown in units of 1/1024: min(2^31 - 1, max(1024, floor(1024 * turn / max(jct, tau)))), in 64-bit
// integers.  turn = end - arrive >= 0 and tau >= 1, so the quotient is a floor and the divisor is >= 1; 1024 * turn
// < 2^41.
GS_SUM_HD int gs_sd_value(int turn, int jct, long long tau) {
  const long long den = (long long)jct > tau ? (long long)jct : tau;
  const long long q = 1024ll * turn / den;
  return q < 1024 ? 1024 : q > GS_SD_MAX ? (int)GS_SD_MAX : (int)q;
}

// A slowdown setting from the C ABI's struct, or false (the message in *why) when it is not valid.  cfg == NULL is off.
static inline bool gs_sd_make_cfg(const gs_slowdown_cfg *in, GsSdCfg &cfg, const char **why) {
  cfg = GsSdCfg{};
  if (!in || in->nclasses == 0) return true;
  *why = "key must be GS_JKEY_GPUS, GS_JKEY_LENGTH or GS_JKEY_GPU_TIME";
  if (in->key != GS_JKEY_GPUS && in->key != GS_JKEY_LENGTH && in->key != GS_JKEY_GPU_TIME) return false;
  *why = "nclasses must be in 0..8, nedges and nsd_edges in 0..255";
  if (in->nclasses < 0 || in->nclasses > GS_JOBDIST_MAX_CLASSES || in->nedges < 0 || in->nedges > GS_JOBDIST_MAX_EDGES ||
      in->nsd_edges < 0 || in->nsd_edges > GS_SLOWDOWN_MAX_EDGES) return false;
  *why = "tau must be >= 1";
  if (in->tau < 1) return false;
  *why = "a NULL array with a positive count";
  if ((in->nedges > 0 && !in->edges) || (in->nsd_edges > 0 && !in->sd_edges)) return false;
  *why = "the class bounds must be >= 1 and strictly increasing";
  for (int i = 0; i < in->nclasses - 1; ++i)
    if (in->bounds[i] < 1 || (i > 0 && in->bounds[i] <= in->bounds[i - 1])) return false;
  *why = "the edges must be strictly increasing";
  for (int i = 1; i < in->nedges; ++i)
    if (in->edges[i] <= in->edges[i - 1]) return false;
  *why = "the sd edges must be strictly increasing";
  for (int i = 1; i < in->nsd_edges; ++i)
    if (in->sd_edges[i] <= in->sd_edges[i - 1]) return false;
  cfg.key = in->key; cfg.nclasses = in->nclasses; cfg.nedges = in->nedges; cfg.nsd = in->nsd_edges; cfg.tau = in->tau;
  for (int i = 0; i < in->nclasses - 1; ++i) cfg.bounds[i] = in->bounds[i];
  for (int i = 0; i < in->nedges; ++i) cfg.edges[i] = in->edges[i];
  for (int i = 0; i < in->nsd_edges; ++i) cfg.sd_edges[i] = in->sd_edges[i];
  return true;
}

// uint32 counts per (replica, class): wait, turnaround and jct E + 1 each, then sd Esd + 1.
GS_SUM_HD long long gs_sd_row_len(const GsSdCfg &cfg) { return 3ll * (cfg.nedges + 1) + cfg.nsd + 1; }

// ---- job statistics by arrival time (gs_abin, include/gsched.h)
static_assert(sizeof(gs_abin) == 240 && sizeof(gs_abin) % 8 == 0, "gs_abin is 240 bytes, a multiple of 8");
#define GS_ARR_ROWS 7                // scratch rows per job: wait, turnaround, jct, sd, preempt, gpus, arrival tick
#define GS_ARR_CUT 256               // a bin of at most this many finished jobs is finished by one warp, larger ones by the block

// An arrivals setting; nbins = 0: off.  A job's bin is gs_tl_bin(arrival tick, width, nbins), the timeline's rule.
struct GsArrCfg {
  long long width, tau;
  int nbins;
};

// An arrivals setting from the C ABI's arguments, or false (the message in *why) when it is not valid.
static inline bool gs_arr_make_cfg(long long width, int nbins, long long tau, GsArrCfg &cfg, const char **why) {
  cfg = GsArrCfg{};
  *why = "nbins must be in 0..1024";
  if (nbins < 0 || nbins > GS_ARRIVALS_MAX_BINS) return false;
  if (nbins == 0) return true;
  *why = "bin_width must be >= 1";
  if (width < 1) return false;
  *why = "tau must be >= 1";
  if (tau < 1) return false;
  cfg.width = width; cfg.tau = tau; cfg.nbins = nbins;
  return true;
}

// ---- time-weighted occupancy (gs_occ, include/gsched.h)
static_assert(sizeof(gs_occ) == 72, "gs_occ is 72 bytes");
#define GS_OCC_MAX_GPUS 65535
#define GS_OCC_SMEM_COUNTERS 3072   // H_all and H_wait in shared memory when 2 * (G + 1) counters fit (24 KB)

// The queue edges, passed to the kernel by value (the edges are staged in shared memory).
struct GsOccCfg {
  int nedges;
  int edges[GS_OCC_MAX_EDGES];
};

// The last row of an unfinished window of an event-driven run, weighed once its successor (or the end) is seen.
struct GsOccCarry {
  long long delta;
  int busy, running, queued, valid;
};

// Partial sums of a fold: GS_OCC_NSUM sums, then two maxima (gs_sum_block_vec's layout).
enum { GS_OCC_ROWS, GS_OCC_TICKS, GS_OCC_BUSY, GS_OCC_RUNNING, GS_OCC_QUEUED, GS_OCC_WAIT, GS_OCC_IDLE, GS_OCC_NSUM,
       GS_OCC_RMAX = GS_OCC_NSUM, GS_OCC_QMAX, GS_OCC_N };

// A queue edge setting from the C ABI's array, or false (the message in *why) when it is not valid.
static inline bool gs_occ_make_cfg(int32_t nedges, const int32_t *edges, GsOccCfg &cfg, const char **why) {
  *why = "nedges must be in 0..255";
  if (nedges < 0 || nedges > GS_OCC_MAX_EDGES) return false;
  *why = "a NULL array with a positive count";
  if (nedges > 0 && !edges) return false;
  *why = "the edges must be >= 0 and strictly increasing";
  for (int i = 0; i < nedges; ++i)
    if (edges[i] < 0 || (i > 0 && edges[i] <= edges[i - 1])) return false;
  cfg = GsOccCfg{};
  cfg.nedges = nedges;
  for (int i = 0; i < nedges; ++i) cfg.edges[i] = edges[i];
  return true;
}

GS_SUM_HD void gs_occ_zero(long long (&v)[GS_OCC_N]) {
  for (int e = 0; e < GS_OCC_N; ++e) v[e] = 0;
}

// `nrows` rows that hold (busy, running, queued) for w ticks in all, into the partial sums.
GS_SUM_HD void gs_occ_part(long long (&v)[GS_OCC_N], int G, int busy, int running, int queued, long long nrows, long long w) {
  v[GS_OCC_ROWS] += nrows;
  if (w <= 0) return;
  v[GS_OCC_TICKS] += w;
  v[GS_OCC_BUSY] += w * busy; v[GS_OCC_RUNNING] += w * running; v[GS_OCC_QUEUED] += w * queued;
  if (queued > 0) { v[GS_OCC_WAIT] += w; v[GS_OCC_IDLE] += w * (G - busy); }
  v[GS_OCC_RMAX] = running > v[GS_OCC_RMAX] ? running : v[GS_OCC_RMAX];
  v[GS_OCC_QMAX] = queued > v[GS_OCC_QMAX] ? queued : v[GS_OCC_QMAX];
}

GS_SUM_HD void gs_occ_add(gs_occ &o, const long long (&v)[GS_OCC_N]) {
  o.rows += v[GS_OCC_ROWS]; o.ticks += v[GS_OCC_TICKS];
  o.busy_sum += v[GS_OCC_BUSY]; o.running_sum += v[GS_OCC_RUNNING]; o.queued_sum += v[GS_OCC_QUEUED];
  o.wait_ticks += v[GS_OCC_WAIT]; o.idle_wait_sum += v[GS_OCC_IDLE];
  o.running_max = (int)(v[GS_OCC_RMAX] > o.running_max ? v[GS_OCC_RMAX] : o.running_max);
  o.queued_max = (int)(v[GS_OCC_QMAX] > o.queued_max ? v[GS_OCC_QMAX] : o.queued_max);
}

// Histograms of one replica: H_all and H_wait (G + 1 counters each) and the queue's E + 1 counters.
struct GsOccHist {
  unsigned long long *all, *wait, *q;
};

// One stretch of w ticks into the partial sums and, serially, the histograms.
GS_SUM_HD void gs_occ_stretch(long long (&v)[GS_OCC_N], const GsOccHist &H, const GsOccCfg &cfg, int G, int busy, int running, int queued,
                              long long nrows, long long w) {
  gs_occ_part(v, G, busy, running, queued, nrows, w);
  if (w <= 0) return;
  H.all[busy] += (unsigned long long)w;
  if (queued > 0) H.wait[busy] += (unsigned long long)w;
  H.q[gs_jd_bin(cfg.edges, cfg.nedges, queued)] += (unsigned long long)w;
}

// Host and device serial fold, `gs_occ_serial`: rows lo .. hi - 1 (rows[i - base]) into one replica's record and
// histograms.  per_tick (horus): every row weighs 1.  Otherwise (event-driven policies) a row weighs the step of
// `delta` to its successor, clamped at 0: the carry holds the last row seen, which the next row -- of this call or of
// a later one -- weighs; at the end of a finished run (done) it weighs 1 and the carry is cleared.
GS_SUM_HD void gs_occ_serial(gs_occ &o, GsOccCarry &c, const GsOccHist &H, const GsOccCfg &cfg, const gs_tick_row *rows, long long base,
                             long long lo, long long hi, int done, int per_tick) {
  long long v[GS_OCC_N];
  gs_occ_zero(v);
  const int G = o.total_gpus;
  for (long long i = lo; i < hi; ++i) {
    const gs_tick_row &r = rows[i - base];
    if (per_tick) { gs_occ_stretch(v, H, cfg, G, r.busy_gpus, r.running, r.queued, 1, 1); continue; }
    if (c.valid) gs_occ_stretch(v, H, cfg, G, c.busy, c.running, c.queued, 1, r.now > c.delta ? r.now - c.delta : 0);
    c.delta = r.now; c.busy = r.busy_gpus; c.running = r.running; c.queued = r.queued; c.valid = 1;
  }
  if (!per_tick && c.valid && done) { gs_occ_stretch(v, H, cfg, G, c.busy, c.running, c.queued, 1, 1); c.valid = 0; }
  gs_occ_add(o, v);
}

// fifo: the records of a window, rows with `delta` <= wm skipped (gs_sum_fold_records' rows), every row one tick.
GS_SUM_HD void gs_occ_records_serial(gs_occ &o, const GsOccHist &H, const GsOccCfg &cfg, const gs_evrow *ev, int nev, long long ticks,
                                     long long wm) {
  long long v[GS_OCC_N];
  gs_occ_zero(v);
  for (int k = 0; k < nev; ++k) {
    const long long t_last = k + 1 < nev ? (long long)ev[k + 1].now - 1 : ticks;
    const long long v_lo = ev[k].now > wm + 1 ? (long long)ev[k].now : wm + 1;
    if (t_last >= v_lo) gs_occ_stretch(v, H, cfg, o.total_gpus, ev[k].busy_gpus, ev[k].running, ev[k].queued, t_last - v_lo + 1, t_last - v_lo + 1);
  }
  gs_occ_add(o, v);
}

// ---- interference statistics of the utilisation-aware engine (gs_ifclass, include/gsched_horus.h)
static_assert(sizeof(gs_ifclass) == 440 && sizeof(gs_ifclass) % 8 == 0, "gs_ifclass is 440 bytes, a multiple of 8");
#define GS_IF_MAX 0x7fffffffll       // the saturated fixed-point duration, 2^31 - 1 (units of 2^-10 tick)
#define GS_IF_ROWS 8                 // scratch rows per job: wait, turnaround, jct, a, o, e, gpus, preempt

// What the engine's record says of a finished job: its GPUs, Job.duration and Job.get_duration().
struct GsIfDur { int gpus; double original, actual; };
// Its fixed-point values: a = fp(actual), o = fp(original), e = fp(actual - original) when degraded (else 0).
struct GsIfVal { int a, o, e, degraded, clamped; };

// fp(x) = min(2^31 - 1, max(0, round-half-even(1024 * x))); clamped |= 1 when the bound applies or x is NaN.
GS_SUM_HD int gs_if_fp(double x, int &clamped) {
#ifdef __CUDA_ARCH__
  const long long r = __double2ll_rn(__dmul_rn(1024.0, x));            // NaN gives -2^63
#else
  const double d = nearbyint(1024.0 * x);                              // the default rounding mode: to nearest, ties to even
  const long long r = d != d || d < -9.0e18 ? (long long)(-0x7fffffffffffffffll - 1) : d > 9.0e18 ? 0x7fffffffffffffffll : (long long)d;
#endif
  if (r < 0) { clamped = 1; return 0; }
  if (r > GS_IF_MAX) { clamped = 1; return (int)GS_IF_MAX; }
  return (int)r;
}

GS_SUM_HD GsIfVal gs_if_value(double original, double actual) {
  GsIfVal v;
  v.clamped = 0;
  v.degraded = actual > original;
  v.a = gs_if_fp(actual, v.clamped);
  v.o = gs_if_fp(original, v.clamped);
#ifdef __CUDA_ARCH__
  v.e = v.degraded ? gs_if_fp(__dsub_rn(actual, original), v.clamped) : 0;
#else
  v.e = v.degraded ? gs_if_fp(actual - original, v.clamped) : 0;
#endif
  return v;
}

#ifndef __CUDACC__
#include <algorithm>
#include <vector>
// Host forms of the job part (the host-emulation build of gs_horus.cu, CPU tests): the same sums, and the same radix
// select run serially, one target at a time.
static inline void gs_sum_select_serial(const int *v, long long k, int out[5]) {
  if (k == 0) { for (int t = 0; t < 5; ++t) out[t] = 0; return; }
  int mn = v[0], mx = v[0];
  for (long long i = 1; i < k; ++i) { mn = v[i] < mn ? v[i] : mn; mx = v[i] > mx ? v[i] : mx; }
  const int passes = gs_sum_passes((unsigned long long)((long long)mx - mn));
  unsigned hist[GS_SUM_BINS];
  for (int t = 0; t < 5; ++t) {
    long long rank = gs_sum_rank(gs_sum_permille(t), k);
    unsigned long long prefix = 0;
    for (int p = 0; p < passes; ++p) {
      const int shift = (passes - 1 - p) * 9;
      for (int b = 0; b < GS_SUM_BINS; ++b) hist[b] = 0;
      for (long long i = 0; i < k; ++i) {
        const unsigned long long u = (unsigned long long)((long long)v[i] - mn);
        if ((u >> (shift + 9)) == prefix) hist[(u >> shift) & (GS_SUM_BINS - 1)] += 1;
      }
      prefix = (prefix << 9) | gs_sum_pick(hist, rank);
    }
    out[t] = (int)((long long)mn + (long long)prefix);
  }
}

static inline void gs_sum_jobs_serial(const GsSumJob *jobs, long long k, gs_summary &s) {
  s.finished = k;
  s.wait_sum = s.turnaround_sum = s.jct_sum = s.preempt_sum = s.gpu_ticks_sum = 0;
  int *vals = new int[(size_t)(3 * (k > 0 ? k : 1))];
  for (long long i = 0; i < k; ++i) {
    const GsSumJob &v = jobs[i];
    s.wait_sum += v.wait; s.turnaround_sum += v.turn; s.jct_sum += v.jct; s.preempt_sum += v.preempt;
    s.gpu_ticks_sum += (long long)v.gpus * v.jct;
    vals[i] = v.wait; vals[k + i] = v.turn; vals[2 * k + i] = v.jct;
  }
  gs_sum_select_serial(vals, k, s.wait_q);
  gs_sum_select_serial(vals + k, k, s.turnaround_q);
  gs_sum_select_serial(vals + 2 * k, k, s.jct_q);
  delete[] vals;
}

// jobdist of k finished jobs: classes[0 .. C) and hist[C][3][E + 1] (overwritten).  The kernel's steps, serially:
// count per class, write the values into per-class segments, fold each segment, select within it.
static inline void gs_jd_jobs_serial(const GsSumJob *jobs, long long k, const GsJdCfg &cfg, gs_jclass *classes, uint32_t *hist) {
  const int C = cfg.nclasses, nb = cfg.nedges + 1;
  long long off[GS_JOBDIST_MAX_CLASSES + 1] = {0};
  for (int c = 0; c < C; ++c) classes[c] = gs_jclass{};
  for (long long i = 0; i < (long long)C * 3 * nb; ++i) hist[i] = 0;
  for (long long i = 0; i < k; ++i) off[gs_jd_class(cfg.bounds, C - 1, jobs[i].gpus) + 1] += 1;
  for (int c = 0; c < C; ++c) off[c + 1] += off[c];
  const long long pitch = k > 0 ? k : 1;
  int *vals = new int[(size_t)(3 * pitch)];
  long long cur[GS_JOBDIST_MAX_CLASSES];
  for (int c = 0; c < C; ++c) cur[c] = off[c];
  for (long long i = 0; i < k; ++i) {
    const GsSumJob &v = jobs[i];
    const int c = gs_jd_class(cfg.bounds, C - 1, v.gpus);
    gs_jclass &J = classes[c];
    J.preempt_sum += v.preempt; J.gpu_ticks_sum += (long long)v.gpus * v.jct;
    const long long pos = cur[c]++;
    vals[pos] = v.wait; vals[pitch + pos] = v.turn; vals[2 * pitch + pos] = v.jct;
  }
  for (int c = 0; c < C; ++c) {
    gs_jclass &J = classes[c];
    const long long kc = off[c + 1] - off[c];
    const int *seg = vals + off[c];
    J.jobs = kc;
    uint32_t *hc = hist + (size_t)c * 3 * nb;
    for (long long i = 0; i < kc; ++i) {
      const int w = seg[i], t = seg[pitch + i], j = seg[2 * pitch + i];
      J.wait_sum += w; J.turnaround_sum += t; J.jct_sum += j;
      gs_jd_add_sq(J.wait_sq_lo, J.wait_sq_hi, w);
      gs_jd_add_sq(J.turnaround_sq_lo, J.turnaround_sq_hi, t);
      gs_jd_add_sq(J.jct_sq_lo, J.jct_sq_hi, j);
      hc[gs_jd_bin(cfg.edges, cfg.nedges, w)] += 1;
      hc[nb + gs_jd_bin(cfg.edges, cfg.nedges, t)] += 1;
      hc[2 * nb + gs_jd_bin(cfg.edges, cfg.nedges, j)] += 1;
    }
    gs_sum_select_serial(seg, kc, J.wait_q);
    gs_sum_select_serial(seg + pitch, kc, J.turnaround_q);
    gs_sum_select_serial(seg + 2 * pitch, kc, J.jct_q);
  }
  delete[] vals;
}

// Paired comparison of one pair (gs_jpair): ja / jb the job values of runs a and b by trace index j < n (read only for
// jobs finished in that run, except `gpus`, which both share), fin_a / fin_b their finish orders.  out[0 .. C) and
// hist[C][3][E + 1] are overwritten.  The kernel's steps, serially: membership words, per-class counts, differences
// scattered into per-class segments, then per class the fold and the two selects (ascending, then negated).  The
// traces' equality is the caller's to check.
static inline void gs_cmp_pair_serial(const GsSumJob *ja, const GsSumJob *jb, long long n, const int *fin_a, long long ka,
                                      const int *fin_b, long long kb, const GsJdCfg &cfg, gs_jpair *out, uint32_t *hist) {
  const int C = cfg.nclasses, nb = cfg.nedges + 1;
  const long long pitch = n > 0 ? n : 1;
  std::vector<int> mem((size_t)pitch, 0), vals((size_t)(3 * pitch));
  for (long long i = 0; i < ka; ++i) mem[(size_t)fin_a[i]] = 1;
  for (long long i = 0; i < kb; ++i) mem[(size_t)fin_b[i]] |= 2;
  long long cnt[3][GS_JOBDIST_MAX_CLASSES] = {};          // jobs, only_a, only_b
  for (long long j = 0; j < n; ++j) {
    const int w = mem[(size_t)j];
    if (w == 0) continue;
    const int c = gs_jd_class(cfg.bounds, C - 1, ja[j].gpus);
    cnt[w == 3 ? 0 : w == 1 ? 1 : 2][c] += 1;
  }
  long long cur[GS_JOBDIST_MAX_CLASSES], off = 0;
  for (int c = 0; c < C; ++c) { cur[c] = off; off += cnt[0][c]; }
  for (long long j = 0; j < n; ++j) {
    if (mem[(size_t)j] != 3) continue;
    const long long pos = cur[gs_jd_class(cfg.bounds, C - 1, ja[j].gpus)]++;
    vals[(size_t)pos] = jb[j].wait - ja[j].wait;
    vals[(size_t)(pitch + pos)] = jb[j].turn - ja[j].turn;
    vals[(size_t)(2 * pitch + pos)] = jb[j].jct - ja[j].jct;
  }
  for (long long i = 0; i < (long long)C * 3 * nb; ++i) hist[i] = 0;
  off = 0;
  for (int c = 0; c < C; ++c) {
    gs_jpair &P = out[c];
    P = gs_jpair{};
    const long long kc = cnt[0][c];
    P.jobs = kc; P.only_a = cnt[1][c]; P.only_b = cnt[2][c];
    uint32_t *hc = hist + (size_t)c * 3 * nb;
    for (int m = 0; m < 3; ++m) {
      int *seg = vals.data() + m * pitch + off;
      for (long long i = 0; i < kc; ++i) {
        const int d = seg[i];
        P.lt[m] += d < 0; P.eq[m] += d == 0; P.gt[m] += d > 0;
        P.d_sum[m] += d;
        gs_jd_add_sq(P.d_sq_lo[m], P.d_sq_hi[m], d);
        hc[m * nb + gs_jd_bin(cfg.edges, cfg.nedges, d)] += 1;
      }
      gs_sum_select_serial(seg, kc, P.q_hi[m]);
      for (long long i = 0; i < kc; ++i) seg[i] = -seg[i];
      int q[5];
      gs_sum_select_serial(seg, kc, q);
      for (int t = 0; t < 5; ++t) P.q_lo[m][t] = -q[t];
    }
    off += kc;
  }
}

// Slowdown statistics of k finished jobs: out[0 .. C) and hist[C][3 * (E + 1) + Esd + 1] (overwritten).  The kernel's
// steps, serially: count per class (and sum the keys), write wait / turnaround / jct / sd into per-class segments, fold
// each segment, select within it.
static inline void gs_sd_serial(const GsSumJob *jobs, long long k, const GsSdCfg &cfg, gs_sdclass *out, uint32_t *hist) {
  const int C = cfg.nclasses, nb = cfg.nedges + 1;
  const long long row = gs_sd_row_len(cfg);
  long long off[GS_JOBDIST_MAX_CLASSES + 1] = {0};
  for (int c = 0; c < C; ++c) out[c] = gs_sdclass{};
  for (long long i = 0; i < (long long)C * row; ++i) hist[i] = 0;
  std::vector<int> cls((size_t)(k > 0 ? k : 1));
  for (long long i = 0; i < k; ++i) {
    const GsSumJob &v = jobs[i];
    const long long key = gs_sd_key(cfg.key, v.gpus, v.jct);
    const int c = gs_sd_class(cfg.bounds, C - 1, key);
    cls[(size_t)i] = c;
    off[c + 1] += 1;
    gs_sdclass &S = out[c];
    S.jc.preempt_sum += v.preempt; S.jc.gpu_ticks_sum += (long long)v.gpus * v.jct;
    gs_sum_add128(S.key_sum_lo, S.key_sum_hi, (gs_i128)key);
  }
  for (int c = 0; c < C; ++c) off[c + 1] += off[c];
  const long long pitch = k > 0 ? k : 1;
  std::vector<int> vals((size_t)(4 * pitch));
  long long cur[GS_JOBDIST_MAX_CLASSES];
  for (int c = 0; c < C; ++c) cur[c] = off[c];
  for (long long i = 0; i < k; ++i) {
    const GsSumJob &v = jobs[i];
    const long long pos = cur[cls[(size_t)i]]++;
    vals[(size_t)pos] = v.wait; vals[(size_t)(pitch + pos)] = v.turn; vals[(size_t)(2 * pitch + pos)] = v.jct;
    vals[(size_t)(3 * pitch + pos)] = gs_sd_value(v.turn, v.jct, cfg.tau);
  }
  for (int c = 0; c < C; ++c) {
    gs_sdclass &S = out[c];
    gs_jclass &J = S.jc;
    const long long kc = off[c + 1] - off[c];
    const int *seg = vals.data() + off[c];
    J.jobs = kc;
    uint32_t *hc = hist + (size_t)c * row;
    for (long long i = 0; i < kc; ++i) {
      const int w = seg[i], t = seg[pitch + i], j = seg[2 * pitch + i], sd = seg[3 * pitch + i];
      J.wait_sum += w; J.turnaround_sum += t; J.jct_sum += j;
      gs_jd_add_sq(J.wait_sq_lo, J.wait_sq_hi, w);
      gs_jd_add_sq(J.turnaround_sq_lo, J.turnaround_sq_hi, t);
      gs_jd_add_sq(J.jct_sq_lo, J.jct_sq_hi, j);
      S.sd_sum += sd;
      gs_jd_add_sq(S.sd_sq_lo, S.sd_sq_hi, sd);
      S.sd_min = i == 0 || sd < S.sd_min ? sd : S.sd_min;
      S.sd_clamped += sd == (int)GS_SD_MAX;
      hc[gs_jd_bin(cfg.edges, cfg.nedges, w)] += 1;
      hc[nb + gs_jd_bin(cfg.edges, cfg.nedges, t)] += 1;
      hc[2 * nb + gs_jd_bin(cfg.edges, cfg.nedges, j)] += 1;
      hc[3 * nb + gs_jd_bin(cfg.sd_edges, cfg.nsd, sd)] += 1;
    }
    gs_sum_select_serial(seg, kc, J.wait_q);
    gs_sum_select_serial(seg + pitch, kc, J.turnaround_q);
    gs_sum_select_serial(seg + 2 * pitch, kc, J.jct_q);
    gs_sum_select_serial(seg + 3 * pitch, kc, S.sd_q);
  }
}

// Arrival-bin statistics of k finished jobs (jobs[i] arrived at tick arrive[i], in finish order) of a trace whose n
// jobs arrived at trace_arrive[0 .. n): out[0 .. B) (overwritten).  Each bin's finished jobs are one class of
// gs_sd_serial (no edges), whose key sum is then replaced by the sum of their arrival ticks.
static inline void gs_arr_serial(const GsSumJob *jobs, const int *arrive, long long k, const int *trace_arrive, long long n,
                                 const GsArrCfg &cfg, gs_abin *out) {
  const int B = cfg.nbins;
  GsSdCfg one{};
  one.key = GS_JKEY_GPUS; one.nclasses = 1; one.tau = cfg.tau;
  std::vector<std::vector<GsSumJob>> bins((size_t)B);
  std::vector<long long> key((size_t)B, 0);
  for (int b = 0; b < B; ++b) out[b] = gs_abin{};
  for (long long j = 0; j < n; ++j) out[gs_tl_bin(trace_arrive[j], cfg.width, B)].arrived += 1;
  for (long long i = 0; i < k; ++i) {
    const int b = gs_tl_bin(arrive[i], cfg.width, B);
    bins[(size_t)b].push_back(jobs[i]);
    key[(size_t)b] += arrive[i];
  }
  uint32_t hist[4];
  for (int b = 0; b < B; ++b) {
    gs_sd_serial(bins[(size_t)b].data(), (long long)bins[(size_t)b].size(), one, &out[b].s, hist);
    out[b].s.key_sum_lo = out[b].s.key_sum_hi = 0;
    gs_sum_add128(out[b].s.key_sum_lo, out[b].s.key_sum_hi, (gs_i128)key[(size_t)b]);
  }
}
// Interference statistics of k finished jobs (jobs[i] and durs[i] of the same job): out[0 .. C) (overwritten).  Each
// group (class, degraded or clean) takes gs_jd_jobs_serial's record as a class of its own; the rest are plain sums
// and order statistics, the middle ones by std::nth_element.
static inline void gs_if_serial(const GsSumJob *jobs, const GsIfDur *durs, long long k, const GsJdCfg &cfg, gs_ifclass *out) {
  const int C = cfg.nclasses;
  GsJdCfg one{};
  one.nclasses = 1;
  std::vector<GsSumJob> grp[2 * GS_JOBDIST_MAX_CLASSES];
  std::vector<int> av[GS_JOBDIST_MAX_CLASSES], djct[GS_JOBDIST_MAX_CLASSES];
  for (int c = 0; c < C; ++c) out[c] = gs_ifclass{};
  for (long long i = 0; i < k; ++i) {
    const GsSumJob &v = jobs[i];
    const int c = gs_jd_class(cfg.bounds, C - 1, durs[i].gpus);
    const GsIfVal x = gs_if_value(durs[i].original, durs[i].actual);
    gs_ifclass &F = out[c];
    grp[2 * c + x.degraded].push_back(v);
    av[c].push_back(x.a);
    if (x.degraded) {
      djct[c].push_back(v.jct);
      F.excess_sum += x.e;
      F.excess_max = x.e > F.excess_max ? x.e : F.excess_max;
      gs_sum_add128(F.lost_gpu_time_lo, F.lost_gpu_time_hi, (gs_i128)((long long)v.gpus * x.e));
    }
    F.actual_sum += x.a;
    gs_jd_add_sq(F.actual_sq_lo, F.actual_sq_hi, x.a);
    F.original_sum += x.o;
    F.preempted_jobs += v.preempt > 1;
    F.preempt_max = v.preempt > F.preempt_max ? v.preempt : F.preempt_max;
    F.clamped += x.clamped;
  }
  auto mid = [](std::vector<int> v, int out2[2]) {
    const long long n = (long long)v.size();
    if (n == 0) { out2[0] = out2[1] = 0; return; }
    std::nth_element(v.begin(), v.begin() + (n - 1) / 2, v.end());
    out2[0] = v[(size_t)((n - 1) / 2)];
    std::nth_element(v.begin(), v.begin() + n / 2, v.end());
    out2[1] = v[(size_t)(n / 2)];
  };
  uint32_t hist[3];
  for (int c = 0; c < C; ++c) {
    gs_ifclass &F = out[c];
    gs_jd_jobs_serial(grp[2 * c].data(), (long long)grp[2 * c].size(), one, &F.clean, hist);
    gs_jd_jobs_serial(grp[2 * c + 1].data(), (long long)grp[2 * c + 1].size(), one, &F.degraded, hist);
    gs_sum_select_serial(av[c].data(), (long long)av[c].size(), F.actual_q);
    mid(av[c], F.actual_mid);
    mid(djct[c], F.degraded_jct_mid);
  }
}
#endif

#ifdef __CUDACC__
namespace {

__device__ __forceinline__ GsSumPart gs_sum_shfl_down(const GsSumPart &p, int o) {
  GsSumPart q;
  q.rows = __shfl_down_sync(0xffffffffu, p.rows, o); q.busy = __shfl_down_sync(0xffffffffu, p.busy, o);
  q.running = __shfl_down_sync(0xffffffffu, p.running, o); q.queued = __shfl_down_sync(0xffffffffu, p.queued, o);
  q.pending_rows = __shfl_down_sync(0xffffffffu, p.pending_rows, o);
  q.busy_max = __shfl_down_sync(0xffffffffu, p.busy_max, o); q.running_max = __shfl_down_sync(0xffffffffu, p.running_max, o);
  q.queued_max = __shfl_down_sync(0xffffffffu, p.queued_max, o); q.pend_max = __shfl_down_sync(0xffffffffu, p.pend_max, o);
  const unsigned long long plo = __shfl_down_sync(0xffffffffu, (unsigned long long)p.pend, o);
  const unsigned long long phi = __shfl_down_sync(0xffffffffu, (unsigned long long)((gs_u128)p.pend >> 64), o);
  const unsigned long long mlo = __shfl_down_sync(0xffffffffu, (unsigned long long)p.mem, o);
  const unsigned long long mhi = __shfl_down_sync(0xffffffffu, (unsigned long long)((gs_u128)p.mem >> 64), o);
  q.pend = (gs_i128)(((gs_u128)phi << 64) | plo); q.mem = (gs_i128)(((gs_u128)mhi << 64) | mlo);
  q.avg = __shfl_down_sync(0xffffffffu, p.avg, o); q.util = __shfl_down_sync(0xffffffffu, p.util, o);
  return q;
}

// Block sum of the threads' folds: thread 0 returns with the total (warps merged in a fixed order: deterministic).
__device__ void gs_sum_block_reduce(GsSumPart &p) {
  __shared__ GsSumPart warp_part[GS_SUM_THREADS / 32];
  for (int o = 16; o > 0; o >>= 1) { const GsSumPart q = gs_sum_shfl_down(p, o); gs_sum_merge(p, q); }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();                                          // warp_part may still be read by an earlier reduction
  if (lane == 0) warp_part[warp] = p;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) gs_sum_merge(p, warp_part[w]);
}

// fifo: fold the window's records (block-cooperative: every thread calls it).  Rows already folded (`delta` <= wm) are
// skipped.  The gs_qrow of a record with a queue is found by counting such records (one gs_qrow each, in order);
// a binary search by `now` checks and, should the streams not line up, finds it.
__device__ void gs_sum_fold_records(GsSumPart &p, const gs_evrow *ev, int nev, const gs_qrow *qr, int nq, long long ticks,
                                    long long wm) {
  __shared__ int warp_cnt[GS_SUM_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  int qbase = 0;
  for (int t0 = 0; t0 < nev; t0 += blockDim.x) {
    const int k = t0 + threadIdx.x;
    const bool in = k < nev;
    gs_evrow e;
    if (in) e = ev[k];
    const bool hasq = in && e.queued > 0;
    const unsigned bal = __ballot_sync(0xffffffffu, hasq);
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    __syncthreads();
    int off = __popc(bal & ((1u << lane) - 1u)), total = 0;
    for (int w = 0; w < nwarps; ++w) { const int c = warp_cnt[w]; off += w < warp ? c : 0; total += c; }
    __syncthreads();
    if (in) {
      const long long t_first = e.now;
      const long long t_last = k + 1 < nev ? (long long)ev[k + 1].now - 1 : ticks;
      const long long v_lo = t_first > wm + 1 ? t_first : wm + 1;
      if (t_last >= v_lo) {
        long long arrive_sum = 0; int oldest = 0;
        if (hasq) {
          int qi = qbase + off;
          if (qi >= nq || qr[qi].now != e.now) {
            int lo = 0, hi = nq - 1;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (qr[mid].now < e.now) lo = mid + 1; else hi = mid; }
            qi = lo;
          }
          const gs_qrow b = qr[qi];
          arrive_sum = b.arrive_sum; oldest = b.oldest_arrive;
        }
        gs_sum_record(p, e, arrive_sum, oldest, v_lo, t_last);
      }
    }
    qbase += total;
  }
}

// ---- timeline bin kernels' block functions.  Every bin is folded by ONE warp (bins b = warp, warp + 8, ...): lanes
// stride over the bin's rows / records, a fixed shuffle tree merges the lanes, lane 0 adds the result to the bin.  So
// each fp64 sum has one fixed order and the same call gives the same bits.  The bins' row ranges come from one pass
// that writes, for every bin b, the first row (record) whose bin is >= b -- which needs rows ordered by `delta`.
__device__ __forceinline__ GsTlPart gs_tl_shfl_down(const GsTlPart &p, int o) {
  GsTlPart q;
  q.s = gs_sum_shfl_down(p.s, o);
  q.dmin = __shfl_down_sync(0xffffffffu, p.dmin, o); q.dmax = __shfl_down_sync(0xffffffffu, p.dmax, o);
  q.last = __shfl_down_sync(0xffffffffu, p.last, o); q.fin = __shfl_down_sync(0xffffffffu, p.fin, o);
  return q;
}

__device__ __forceinline__ void gs_tl_warp_add(gs_tbin &t, GsTlPart &p) {
  for (int o = 16; o > 0; o >>= 1) { const GsTlPart q = gs_tl_shfl_down(p, o); gs_tl_merge(p, q); }
  if ((threadIdx.x & 31) == 0) gs_tl_add(t, p);
}

// Rows lo .. hi - 1 (rows[i - base], util may be NULL) into bins[0 .. B).  Rows whose `delta` never decreases take the
// warp-per-bin path; otherwise thread 0 folds them in row order (gs_tl_fold_rows_serial).  Block-cooperative.
__device__ void gs_tl_fold_rows(gs_tbin *bins, int B, long long W, const gs_tick_row *rows, const double *util, long long base,
                                long long lo, long long hi) {
  __shared__ int start[GS_TIMELINE_MAX_BINS + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  int down = 0;
  for (long long i = lo + 1 + threadIdx.x; i < hi; i += blockDim.x) down |= rows[i - base].now < rows[i - 1 - base].now;
  if (__syncthreads_or(down)) {
    if (threadIdx.x == 0) gs_tl_fold_rows_serial(bins, B, W, rows, util, base, lo, hi);
    return;
  }
  for (int b = threadIdx.x; b <= B; b += blockDim.x) start[b] = (int)(hi - lo);
  __syncthreads();
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const int k = gs_tl_bin(rows[i - base].now, W, B), kp = i > lo ? gs_tl_bin(rows[i - 1 - base].now, W, B) : -1;
    for (int b = kp + 1; b <= k; ++b) start[b] = (int)(i - lo);
  }
  __syncthreads();
  for (int b = warp; b < B; b += nwarps) {
    const long long s = lo + start[b], e = lo + start[b + 1];
    if (s >= e) continue;                                   // (warp-uniform)
    GsTlPart p;
    gs_tl_zero(p);
    for (long long i = s + lane; i < e; i += 32) gs_tl_row(p, rows[i - base], util ? util[i - base] : 0.0, i);
    gs_tl_warp_add(bins[b], p);
  }
}

// fifo: the window's records into bins[0 .. B), rows with `delta` <= wm skipped (gs_sum_fold_records' rows).  A record
// covers the ticks now_k .. t_last_k; bin b takes the records from the first one with bin(t_last) >= b up to and
// including the first one with bin(t_last) > b, each clipped to the bin's ticks with gs_sum_record -- a record that
// straddles a boundary is split there.  The gs_qrow of a record with a queue is found by counting such records (the
// pass that finds the ranges also stores each bin's count), checked, and searched for by `now` should it not match.
__device__ void gs_tl_fold_records(gs_tbin *bins, int B, long long W, const gs_evrow *ev, int nev, const gs_qrow *qr, int nq,
                                   long long ticks, long long wm) {
  __shared__ int start[GS_TIMELINE_MAX_BINS + 1], qstart[GS_TIMELINE_MAX_BINS + 1];
  __shared__ int warp_cnt[GS_SUM_THREADS / 32];
  __shared__ int k0_sh;
  if (ticks <= wm || nev == 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  auto t_last = [&](int k) -> long long { return k + 1 < nev ? (long long)ev[k + 1].now - 1 : ticks; };
  if (threadIdx.x == 0) {                                   // first record with ticks past the watermark
    int a = 0, z = nev - 1;
    while (a < z) { const int mid = (a + z) >> 1; if (t_last(mid) > wm) z = mid; else a = mid + 1; }
    k0_sh = a;
  }
  for (int b = threadIdx.x; b <= B; b += blockDim.x) { start[b] = nev; qstart[b] = 0; }
  __syncthreads();
  const int k0 = k0_sh;
  int qbase = 0;
  for (int t0 = 0; t0 < nev; t0 += blockDim.x) {
    const int k = t0 + threadIdx.x;
    const bool in = k < nev;
    const bool hasq = in && ev[k].queued > 0;
    const unsigned bal = __ballot_sync(0xffffffffu, hasq);
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    __syncthreads();
    int off = __popc(bal & ((1u << lane) - 1u)), total = 0;
    for (int w = 0; w < nwarps; ++w) { const int c = warp_cnt[w]; off += w < warp ? c : 0; total += c; }
    __syncthreads();
    if (in && k >= k0) {
      const int kh = gs_tl_bin(t_last(k), W, B), kp = k > k0 ? gs_tl_bin(t_last(k - 1), W, B) : -1;
      for (int b = kp + 1; b <= kh; ++b) { start[b] = k; qstart[b] = qbase + off; }
    }
    qbase += total;
  }
  __syncthreads();
  for (int b = warp; b < B; b += nwarps) {
    const int s = start[b];
    if (s >= nev) continue;                                 // (warp-uniform)
    const int e = start[b + 1] < nev - 1 ? start[b + 1] : nev - 1;
    const long long b_lo = (long long)b * W, b_hi = b == B - 1 ? 0x7fffffffffffffffll : ((long long)b + 1) * W - 1;
    GsTlPart p;
    gs_tl_zero(p);
    int qb = qstart[b];
    for (int c = s; c <= e; c += 32) {
      const int k = c + lane;
      const bool in = k <= e;
      gs_evrow rec;
      if (in) rec = ev[k];
      const bool hasq = in && rec.queued > 0;
      const unsigned bal = __ballot_sync(0xffffffffu, hasq);
      if (in) {
        long long v_lo = rec.now > wm + 1 ? (long long)rec.now : wm + 1;
        v_lo = v_lo > b_lo ? v_lo : b_lo;
        const long long tl = t_last(k), v_hi = tl < b_hi ? tl : b_hi;
        if (v_hi >= v_lo) {
          long long arrive_sum = 0; int oldest = 0;
          if (hasq) {
            int qi = qb + __popc(bal & ((1u << lane) - 1u));
            if (qi >= nq || qr[qi].now != rec.now) {
              int a = 0, z = nq - 1;
              while (a < z) { const int mid = (a + z) >> 1; if (qr[mid].now < rec.now) a = mid + 1; else z = mid; }
              qi = a;
            }
            const gs_qrow q = qr[qi];
            arrive_sum = q.arrive_sum; oldest = q.oldest_arrive;
          }
          gs_tl_record(p, rec, arrive_sum, oldest, v_lo, v_hi);
        }
      }
      qb += __popc(bal);
    }
    gs_tl_warp_add(bins[b], p);
  }
}

// util_sum of bins[0 .. B) = NaN (gs_summarize: the column is sampled on the host).  After the fold, block-cooperative.
__device__ void gs_tl_util_nan(gs_tbin *bins, int B) {
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) bins[b].util_sum = __longlong_as_double(0x7ff8000000000000ll);
}

// Block reduction of N 64-bit values: the first NSUM are summed, the next NMIN take the minimum, the rest the maximum;
// every thread returns with the results.
template <int N, int NSUM, int NMIN>
__device__ __forceinline__ long long gs_sum_op(int e, long long a, long long b) {
  return e < NSUM ? a + b : e < NSUM + NMIN ? (b < a ? b : a) : (b > a ? b : a);
}
template <int N, int NSUM, int NMIN>
__device__ void gs_sum_block_vec(long long (&v)[N]) {
  __shared__ long long sh[GS_SUM_THREADS / 32][N];
  __shared__ long long res[N];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
  for (int e = 0; e < N; ++e) {
    for (int o = 16; o > 0; o >>= 1) {
      v[e] = gs_sum_op<N, NSUM, NMIN>(e, v[e], __shfl_down_sync(0xffffffffu, v[e], o));
    }
    if (lane == 0) sh[warp][e] = v[e];
  }
  __syncthreads();
  if (threadIdx.x < N) {
    const int e = threadIdx.x;
    long long a = sh[0][e];
    for (int w = 1; w < nwarps; ++w) a = gs_sum_op<N, NSUM, NMIN>(e, a, sh[w][e]);
    res[e] = a;
  }
  __syncthreads();
#pragma unroll
  for (int e = 0; e < N; ++e) v[e] = res[e];
  __syncthreads();
}

// ---- occupancy block function.  One block per replica; every thread folds one fifo record or one row at a time into
// its partial sums and the histograms.  H_all / H_wait live in dynamic shared memory when their 2 * (G + 1) counters
// fit GS_OCC_SMEM_COUNTERS, else in the replica's global slot.  Lanes of a warp that
// add to the same counter sum their weights first and the lowest of them adds once: on a nearly full cluster most
// stretches hit one busy bin.  Integer adds only, so the result does not depend on the order.
enum { GS_OCC_FIFO = 0, GS_OCC_EVENTS = 1, GS_OCC_PER_TICK = 2 };

__device__ __forceinline__ void gs_occ_warp_hist(unsigned long long *stage, unsigned long long *all, unsigned long long *wait,
                                                 unsigned long long *q, const int *edges, int E, bool has, int busy, int queued,
                                                 long long w) {
  const int lane = threadIdx.x & 31;
  unsigned long long *st = stage + (threadIdx.x & ~31);
  st[lane] = has ? (unsigned long long)w : 0ull;
  __syncwarp();
  const int kb = has ? 2 * busy + (queued > 0) : -1;
  unsigned g = __match_any_sync(0xffffffffu, kb);
  if (kb >= 0 && lane == __ffs(g) - 1) {
    unsigned long long s = 0;
    for (unsigned m = g; m; m &= m - 1) s += st[__ffs(m) - 1];
    atomicAdd(all + busy, s);
    if (queued > 0) atomicAdd(wait + busy, s);
  }
  const int kq = has ? gs_jd_bin(edges, E, queued) : -1;
  g = __match_any_sync(0xffffffffu, kq);
  if (kq >= 0 && lane == __ffs(g) - 1) {
    unsigned long long s = 0;
    for (unsigned m = g; m; m &= m - 1) s += st[__ffs(m) - 1];
    atomicAdd(q + kq, s);
  }
  __syncwarp();
}

// Block-cooperative fold of one replica into rec, its carry (GS_OCC_EVENTS), and its histograms hall[0 .. G] /
// hwait[0 .. G] / hq[0 .. E] in global memory (added to); sh: the kernel's GS_OCC_SMEM_COUNTERS shared counters.  GS_OCC_FIFO: the records ev[0 .. nev) past `delta` = wm
// (gs_occ_records_serial); otherwise rows lo .. hi - 1 (rows[i - base]) as gs_occ_serial folds them: thread i reads rows
// i and i + 1, and thread 0 weighs the carry.
__device__ void gs_occ_fold(int mode, unsigned long long *occ_dyn, gs_occ *rec, GsOccCarry *carry, unsigned long long *hall,
                            unsigned long long *hwait, unsigned long long *hq, const GsOccCfg &cfg, int G, const gs_evrow *ev, int nev,
                            long long ticks, long long wm, const gs_tick_row *rows, long long base, long long lo, long long hi, int done) {
  __shared__ unsigned long long q_sh[GS_OCC_MAX_EDGES + 1];
  __shared__ unsigned long long stage[GS_SUM_THREADS];
  __shared__ int e_sh[GS_OCC_MAX_EDGES];
  const int E = cfg.nedges;
  const bool sm = 2 * (G + 1) <= GS_OCC_SMEM_COUNTERS;
  for (int i = threadIdx.x; i < E; i += blockDim.x) e_sh[i] = cfg.edges[i];
  for (int i = threadIdx.x; i <= E; i += blockDim.x) q_sh[i] = 0;
  if (sm)
    for (int i = threadIdx.x; i < 2 * (G + 1); i += blockDim.x) occ_dyn[i] = 0;
  __syncthreads();
  unsigned long long *all = sm ? occ_dyn : hall, *wait = sm ? occ_dyn + G + 1 : hwait;
  long long v[GS_OCC_N];
  gs_occ_zero(v);
  if (mode == GS_OCC_FIFO) {
    for (int t0 = 0; t0 < nev; t0 += blockDim.x) {
      const int k = t0 + threadIdx.x;
      int busy = 0, running = 0, queued = 0;
      long long L = 0;
      if (k < nev) {
        const gs_evrow e = ev[k];
        const long long t_last = k + 1 < nev ? (long long)ev[k + 1].now - 1 : ticks;
        const long long v_lo = e.now > wm + 1 ? (long long)e.now : wm + 1;
        L = t_last >= v_lo ? t_last - v_lo + 1 : 0;
        busy = e.busy_gpus; running = e.running; queued = e.queued;
      }
      gs_occ_part(v, G, busy, running, queued, L, L);
      gs_occ_warp_hist(stage, all, wait, q_sh, e_sh, E, L > 0, busy, queued, L);
    }
  } else {
    GsOccCarry c{0, 0, 0, 0, 0};
    if (mode == GS_OCC_EVENTS && threadIdx.x < 32) {        // warp 0: the carry, weighed by its successor or the end
      if (threadIdx.x == 0) c = *carry;
      const bool has = threadIdx.x == 0 && c.valid && (hi > lo || done);
      const long long w = !has ? 0 : hi > lo ? (rows[lo - base].now > c.delta ? rows[lo - base].now - c.delta : 0) : 1;
      if (has) gs_occ_part(v, G, c.busy, c.running, c.queued, 1, w);
      gs_occ_warp_hist(stage, all, wait, q_sh, e_sh, E, has && w > 0, c.busy, c.queued, w);
    }
    for (long long t0 = lo; t0 < hi; t0 += blockDim.x) {
      const long long i = t0 + threadIdx.x;
      int busy = 0, running = 0, queued = 0;
      long long n = 0, w = 0;
      if (i < hi) {
        const gs_tick_row &r = rows[i - base];
        busy = r.busy_gpus; running = r.running; queued = r.queued;
        if (mode == GS_OCC_PER_TICK) { n = 1; w = 1; }
        else if (i + 1 < hi) { const long long d = (long long)rows[i + 1 - base].now - r.now; n = 1; w = d > 0 ? d : 0; }
        else if (done) { n = 1; w = 1; }                    // the last row of a finished run; otherwise it becomes the carry
      }
      gs_occ_part(v, G, busy, running, queued, n, w);
      gs_occ_warp_hist(stage, all, wait, q_sh, e_sh, E, w > 0, busy, queued, w);
    }
    if (mode == GS_OCC_EVENTS && threadIdx.x == 0) {
      if (hi > lo && !done) {
        const gs_tick_row &r = rows[hi - 1 - base];
        c.delta = r.now; c.busy = r.busy_gpus; c.running = r.running; c.queued = r.queued; c.valid = 1;
      } else if (done) {
        c.valid = 0;
      }
      *carry = c;
    }
  }
  gs_sum_block_vec<GS_OCC_N, GS_OCC_NSUM, 0>(v);            // ends with a barrier: the shared counters are complete
  if (threadIdx.x == 0) { gs_occ_add(*rec, v); rec->total_gpus = G; }
  if (sm)
    for (int i = threadIdx.x; i < 2 * (G + 1); i += blockDim.x) {
      const unsigned long long x = occ_dyn[i];
      if (x) (i <= G ? hall[i] : hwait[i - G - 1]) += x;
    }
  for (int i = threadIdx.x; i <= E; i += blockDim.x)
    if (q_sh[i]) hq[i] += q_sh[i];
}

// Radix select of the 5 * M order statistics (M value columns x 5 ranks; M = 3 unless stated) of k values per column,
// vals[m * pitch + i] (i < k), whose column minima are mn[0 .. M) and whose largest column range is `span`.  prefix[t]
// (shared) receives target t's value minus its column's minimum; hist: 5 * M * GS_SUM_BINS shared counters.  k = 0: no
// pass is run and prefix is not to be read.  Block-cooperative: every thread calls it with the same arguments, and the
// scratch writes it reads must be published by a barrier before the call.
template <int M = 3>
__device__ __forceinline__ void gs_sum_select(unsigned *hist, unsigned long long *prefix, const int *vals, long long pitch, long long k,
                                              const long long *mn, long long span) {
  constexpr int T = 5 * M;
  static_assert(T <= GS_SUM_TARGETS, "at most GS_SUM_TARGETS targets");
  __shared__ long long rank[T];
  __shared__ int leader[T];
  const int passes = k > 0 ? gs_sum_passes((unsigned long long)span) : 0;
  if (threadIdx.x < T) {
    prefix[threadIdx.x] = 0;
    rank[threadIdx.x] = k > 0 ? gs_sum_rank(gs_sum_permille(threadIdx.x % 5), k) : 0;
  }
  for (int p = 0; p < passes; ++p) {
    const int shift = (passes - 1 - p) * 9;
    for (int i = threadIdx.x; i < T * GS_SUM_BINS; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    if (threadIdx.x < T) {                                 // targets of one value with the same prefix share a histogram
      const int t = threadIdx.x, m0 = (t / 5) * 5;
      int L = t;
      for (int u = m0; u < t; ++u) if (prefix[u] == prefix[t]) { L = u; break; }
      leader[t] = L;
    }
    __syncthreads();
    for (long long i = threadIdx.x; i < k; i += blockDim.x) {
#pragma unroll
      for (int m = 0; m < M; ++m) {
        const unsigned long long u = (unsigned long long)((long long)vals[m * pitch + i] - mn[m]);
        const unsigned long long hp = u >> (shift + 9);
        const unsigned d = (unsigned)(u >> shift) & (GS_SUM_BINS - 1);
        bool placed = false;
#pragma unroll
        for (int q = 0; q < 5; ++q) {
          const int t = m * 5 + q;
          if (!placed && leader[t] == t && prefix[t] == hp) { atomicAdd(&hist[t * GS_SUM_BINS + d], 1u); placed = true; }
        }
      }
    }
    __syncthreads();
    if (threadIdx.x < T) {
      const int t = threadIdx.x;
      long long rk = rank[t];
      const unsigned d = gs_sum_pick(hist + leader[t] * GS_SUM_BINS, rk);
      rank[t] = rk;
      prefix[t] = (prefix[t] << 9) | d;
    }
    __syncthreads();
  }
}

// Job part of replicas first .. first + count - 1, one block per replica in turn (grid-stride).  Src supplies
// finished(r) and job(r, i), the i-th finished job in finish order.  scratch: 3 * pitch ints per block.
template <class Src>
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_sum_jobs_kernel(Src src, int first, int count, gs_summary *acc,
                                                                    int *scratch, long long pitch) {
  __shared__ unsigned hist[GS_SUM_TARGETS * GS_SUM_BINS];
  __shared__ unsigned long long prefix[GS_SUM_TARGETS];
  int *vals = scratch + (size_t)blockIdx.x * 3 * (size_t)pitch;
  for (int b = blockIdx.x; b < count; b += gridDim.x) {
    const int r = first + b;
    const long long k = src.finished(r);
    long long red[11] = {0, 0, 0, 0, 0, 0x7fffffff, 0x7fffffff, 0x7fffffff, -0x80000000ll, -0x80000000ll, -0x80000000ll};
    for (long long i = threadIdx.x; i < k; i += blockDim.x) {
      const GsSumJob v = src.job(r, i);
      vals[i] = v.wait; vals[pitch + i] = v.turn; vals[2 * pitch + i] = v.jct;
      red[0] += v.wait; red[1] += v.turn; red[2] += v.jct; red[3] += v.preempt; red[4] += (long long)v.gpus * v.jct;
      red[5] = min(red[5], (long long)v.wait); red[6] = min(red[6], (long long)v.turn); red[7] = min(red[7], (long long)v.jct);
      red[8] = max(red[8], (long long)v.wait); red[9] = max(red[9], (long long)v.turn); red[10] = max(red[10], (long long)v.jct);
    }
    gs_sum_block_vec<11, 5, 3>(red);                        // (its barriers also publish the scratch writes)
    long long span = 0;
#pragma unroll
    for (int m = 0; m < 3; ++m) span = max(span, red[8 + m] - red[5 + m]);
    gs_sum_select(hist, prefix, vals, pitch, k, red + 5, span);
    if (threadIdx.x == 0) {
      gs_summary &A = acc[r];
      A.finished = k;
      A.wait_sum = red[0]; A.turnaround_sum = red[1]; A.jct_sum = red[2]; A.preempt_sum = red[3]; A.gpu_ticks_sum = red[4];
      for (int t = 0; t < 5; ++t) {
        A.wait_q[t] = k > 0 ? (int)(red[5] + (long long)prefix[t]) : 0;
        A.turnaround_q[t] = k > 0 ? (int)(red[6] + (long long)prefix[5 + t]) : 0;
        A.jct_q[t] = k > 0 ? (int)(red[7] + (long long)prefix[10 + t]) : 0;
      }
    }
    __syncthreads();
  }
}

// jobdist of replicas first .. first + count - 1 (the jobs of gs_sum_jobs_kernel, whose scratch it reuses), one block
// per replica in turn (grid-stride): (1) per-class job counts and preempt / gpu-tick sums, kept in registers per class
// and block-reduced; (2) class offsets; (3) every job's three values written to its class's segment of the scratch
// through shared per-class cursors (warp-aggregated; the order inside a segment is free, nothing depends on it);
// (4) per class in turn: sums, 128-bit sums of squares (as sums of 32-bit halves of the squares) and min / max
// block-reduced, CDF counts by binary search over the shared edges into 3 * (E + 1) shared counters, then
// (5) gs_sum_select over the segment.  Outputs: classes[r * C + c], hists[((r * C + c) * 3 + m) * (E + 1) + bin].
template <class Src>
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_jd_jobs_kernel(Src src, int first, int count, GsJdCfg cfg, gs_jclass *classes,
                                                                   unsigned *hists, int *scratch, long long pitch) {
  __shared__ unsigned hist[GS_SUM_TARGETS * GS_SUM_BINS];
  __shared__ unsigned long long prefix[GS_SUM_TARGETS];
  __shared__ unsigned cdf[3 * (GS_JOBDIST_MAX_EDGES + 1)];
  __shared__ int edges[GS_JOBDIST_MAX_EDGES];
  __shared__ long long cls_sum[3][GS_JOBDIST_MAX_CLASSES];    // jobs, preempt_sum, gpu_ticks_sum per class
  __shared__ long long cursor[GS_JOBDIST_MAX_CLASSES];
  const int C = cfg.nclasses, E = cfg.nedges, nb = E + 1;
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < E; i += blockDim.x) edges[i] = cfg.edges[i];
  int *vals = scratch + (size_t)blockIdx.x * 3 * (size_t)pitch;
  for (int b = blockIdx.x; b < count; b += gridDim.x) {
    const int r = first + b;
    const long long k = src.finished(r);
    long long red[3 * GS_JOBDIST_MAX_CLASSES];
#pragma unroll
    for (int e = 0; e < 3 * GS_JOBDIST_MAX_CLASSES; ++e) red[e] = 0;
    for (long long i = threadIdx.x; i < k; i += blockDim.x) {
      const GsSumJob v = src.job(r, i);
      const int c = gs_jd_class(cfg.bounds, C - 1, v.gpus);
#pragma unroll
      for (int u = 0; u < GS_JOBDIST_MAX_CLASSES; ++u) {
        if (c == u) { red[u] += 1; red[GS_JOBDIST_MAX_CLASSES + u] += v.preempt; red[2 * GS_JOBDIST_MAX_CLASSES + u] += (long long)v.gpus * v.jct; }
      }
    }
    gs_sum_block_vec<3 * GS_JOBDIST_MAX_CLASSES, 3 * GS_JOBDIST_MAX_CLASSES, 0>(red);
    if (threadIdx.x < GS_JOBDIST_MAX_CLASSES) {
      const int c = threadIdx.x;
      long long off = 0;
#pragma unroll
      for (int u = 0; u < GS_JOBDIST_MAX_CLASSES; ++u) off += u < c ? red[u] : 0;
#pragma unroll
      for (int u = 0; u < GS_JOBDIST_MAX_CLASSES; ++u) {
        if (u == c) { cls_sum[0][c] = red[u]; cls_sum[1][c] = red[GS_JOBDIST_MAX_CLASSES + u]; cls_sum[2][c] = red[2 * GS_JOBDIST_MAX_CLASSES + u]; }
      }
      cursor[c] = off;
    }
    __syncthreads();
    for (long long i0 = 0; i0 < k; i0 += blockDim.x) {     // (warp-uniform trip count: the shuffles see full warps)
      const long long i = i0 + threadIdx.x;
      const bool in = i < k;
      GsSumJob v;
      int c = -1;
      if (in) { v = src.job(r, i); c = gs_jd_class(cfg.bounds, C - 1, v.gpus); }
      const unsigned peers = __match_any_sync(0xffffffffu, c);
      const int head = __ffs(peers) - 1;
      long long base = 0;
      if (in && lane == head) base = atomicAdd((unsigned long long *)&cursor[c], (unsigned long long)__popc(peers));
      base = __shfl_sync(0xffffffffu, base, head);
      if (in) {
        const long long pos = base + __popc(peers & ((1u << lane) - 1u));
        vals[pos] = v.wait; vals[pitch + pos] = v.turn; vals[2 * pitch + pos] = v.jct;
      }
    }
    __syncthreads();
    long long off = 0;
    for (int c = 0; c < C; ++c) {
      const long long kc = cls_sum[0][c];
      const int *seg = vals + off;
      for (int i = threadIdx.x; i < 3 * nb; i += blockDim.x) cdf[i] = 0;
      __syncthreads();
      // sums; squares as the sums of their high and low 32-bit halves (each fits 64 bits); minima; maxima
      long long s[15] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0x7fffffff, 0x7fffffff, 0x7fffffff, -0x80000000ll, -0x80000000ll, -0x80000000ll};
      for (long long i = threadIdx.x; i < kc; i += blockDim.x) {
#pragma unroll
        for (int m = 0; m < 3; ++m) {
          const int v = seg[m * pitch + i];
          const unsigned long long sq = (unsigned long long)((long long)v * v);
          s[m] += v; s[3 + m] += (long long)(sq >> 32); s[6 + m] += (long long)(sq & 0xffffffffull);
          s[9 + m] = min(s[9 + m], (long long)v); s[12 + m] = max(s[12 + m], (long long)v);
          atomicAdd(&cdf[m * nb + gs_jd_bin(edges, E, v)], 1u);
        }
      }
      gs_sum_block_vec<15, 9, 3>(s);                        // (its barriers also publish the CDF counts)
      unsigned *hout = hists + ((size_t)r * C + c) * 3 * (size_t)nb;
      for (int i = threadIdx.x; i < 3 * nb; i += blockDim.x) hout[i] = cdf[i];
      long long span = 0;
#pragma unroll
      for (int m = 0; m < 3; ++m) span = max(span, s[12 + m] - s[9 + m]);
      gs_sum_select(hist, prefix, seg, pitch, kc, s + 9, span);
      if (threadIdx.x == 0) {
        gs_jclass J = {};
        J.jobs = kc; J.wait_sum = s[0]; J.turnaround_sum = s[1]; J.jct_sum = s[2];
        J.preempt_sum = cls_sum[1][c]; J.gpu_ticks_sum = cls_sum[2][c];
        gs_sum_add128(J.wait_sq_lo, J.wait_sq_hi, ((gs_i128)s[3] << 32) + s[6]);
        gs_sum_add128(J.turnaround_sq_lo, J.turnaround_sq_hi, ((gs_i128)s[4] << 32) + s[7]);
        gs_sum_add128(J.jct_sq_lo, J.jct_sq_hi, ((gs_i128)s[5] << 32) + s[8]);
        for (int t = 0; t < 5; ++t) {
          J.wait_q[t] = kc > 0 ? (int)(s[9] + (long long)prefix[t]) : 0;
          J.turnaround_q[t] = kc > 0 ? (int)(s[10] + (long long)prefix[5 + t]) : 0;
          J.jct_q[t] = kc > 0 ? (int)(s[11] + (long long)prefix[10 + t]) : 0;
        }
        classes[(size_t)r * C + c] = J;
      }
      __syncthreads();
      off += kc;
    }
  }
}

// Slowdown statistics (gs_sdclass) of replicas first .. first + count - 1 (the jobs of gs_sum_jobs_kernel, whose
// scratch it reuses with a fourth row), one block per replica in turn (grid-stride), in gs_jd_jobs_kernel's steps:
// (1) per-class job counts, preempt / gpu-tick sums and key sums (as sums of the keys' 32-bit halves), kept in registers
// per class and block-reduced; (2) class offsets; (3) every job's wait, turnaround, jct and sd written to its class's
// segment of the scratch through warp-aggregated shared cursors; (4) per class in turn: jobdist's fold of the three
// values (sums, 128-bit sums of squares as sums of 32-bit halves, min / max, CDF counts), then the same fold of sd
// (with the count of saturated values), then gs_sum_select over the three rows and a second, one-row gs_sum_select
// over the sd row (a widened 20-target select would need 40 KB of histogram counters on its own).
// Outputs: recs[r * C + c], hists[(r * C + c) * (3 * (E + 1) + Esd + 1) + ...] ([wait, turnaround, jct, sd][bin]).
template <class Src>
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_sd_jobs_kernel(Src src, int first, int count, GsSdCfg cfg, gs_sdclass *recs,
                                                                   unsigned *hists, int *scratch, long long pitch) {
  constexpr int NC = GS_JOBDIST_MAX_CLASSES;
  __shared__ unsigned hist[GS_SUM_TARGETS * GS_SUM_BINS];
  __shared__ unsigned long long prefix[GS_SUM_TARGETS];
  __shared__ unsigned cdf[3 * (GS_JOBDIST_MAX_EDGES + 1) + GS_SLOWDOWN_MAX_EDGES + 1];
  __shared__ int edges[GS_JOBDIST_MAX_EDGES], sd_edges[GS_SLOWDOWN_MAX_EDGES];
  __shared__ long long cls_sum[5][NC];          // jobs, preempt_sum, gpu_ticks_sum, key low halves, key high halves
  __shared__ long long cursor[NC];
  __shared__ gs_sdclass rec;
  const int C = cfg.nclasses, E = cfg.nedges, nb = E + 1, Es = cfg.nsd;
  const int row = 3 * nb + Es + 1;
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < E; i += blockDim.x) edges[i] = cfg.edges[i];
  for (int i = threadIdx.x; i < Es; i += blockDim.x) sd_edges[i] = cfg.sd_edges[i];
  int *vals = scratch + (size_t)blockIdx.x * 4 * (size_t)pitch;
  for (int b = blockIdx.x; b < count; b += gridDim.x) {
    const int r = first + b;
    const long long k = src.finished(r);
    long long red[5 * NC];
#pragma unroll
    for (int e = 0; e < 5 * NC; ++e) red[e] = 0;
    for (long long i = threadIdx.x; i < k; i += blockDim.x) {
      const GsSumJob v = src.job(r, i);
      const long long key = gs_sd_key(cfg.key, v.gpus, v.jct);
      const int c = gs_sd_class(cfg.bounds, C - 1, key);
#pragma unroll
      for (int u = 0; u < NC; ++u) {
        if (c == u) {
          red[u] += 1; red[NC + u] += v.preempt; red[2 * NC + u] += (long long)v.gpus * v.jct;
          red[3 * NC + u] += key & 0xffffffffll; red[4 * NC + u] += key >> 32;
        }
      }
    }
    gs_sum_block_vec<5 * NC, 5 * NC, 0>(red);
    if (threadIdx.x < NC) {
      const int c = threadIdx.x;
      long long off = 0;
#pragma unroll
      for (int u = 0; u < NC; ++u) off += u < c ? red[u] : 0;
#pragma unroll
      for (int u = 0; u < NC; ++u) {
        if (u == c)
          for (int m = 0; m < 5; ++m) cls_sum[m][c] = red[m * NC + u];
      }
      cursor[c] = off;
    }
    __syncthreads();
    for (long long i0 = 0; i0 < k; i0 += blockDim.x) {     // (warp-uniform trip count: the shuffles see full warps)
      const long long i = i0 + threadIdx.x;
      const bool in = i < k;
      GsSumJob v;
      int c = -1;
      if (in) { v = src.job(r, i); c = gs_sd_class(cfg.bounds, C - 1, gs_sd_key(cfg.key, v.gpus, v.jct)); }
      const unsigned peers = __match_any_sync(0xffffffffu, c);
      const int head = __ffs(peers) - 1;
      long long base = 0;
      if (in && lane == head) base = atomicAdd((unsigned long long *)&cursor[c], (unsigned long long)__popc(peers));
      base = __shfl_sync(0xffffffffu, base, head);
      if (in) {
        const long long pos = base + __popc(peers & ((1u << lane) - 1u));
        vals[pos] = v.wait; vals[pitch + pos] = v.turn; vals[2 * pitch + pos] = v.jct;
        vals[3 * pitch + pos] = gs_sd_value(v.turn, v.jct, cfg.tau);
      }
    }
    __syncthreads();
    long long off = 0;
    for (int c = 0; c < C; ++c) {
      const long long kc = cls_sum[0][c];
      const int *seg = vals + off;
      for (int i = threadIdx.x; i < row; i += blockDim.x) cdf[i] = 0;
      __syncthreads();
      // wait, turnaround, jct: sums; squares as the sums of their high and low 32-bit halves; minima; maxima
      long long s[15] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0x7fffffff, 0x7fffffff, 0x7fffffff, -0x80000000ll, -0x80000000ll, -0x80000000ll};
      for (long long i = threadIdx.x; i < kc; i += blockDim.x) {
#pragma unroll
        for (int m = 0; m < 3; ++m) {
          const int v = seg[m * pitch + i];
          const unsigned long long sq = (unsigned long long)((long long)v * v);
          s[m] += v; s[3 + m] += (long long)(sq >> 32); s[6 + m] += (long long)(sq & 0xffffffffull);
          s[9 + m] = min(s[9 + m], (long long)v); s[12 + m] = max(s[12 + m], (long long)v);
          atomicAdd(&cdf[m * nb + gs_jd_bin(edges, E, v)], 1u);
        }
      }
      gs_sum_block_vec<15, 9, 3>(s);
      // sd: sum, square halves, saturated count, minimum, maximum
      long long t[6] = {0, 0, 0, 0, GS_SD_MAX, 0};
      for (long long i = threadIdx.x; i < kc; i += blockDim.x) {
        const int v = seg[3 * pitch + i];
        const unsigned long long sq = (unsigned long long)((long long)v * v);
        t[0] += v; t[1] += (long long)(sq >> 32); t[2] += (long long)(sq & 0xffffffffull); t[3] += v == (int)GS_SD_MAX;
        t[4] = min(t[4], (long long)v); t[5] = max(t[5], (long long)v);
        atomicAdd(&cdf[3 * nb + gs_jd_bin(sd_edges, Es, v)], 1u);
      }
      gs_sum_block_vec<6, 4, 1>(t);                         // (its barriers also publish the CDF counts)
      unsigned *hout = hists + ((size_t)r * C + c) * (size_t)row;
      for (int i = threadIdx.x; i < row; i += blockDim.x) hout[i] = cdf[i];
      long long span = 0;
#pragma unroll
      for (int m = 0; m < 3; ++m) span = max(span, s[12 + m] - s[9 + m]);
      gs_sum_select(hist, prefix, seg, pitch, kc, s + 9, span);
      if (threadIdx.x == 0) {
        rec = gs_sdclass{};
        gs_jclass &J = rec.jc;
        J.jobs = kc; J.wait_sum = s[0]; J.turnaround_sum = s[1]; J.jct_sum = s[2];
        J.preempt_sum = cls_sum[1][c]; J.gpu_ticks_sum = cls_sum[2][c];
        gs_sum_add128(J.wait_sq_lo, J.wait_sq_hi, ((gs_i128)s[3] << 32) + s[6]);
        gs_sum_add128(J.turnaround_sq_lo, J.turnaround_sq_hi, ((gs_i128)s[4] << 32) + s[7]);
        gs_sum_add128(J.jct_sq_lo, J.jct_sq_hi, ((gs_i128)s[5] << 32) + s[8]);
        for (int q = 0; q < 5; ++q) {
          J.wait_q[q] = kc > 0 ? (int)(s[9] + (long long)prefix[q]) : 0;
          J.turnaround_q[q] = kc > 0 ? (int)(s[10] + (long long)prefix[5 + q]) : 0;
          J.jct_q[q] = kc > 0 ? (int)(s[11] + (long long)prefix[10 + q]) : 0;
        }
        rec.sd_sum = t[0];
        gs_sum_add128(rec.sd_sq_lo, rec.sd_sq_hi, ((gs_i128)t[1] << 32) + t[2]);
        rec.sd_clamped = t[3];
        rec.sd_min = kc > 0 ? (int)t[4] : 0;
        gs_sum_add128(rec.key_sum_lo, rec.key_sum_hi, ((gs_i128)cls_sum[4][c] << 32) + cls_sum[3][c]);
      }
      __syncthreads();                                      // thread 0 has read prefix before the second select
      gs_sum_select<1>(hist, prefix, seg + 3 * pitch, pitch, kc, t + 4, t[5] - t[4]);
      if (threadIdx.x == 0) {
        for (int q = 0; q < 5; ++q) rec.sd_q[q] = kc > 0 ? (int)(t[4] + (long long)prefix[q]) : 0;
        recs[(size_t)r * C + c] = rec;
      }
      __syncthreads();
      off += kc;
    }
  }
}

// ---- job statistics by arrival time.  Every lane of a warp calls gs_arr_count with its bin (b < 0: nothing to
// count); the lanes of one bin add once.
__device__ __forceinline__ void gs_arr_count(unsigned *ctr, int b) {
  const unsigned peers = __match_any_sync(0xffffffffu, b);
  if (b >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&ctr[b], (unsigned)__popc(peers));
}

// Bitonic sort of buf[0 .. P) ascending by one warp (P a power of two, 2 <= P); every lane calls it, after a __syncwarp
// that publishes buf, and returns after one.
__device__ __forceinline__ void gs_arr_warp_sort(int *buf, int P) {
  const int lane = threadIdx.x & 31;
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = lane; t < P / 2; t += 32) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;   // the pair (lo, lo + stride), lo's stride bit clear
        const int x = buf[lo], y = buf[hi];
        if ((x > y) == ((lo & size) == 0)) { buf[lo] = y; buf[hi] = x; }
      }
      __syncwarp();
    }
  }
}

// One bin of m <= GS_ARR_CUT finished jobs, seg[row * pitch + i] (i < m, rows as in gs_arr_jobs_kernel), finished by
// one warp: the sums by lane partials and shuffles; then each value row copied to buf (GS_ARR_CUT ints), padded with
// 2^31 - 1 to a power of two, sorted, and the five ranks read off (the padding sorts last, past every rank < m).  The
// record is staged in *wr (shared) and copied to *out as 30 words.  Every lane calls it.
__device__ void gs_arr_warp_bin(const int *seg, long long pitch, int m, unsigned arrived, int *buf, gs_abin *wr, gs_abin *out) {
  const int lane = threadIdx.x & 31;
  // wait, turnaround, jct, sd: sums, square high halves, square low halves; then saturated sd, preempt, gpu ticks, arrivals
  long long a[16];
#pragma unroll
  for (int e = 0; e < 16; ++e) a[e] = 0;
  for (int i = lane; i < m; i += 32) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int v = seg[c * pitch + i];
      const unsigned long long sq = (unsigned long long)((long long)v * v);
      a[c] += v; a[4 + c] += (long long)(sq >> 32); a[8 + c] += (long long)(sq & 0xffffffffull);
    }
    a[12] += seg[3 * pitch + i] == (int)GS_SD_MAX;
    a[13] += seg[4 * pitch + i];
    a[14] += (long long)seg[5 * pitch + i] * seg[2 * pitch + i];
    a[15] += seg[6 * pitch + i];
  }
#pragma unroll
  for (int e = 0; e < 16; ++e)
    for (int o = 16; o > 0; o >>= 1) a[e] += __shfl_xor_sync(0xffffffffu, a[e], o);
  unsigned long long *w = reinterpret_cast<unsigned long long *>(wr);
  if (lane < (int)(sizeof(gs_abin) / 8)) w[lane] = 0;
  __syncwarp();
  if (lane == 0) {
    gs_jclass &J = wr->s.jc;
    J.jobs = m; J.wait_sum = a[0]; J.turnaround_sum = a[1]; J.jct_sum = a[2]; J.preempt_sum = a[13]; J.gpu_ticks_sum = a[14];
    gs_sum_add128(J.wait_sq_lo, J.wait_sq_hi, ((gs_i128)a[4] << 32) + a[8]);
    gs_sum_add128(J.turnaround_sq_lo, J.turnaround_sq_hi, ((gs_i128)a[5] << 32) + a[9]);
    gs_sum_add128(J.jct_sq_lo, J.jct_sq_hi, ((gs_i128)a[6] << 32) + a[10]);
    wr->s.sd_sum = a[3];
    gs_sum_add128(wr->s.sd_sq_lo, wr->s.sd_sq_hi, ((gs_i128)a[7] << 32) + a[11]);
    wr->s.sd_clamped = a[12];
    gs_sum_add128(wr->s.key_sum_lo, wr->s.key_sum_hi, (gs_i128)a[15]);
    wr->arrived = arrived;
  }
  if (m > 0) {
    int P = 32;
    while (P < m) P <<= 1;
    for (int c = 0; c < 4; ++c) {
      for (int i = lane; i < P; i += 32) buf[i] = i < m ? seg[c * pitch + i] : 0x7fffffff;
      __syncwarp();
      gs_arr_warp_sort(buf, P);
      if (lane < 5) {
        int *q = c == 0 ? wr->s.jc.wait_q : c == 1 ? wr->s.jc.turnaround_q : c == 2 ? wr->s.jc.jct_q : wr->s.sd_q;
        q[lane] = buf[gs_sum_rank(gs_sum_permille(lane), m)];
      }
      if (c == 3 && lane == 0) wr->s.sd_min = buf[0];
      __syncwarp();                                         // buf is read before the next row overwrites it
    }
  }
  __syncwarp();
  if (lane < (int)(sizeof(gs_abin) / 8)) reinterpret_cast<unsigned long long *>(out)[lane] = w[lane];
  __syncwarp();                                             // *wr is read before the warp's next bin
}

// Arrival-bin statistics (gs_abin) of replicas first .. first + count - 1 (the jobs of gs_sum_jobs_kernel), one block
// per replica in turn (grid-stride).  Src supplies n(r), finished(r), order(r, i), job_at(r, j) and arrive_at(r, j).
// Its own scratch: GS_ARR_ROWS * pitch ints per block, rows wait, turnaround, jct, sd, preempt, gpus, arrival tick.
// (1) finished jobs per bin, and every trace job per bin (`arrived`), in shared counters (warp-aggregated adds);
// (2) an exclusive scan of the finished counts gives each bin's segment; (3) every finished job's seven values are
// written to its bin's segment through warp-aggregated shared cursors (the order inside a segment is free, nothing
// depends on it); (4) each bin of at most GS_ARR_CUT jobs is finished by one warp (gs_arr_warp_bin: sums by shuffles,
// order statistics by a bitonic sort in shared memory), eight bins in flight; (5) each larger bin is finished by the
// block, as gs_sd_jobs_kernel finishes a class: sums, minima and maxima block-reduced, gs_sum_select over the three
// rows and a one-row gs_sum_select over sd.  Both paths are exact, so a bin's record does not depend on its path.
// The warps' sort buffers and staging records live in the selects' histogram space, which (4) and (5) use in turn.
template <class Src>
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_arr_jobs_kernel(Src src, int first, int count, GsArrCfg cfg, gs_abin *recs,
                                                                    int *scratch, long long pitch) {
  constexpr int NW = GS_SUM_THREADS / 32;
  static_assert(GS_ARRIVALS_MAX_BINS <= 4 * GS_SUM_THREADS, "the scan takes four bins per thread");
  static_assert(NW * (GS_ARR_CUT * sizeof(int) + sizeof(gs_abin)) <= GS_SUM_TARGETS * GS_SUM_BINS * sizeof(unsigned),
                "the warps' buffers fit the histogram space");
  __shared__ __align__(16) unsigned hist[GS_SUM_TARGETS * GS_SUM_BINS];
  __shared__ unsigned long long prefix[GS_SUM_TARGETS];
  __shared__ unsigned cnt[GS_ARRIVALS_MAX_BINS + 1];      // finished jobs per bin, then the segments' first positions
  __shared__ unsigned cursor[GS_ARRIVALS_MAX_BINS];
  __shared__ unsigned arrived[GS_ARRIVALS_MAX_BINS];
  __shared__ unsigned wtot[NW];
  __shared__ gs_abin rec;
  const int B = cfg.nbins, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int *buf = reinterpret_cast<int *>(hist) + warp * GS_ARR_CUT;
  gs_abin *wr = reinterpret_cast<gs_abin *>(hist + NW * GS_ARR_CUT) + warp;
  int *vals = scratch + (size_t)blockIdx.x * GS_ARR_ROWS * (size_t)pitch;
  for (int rb = blockIdx.x; rb < count; rb += gridDim.x) {
    const int r = first + rb;
    const long long n = src.n(r), k = src.finished(r);
    for (int i = threadIdx.x; i < B; i += blockDim.x) { cnt[i] = 0; arrived[i] = 0; }
    __syncthreads();
    for (long long i0 = 0; i0 < n; i0 += blockDim.x) {     // (warp-uniform trip count: the matches see full warps)
      const long long i = i0 + threadIdx.x;
      gs_arr_count(arrived, i < n ? gs_tl_bin(src.arrive_at(r, (int)i), cfg.width, B) : -1);
      gs_arr_count(cnt, i < k ? gs_tl_bin(src.arrive_at(r, src.order(r, i)), cfg.width, B) : -1);
    }
    __syncthreads();
    {                                                       // cnt[b] := jobs of bins < b; cnt[B] = k
      unsigned v[4], sum = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int b = 4 * threadIdx.x + q;
        v[q] = b < B ? cnt[b] : 0u;
        sum += v[q];
      }
      unsigned inc = sum;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      if (lane == 31) wtot[warp] = inc;
      __syncthreads();
      unsigned base = inc - sum;
      for (int u = 0; u < warp; ++u) base += wtot[u];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int b = 4 * threadIdx.x + q;
        if (b < B) { cnt[b] = base; cursor[b] = base; }
        base += v[q];
      }
      if (threadIdx.x == 0) cnt[B] = (unsigned)k;
    }
    __syncthreads();
    for (long long i0 = 0; i0 < k; i0 += blockDim.x) {     // (warp-uniform trip count: the shuffles see full warps)
      const long long i = i0 + threadIdx.x;
      const bool in = i < k;
      GsSumJob v;
      int a = 0, b = -1;
      if (in) {
        const int j = src.order(r, i);
        v = src.job_at(r, j);
        a = src.arrive_at(r, j);
        b = gs_tl_bin(a, cfg.width, B);
      }
      const unsigned peers = __match_any_sync(0xffffffffu, b);
      const int head = __ffs(peers) - 1;
      unsigned base = 0;
      if (in && lane == head) base = atomicAdd(&cursor[b], (unsigned)__popc(peers));
      base = __shfl_sync(0xffffffffu, base, head);
      if (in) {
        const long long pos = (long long)base + __popc(peers & ((1u << lane) - 1u));
        vals[pos] = v.wait; vals[pitch + pos] = v.turn; vals[2 * pitch + pos] = v.jct;
        vals[3 * pitch + pos] = gs_sd_value(v.turn, v.jct, cfg.tau);
        vals[4 * pitch + pos] = v.preempt; vals[5 * pitch + pos] = v.gpus; vals[6 * pitch + pos] = a;
      }
    }
    __syncthreads();
    for (int b = warp; b < B; b += NW) {
      const int o = (int)cnt[b], m = (int)(cnt[b + 1] - cnt[b]);
      if (m <= GS_ARR_CUT) gs_arr_warp_bin(vals + o, pitch, m, arrived[b], buf, wr, recs + (size_t)r * B + b);
    }
    __syncthreads();                                        // the warps are done with the histogram space
    for (int b = 0; b < B; ++b) {                           // (uniform: every thread reads the same counts)
      const long long o = cnt[b], m = (long long)cnt[b + 1] - o;
      if (m <= GS_ARR_CUT) continue;
      const int *seg = vals + o;
      // wait, turnaround, jct: sums, square high halves, square low halves; preempt, gpu ticks, arrivals; minima; maxima
      long long s[18] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0x7fffffff, 0x7fffffff, 0x7fffffff, -0x80000000ll, -0x80000000ll, -0x80000000ll};
      for (long long i = threadIdx.x; i < m; i += blockDim.x) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int v = seg[c * pitch + i];
          const unsigned long long sq = (unsigned long long)((long long)v * v);
          s[c] += v; s[3 + c] += (long long)(sq >> 32); s[6 + c] += (long long)(sq & 0xffffffffull);
          s[12 + c] = min(s[12 + c], (long long)v); s[15 + c] = max(s[15 + c], (long long)v);
        }
        s[9] += seg[4 * pitch + i];
        s[10] += (long long)seg[5 * pitch + i] * seg[2 * pitch + i];
        s[11] += seg[6 * pitch + i];
      }
      gs_sum_block_vec<18, 12, 3>(s);
      // sd: sum, square halves, saturated count, minimum, maximum
      long long t[6] = {0, 0, 0, 0, GS_SD_MAX, 0};
      for (long long i = threadIdx.x; i < m; i += blockDim.x) {
        const int v = seg[3 * pitch + i];
        const unsigned long long sq = (unsigned long long)((long long)v * v);
        t[0] += v; t[1] += (long long)(sq >> 32); t[2] += (long long)(sq & 0xffffffffull); t[3] += v == (int)GS_SD_MAX;
        t[4] = min(t[4], (long long)v); t[5] = max(t[5], (long long)v);
      }
      gs_sum_block_vec<6, 4, 1>(t);
      long long span = 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) span = max(span, s[15 + c] - s[12 + c]);
      gs_sum_select(hist, prefix, seg, pitch, m, s + 12, span);
      if (threadIdx.x == 0) {
        rec = gs_abin{};
        gs_jclass &J = rec.s.jc;
        J.jobs = m; J.wait_sum = s[0]; J.turnaround_sum = s[1]; J.jct_sum = s[2]; J.preempt_sum = s[9]; J.gpu_ticks_sum = s[10];
        gs_sum_add128(J.wait_sq_lo, J.wait_sq_hi, ((gs_i128)s[3] << 32) + s[6]);
        gs_sum_add128(J.turnaround_sq_lo, J.turnaround_sq_hi, ((gs_i128)s[4] << 32) + s[7]);
        gs_sum_add128(J.jct_sq_lo, J.jct_sq_hi, ((gs_i128)s[5] << 32) + s[8]);
        for (int q = 0; q < 5; ++q) {
          J.wait_q[q] = (int)(s[12] + (long long)prefix[q]);
          J.turnaround_q[q] = (int)(s[13] + (long long)prefix[5 + q]);
          J.jct_q[q] = (int)(s[14] + (long long)prefix[10 + q]);
        }
        rec.s.sd_sum = t[0];
        gs_sum_add128(rec.s.sd_sq_lo, rec.s.sd_sq_hi, ((gs_i128)t[1] << 32) + t[2]);
        rec.s.sd_clamped = t[3];
        rec.s.sd_min = (int)t[4];
        gs_sum_add128(rec.s.key_sum_lo, rec.s.key_sum_hi, (gs_i128)s[11]);
        rec.arrived = arrived[b];
      }
      __syncthreads();                                      // thread 0 has read prefix before the second select
      gs_sum_select<1>(hist, prefix, seg + 3 * pitch, pitch, m, t + 4, t[5] - t[4]);
      if (threadIdx.x == 0) {
        for (int q = 0; q < 5; ++q) rec.s.sd_q[q] = (int)(t[4] + (long long)prefix[q]);
        recs[(size_t)r * B + b] = rec;
      }
      __syncthreads();
    }
    __syncthreads();                                        // every thread has read cnt before the next replica clears it
  }
}

// Paired comparison (gs_jpair) of pairs (pa[p], pb[p]), p < npairs, one block per pair in turn (grid-stride).  Src
// supplies n(r), finished(r), order(r, i) (the i-th job of the finish order), job_at(r, j) (job j of the trace) and
// same_job(ra, rb, j) (the trace records of job j are equal); the host has checked that both replicas hold n jobs.
// scratch: 4 * pitch ints per block, membership words then three columns of differences.  Per pair:
// (1) membership words: zeroed, bit 1 from a's finish order, bit 2 from b's (each job is at most once in an order, so
// plain stores); (2) one pass in trace order: trace equality (a pair that differs sets flags[p] and stops here) and
// the per-class counts jobs / only_a / only_b, block-reduced; (3) class offsets, and d = x_b - x_a of every job
// finished in both runs scattered into its class's segment through warp-aggregated cursors (jd's step 3); (4) per
// class: counts by sign, sums, 128-bit sums of squares (as sums of 32-bit halves), min / max block-reduced, CDF counts
// into shared counters, gs_sum_select over the segment for q_hi, then the segment negated in place and selected again
// for q_lo = -result.  Outputs recs[p * C + c], hists[((p * C + c) * 3 + m) * (E + 1) + bin].
template <class Src>
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_cmp_pairs_kernel(Src src, int npairs, const int *pa, const int *pb, GsJdCfg cfg,
                                                                     gs_jpair *recs, unsigned *hists, int *flags, int *scratch,
                                                                     long long pitch) {
  __shared__ unsigned hist[GS_SUM_TARGETS * GS_SUM_BINS];
  __shared__ unsigned long long prefix[GS_SUM_TARGETS];
  __shared__ unsigned cdf[3 * (GS_JOBDIST_MAX_EDGES + 1)];
  __shared__ int edges[GS_JOBDIST_MAX_EDGES];
  __shared__ long long cls_cnt[3][GS_JOBDIST_MAX_CLASSES];    // jobs, only_a, only_b per class
  __shared__ long long cursor[GS_JOBDIST_MAX_CLASSES];
  __shared__ gs_jpair rec;
  const int C = cfg.nclasses, E = cfg.nedges, nb = E + 1;
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < E; i += blockDim.x) edges[i] = cfg.edges[i];
  int *mem = scratch + (size_t)blockIdx.x * 4 * (size_t)pitch;
  int *vals = mem + pitch;
  for (int p = blockIdx.x; p < npairs; p += gridDim.x) {
    const int ra = pa[p], rb = pb[p];
    const long long n = src.n(ra), ka = src.finished(ra), kb = src.finished(rb);
    for (long long j = threadIdx.x; j < n; j += blockDim.x) mem[j] = 0;
    __syncthreads();
    for (long long i = threadIdx.x; i < ka; i += blockDim.x) mem[src.order(ra, i)] = 1;
    __syncthreads();
    for (long long i = threadIdx.x; i < kb; i += blockDim.x) mem[src.order(rb, i)] |= 2;
    __syncthreads();
    long long red[3 * GS_JOBDIST_MAX_CLASSES];
#pragma unroll
    for (int e = 0; e < 3 * GS_JOBDIST_MAX_CLASSES; ++e) red[e] = 0;
    int diff = 0;
    for (long long j = threadIdx.x; j < n; j += blockDim.x) {
      diff |= !src.same_job(ra, rb, (int)j);
      const int w = mem[j];
      if (w == 0) continue;
      const int c = gs_jd_class(cfg.bounds, C - 1, src.job_at(ra, (int)j).gpus);
      const int s = w == 3 ? 0 : w == 1 ? GS_JOBDIST_MAX_CLASSES : 2 * GS_JOBDIST_MAX_CLASSES;
#pragma unroll
      for (int u = 0; u < GS_JOBDIST_MAX_CLASSES; ++u) {
        if (c == u) { red[u] += s == 0; red[GS_JOBDIST_MAX_CLASSES + u] += s == GS_JOBDIST_MAX_CLASSES; red[2 * GS_JOBDIST_MAX_CLASSES + u] += s == 2 * GS_JOBDIST_MAX_CLASSES; }
      }
    }
    diff = __syncthreads_or(diff);
    if (threadIdx.x == 0) flags[p] = diff;
    if (diff) continue;                                       // (block-uniform; the host refuses the call)
    gs_sum_block_vec<3 * GS_JOBDIST_MAX_CLASSES, 3 * GS_JOBDIST_MAX_CLASSES, 0>(red);
    if (threadIdx.x < GS_JOBDIST_MAX_CLASSES) {
      const int c = threadIdx.x;
      long long off = 0;
#pragma unroll
      for (int u = 0; u < GS_JOBDIST_MAX_CLASSES; ++u) off += u < c ? red[u] : 0;
#pragma unroll
      for (int u = 0; u < GS_JOBDIST_MAX_CLASSES; ++u) {
        if (u == c) { cls_cnt[0][c] = red[u]; cls_cnt[1][c] = red[GS_JOBDIST_MAX_CLASSES + u]; cls_cnt[2][c] = red[2 * GS_JOBDIST_MAX_CLASSES + u]; }
      }
      cursor[c] = off;
    }
    __syncthreads();
    for (long long j0 = 0; j0 < n; j0 += blockDim.x) {      // (warp-uniform trip count: the shuffles see full warps)
      const long long j = j0 + threadIdx.x;
      const bool in = j < n && mem[j] == 3;
      GsSumJob va, vb;
      int c = -1;
      if (in) { va = src.job_at(ra, (int)j); vb = src.job_at(rb, (int)j); c = gs_jd_class(cfg.bounds, C - 1, va.gpus); }
      const unsigned peers = __match_any_sync(0xffffffffu, c);
      const int head = __ffs(peers) - 1;
      long long base = 0;
      if (in && lane == head) base = atomicAdd((unsigned long long *)&cursor[c], (unsigned long long)__popc(peers));
      base = __shfl_sync(0xffffffffu, base, head);
      if (in) {
        const long long pos = base + __popc(peers & ((1u << lane) - 1u));
        vals[pos] = vb.wait - va.wait; vals[pitch + pos] = vb.turn - va.turn; vals[2 * pitch + pos] = vb.jct - va.jct;
      }
    }
    __syncthreads();
    long long off = 0;
    for (int c = 0; c < C; ++c) {
      const long long kc = cls_cnt[0][c];
      int *seg = vals + off;
      for (int i = threadIdx.x; i < 3 * nb; i += blockDim.x) cdf[i] = 0;
      if (threadIdx.x == 0) { rec = gs_jpair{}; rec.jobs = kc; rec.only_a = cls_cnt[1][c]; rec.only_b = cls_cnt[2][c]; }
      __syncthreads();
      long long mn[3], mx[3];
#pragma unroll
      for (int m = 0; m < 3; ++m) {                         // one quantity at a time (7 values per reduction: no spills)
        // #(d < 0), #(d > 0), sum, squares as the sums of their high and low 32-bit halves, min, max
        long long s[7] = {0, 0, 0, 0, 0, 0x7fffffff, -0x80000000ll};
        for (long long i = threadIdx.x; i < kc; i += blockDim.x) {
          const int d = seg[m * pitch + i];
          const unsigned long long sq = (unsigned long long)((long long)d * d);
          s[0] += d < 0; s[1] += d > 0; s[2] += d;
          s[3] += (long long)(sq >> 32); s[4] += (long long)(sq & 0xffffffffull);
          s[5] = min(s[5], (long long)d); s[6] = max(s[6], (long long)d);
          atomicAdd(&cdf[m * nb + gs_jd_bin(edges, E, d)], 1u);
        }
        gs_sum_block_vec<7, 5, 1>(s);                       // (its barriers also publish the CDF counts)
        mn[m] = s[5]; mx[m] = s[6];
        if (threadIdx.x == 0) {
          rec.lt[m] = s[0]; rec.gt[m] = s[1]; rec.eq[m] = kc - s[0] - s[1]; rec.d_sum[m] = s[2];
          gs_sum_add128(rec.d_sq_lo[m], rec.d_sq_hi[m], ((gs_i128)s[3] << 32) + s[4]);
        }
      }
      unsigned *hout = hists + ((size_t)p * C + c) * 3 * (size_t)nb;
      for (int i = threadIdx.x; i < 3 * nb; i += blockDim.x) hout[i] = cdf[i];
      long long span = 0;
#pragma unroll
      for (int m = 0; m < 3; ++m) span = max(span, mx[m] - mn[m]);
      gs_sum_select(hist, prefix, seg, pitch, kc, mn, span);
      if (threadIdx.x == 0)
        for (int m = 0; m < 3; ++m)
          for (int t = 0; t < 5; ++t) rec.q_hi[m][t] = kc > 0 ? (int)(mn[m] + (long long)prefix[m * 5 + t]) : 0;
      for (long long i = threadIdx.x; i < kc; i += blockDim.x) {
#pragma unroll
        for (int m = 0; m < 3; ++m) seg[m * pitch + i] = -seg[m * pitch + i];
      }
      long long nmin[3];
#pragma unroll
      for (int m = 0; m < 3; ++m) nmin[m] = -mx[m];
      __syncthreads();                                      // thread 0 has read prefix; the negated segment is published
      gs_sum_select(hist, prefix, seg, pitch, kc, nmin, span);
      if (threadIdx.x == 0) {
        for (int m = 0; m < 3; ++m)
          for (int t = 0; t < 5; ++t) rec.q_lo[m][t] = kc > 0 ? (int)-(nmin[m] + (long long)prefix[m * 5 + t]) : 0;
        recs[(size_t)p * C + c] = rec;
      }
      __syncthreads();
      off += kc;
    }
  }
}

// Element `rank` (0 <= rank < k) of vals[0 .. k) sorted ascending, whose minimum is mn and range `span`: the passes of
// gs_sum_select for one target at any rank.  Block-cooperative (every thread returns the value); hist: GS_SUM_BINS
// shared counters.  The scratch writes it reads must be published by a barrier before the call.
__device__ long long gs_if_select1(unsigned *hist, const int *vals, long long k, long long mn, long long span, long long rank) {
  __shared__ unsigned long long pre;
  __shared__ long long rk;
  const int passes = gs_sum_passes((unsigned long long)span);
  if (threadIdx.x == 0) { pre = 0; rk = rank; }
  for (int p = 0; p < passes; ++p) {
    const int shift = (passes - 1 - p) * 9;
    for (int i = threadIdx.x; i < GS_SUM_BINS; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const unsigned long long hp = pre;
    for (long long i = threadIdx.x; i < k; i += blockDim.x) {
      const unsigned long long u = (unsigned long long)((long long)vals[i] - mn);
      if ((u >> (shift + 9)) == hp) atomicAdd(&hist[(u >> shift) & (GS_SUM_BINS - 1)], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) { long long r = rk; const unsigned d = gs_sum_pick(hist, r); rk = r; pre = (hp << 9) | d; }
    __syncthreads();
  }
  const long long out = mn + (long long)pre;
  __syncthreads();                                          // every thread has read `pre` before a later call resets it
  return out;
}

// Interference statistics (gs_ifclass) of replicas first .. first + count - 1, one block per replica in turn
// (grid-stride), jobdist's steps over 2C groups, group = 2 * class + degraded: (1) per-group job counts and per-class
// clamped counts, kept in registers and block-reduced; (2) group offsets: a class's clean and degraded segments are
// adjacent; (3) every job's wait, turnaround, jct, a, o, e, gpus and preempt written to its group's segment of the
// scratch (GS_IF_ROWS rows of `pitch` ints per block) through warp-aggregated shared cursors; (4) per group: jobdist's
// fold of wait / turnaround / jct, then the fold of the other rows (sums, squares of a as sums of 32-bit halves,
// gpus * e as sums of 32-bit halves, minima, maxima), gs_sum_select over the three rows and, for the degraded group,
// the upper middle jct; (5) per class: gs_sum_select<1> and the upper middle over the a row of both segments.
template <class Src>
__global__ void __launch_bounds__(GS_SUM_THREADS) gs_if_jobs_kernel(Src src, int first, int count, GsJdCfg cfg, gs_ifclass *recs,
                                                                   int *scratch, long long pitch) {
  constexpr int NC = GS_JOBDIST_MAX_CLASSES, NG = 2 * NC;
  __shared__ unsigned hist[GS_SUM_TARGETS * GS_SUM_BINS];
  __shared__ unsigned long long prefix[GS_SUM_TARGETS];
  __shared__ long long grp_cnt[NG], cls_clamped[NC];
  __shared__ long long cursor[NG];
  __shared__ gs_ifclass rec;                                // thread 0's alone
  const int C = cfg.nclasses;
  const int lane = threadIdx.x & 31;
  int *vals = scratch + (size_t)blockIdx.x * GS_IF_ROWS * (size_t)pitch;
  for (int b = blockIdx.x; b < count; b += gridDim.x) {
    const int r = first + b;
    const long long k = src.finished(r);
    long long red[NG + NC];
#pragma unroll
    for (int e = 0; e < NG + NC; ++e) red[e] = 0;
    for (long long i = threadIdx.x; i < k; i += blockDim.x) {
      const GsIfDur d = src.if_at(r, src.order(r, i));
      const GsIfVal x = gs_if_value(d.original, d.actual);
      const int g = 2 * gs_jd_class(cfg.bounds, C - 1, d.gpus) + x.degraded;
#pragma unroll
      for (int u = 0; u < NG; ++u) {
        if (g == u) { red[u] += 1; red[NG + u / 2] += x.clamped; }
      }
    }
    gs_sum_block_vec<NG + NC, NG + NC, 0>(red);
    if (threadIdx.x < NG) {
      const int g = threadIdx.x;
      long long off = 0;
#pragma unroll
      for (int u = 0; u < NG; ++u) off += u < g ? red[u] : 0;
#pragma unroll
      for (int u = 0; u < NG; ++u) {
        if (u == g) { grp_cnt[g] = red[u]; if ((g & 1) == 0) cls_clamped[g / 2] = red[NG + u / 2]; }
      }
      cursor[g] = off;
    }
    __syncthreads();
    for (long long i0 = 0; i0 < k; i0 += blockDim.x) {     // (warp-uniform trip count: the shuffles see full warps)
      const long long i = i0 + threadIdx.x;
      const bool in = i < k;
      GsSumJob v;
      GsIfVal x;
      int g = -1;
      if (in) {
        const int j = src.order(r, i);
        const GsIfDur d = src.if_at(r, j);
        v = src.job_at(r, j);
        x = gs_if_value(d.original, d.actual);
        g = 2 * gs_jd_class(cfg.bounds, C - 1, d.gpus) + x.degraded;
      }
      const unsigned peers = __match_any_sync(0xffffffffu, g);
      const int head = __ffs(peers) - 1;
      long long base = 0;
      if (in && lane == head) base = atomicAdd((unsigned long long *)&cursor[g], (unsigned long long)__popc(peers));
      base = __shfl_sync(0xffffffffu, base, head);
      if (in) {
        const long long pos = base + __popc(peers & ((1u << lane) - 1u));
        vals[pos] = v.wait; vals[pitch + pos] = v.turn; vals[2 * pitch + pos] = v.jct;
        vals[3 * pitch + pos] = x.a; vals[4 * pitch + pos] = x.o; vals[5 * pitch + pos] = x.e;
        vals[6 * pitch + pos] = v.gpus; vals[7 * pitch + pos] = v.preempt;
      }
    }
    __syncthreads();
    long long off = 0;
    for (int c = 0; c < C; ++c) {
      const long long off_c = off;
      long long amin = 0x7fffffff, amax = -0x80000000ll;
      if (threadIdx.x == 0) { rec = gs_ifclass{}; rec.clamped = cls_clamped[c]; }
      for (int deg = 0; deg < 2; ++deg) {
        const long long kg = grp_cnt[2 * c + deg];
        const int *seg = vals + off;
        // wait, turnaround, jct: jobdist's sums, square halves, minima and maxima
        long long s[15] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0x7fffffff, 0x7fffffff, 0x7fffffff, -0x80000000ll, -0x80000000ll, -0x80000000ll};
        for (long long i = threadIdx.x; i < kg; i += blockDim.x) {
#pragma unroll
          for (int m = 0; m < 3; ++m) {
            const int v = seg[m * pitch + i];
            const unsigned long long sq = (unsigned long long)((long long)v * v);
            s[m] += v; s[3 + m] += (long long)(sq >> 32); s[6 + m] += (long long)(sq & 0xffffffffull);
            s[9 + m] = min(s[9 + m], (long long)v); s[12 + m] = max(s[12 + m], (long long)v);
          }
        }
        gs_sum_block_vec<15, 9, 3>(s);
        // preempt_sum, gpu_ticks_sum, preempted jobs, a sum, a^2 halves, o sum, e sum, (gpus * e) halves | a min | a max,
        // e max, preempt max
        long long t[14] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0x7fffffff, -0x80000000ll, 0, 0};
        for (long long i = threadIdx.x; i < kg; i += blockDim.x) {
          const int jct = seg[2 * pitch + i], a = seg[3 * pitch + i], o = seg[4 * pitch + i], e = seg[5 * pitch + i];
          const int gpus = seg[6 * pitch + i], pre = seg[7 * pitch + i];
          const unsigned long long sq = (unsigned long long)((long long)a * a);
          const unsigned long long lost = (unsigned long long)((long long)gpus * e);
          t[0] += pre; t[1] += (long long)gpus * jct; t[2] += pre > 1;
          t[3] += a; t[4] += (long long)(sq >> 32); t[5] += (long long)(sq & 0xffffffffull);
          t[6] += o; t[7] += e; t[8] += (long long)(lost >> 32); t[9] += (long long)(lost & 0xffffffffull);
          t[10] = min(t[10], (long long)a); t[11] = max(t[11], (long long)a); t[12] = max(t[12], (long long)e);
          t[13] = max(t[13], (long long)pre);
        }
        gs_sum_block_vec<14, 10, 1>(t);
        amin = min(amin, t[10]); amax = max(amax, t[11]);
        long long span = 0;
#pragma unroll
        for (int m = 0; m < 3; ++m) span = max(span, s[12 + m] - s[9 + m]);
        gs_sum_select(hist, prefix, seg, pitch, kg, s + 9, span);
        if (threadIdx.x == 0) {
          gs_jclass &J = deg ? rec.degraded : rec.clean;
          J.jobs = kg; J.wait_sum = s[0]; J.turnaround_sum = s[1]; J.jct_sum = s[2]; J.preempt_sum = t[0]; J.gpu_ticks_sum = t[1];
          gs_sum_add128(J.wait_sq_lo, J.wait_sq_hi, ((gs_i128)s[3] << 32) + s[6]);
          gs_sum_add128(J.turnaround_sq_lo, J.turnaround_sq_hi, ((gs_i128)s[4] << 32) + s[7]);
          gs_sum_add128(J.jct_sq_lo, J.jct_sq_hi, ((gs_i128)s[5] << 32) + s[8]);
          for (int q = 0; q < 5; ++q) {
            J.wait_q[q] = kg > 0 ? (int)(s[9] + (long long)prefix[q]) : 0;
            J.turnaround_q[q] = kg > 0 ? (int)(s[10] + (long long)prefix[5 + q]) : 0;
            J.jct_q[q] = kg > 0 ? (int)(s[11] + (long long)prefix[10 + q]) : 0;
          }
          rec.preempted_jobs += t[2];
          rec.actual_sum += t[3];
          gs_sum_add128(rec.actual_sq_lo, rec.actual_sq_hi, ((gs_i128)t[4] << 32) + t[5]);
          rec.original_sum += t[6];
          if (deg) {
            rec.excess_sum = t[7];
            rec.excess_max = kg > 0 ? (int)t[12] : 0;
            gs_sum_add128(rec.lost_gpu_time_lo, rec.lost_gpu_time_hi, ((gs_i128)t[8] << 32) + t[9]);
            rec.degraded_jct_mid[0] = J.jct_q[0];                // rank floor((k - 1) / 2): gs_summary's 50 % rank
          }
          rec.preempt_max = kg > 0 && t[13] > rec.preempt_max ? (int)t[13] : rec.preempt_max;
        }
        __syncthreads();                                    // thread 0 has read prefix before the next select
        if (deg && kg > 0) {                                // (block-uniform)
          const long long hi = gs_if_select1(hist, seg + 2 * pitch, kg, s[11], s[14] - s[11], kg / 2);
          if (threadIdx.x == 0) rec.degraded_jct_mid[1] = (int)hi;
        }
        off += kg;
      }
      const long long kc = off - off_c;
      const int *arow = vals + 3 * pitch + off_c;
      gs_sum_select<1>(hist, prefix, arow, pitch, kc, &amin, amax - amin);
      if (threadIdx.x == 0)
        for (int q = 0; q < 5; ++q) rec.actual_q[q] = kc > 0 ? (int)(amin + (long long)prefix[q]) : 0;
      __syncthreads();
      if (kc > 0) {
        const long long hi = gs_if_select1(hist, arow, kc, amin, amax - amin, kc / 2);
        if (threadIdx.x == 0) { rec.actual_mid[0] = rec.actual_q[0]; rec.actual_mid[1] = (int)hi; }
      }
      if (threadIdx.x == 0) recs[(size_t)r * C + c] = rec;
      __syncthreads();
    }
  }
}

}  // namespace
#endif  // __CUDACC__

// TEST INFRASTRUCTURE -- host build of the __host__ __device__ part of gpuschedule_b200/csrc/gs_summary.cuh.
//
// The row fold, the closed-form fold of the fifo engine's compact records and the rank / radix-digit arithmetic of
// the job part are compiled here with g++, exactly as the kernels use them, so that tests/test_summary_cpu.py can
// check them against a numpy summary of rows and job records on a box without a GPU.  The loops around them are the
// serial counterparts of the kernels' block loops.  Built into a temporary directory by the test; the package never
// loads it.
#include <cstring>
#include <vector>

#include "gs_summary.cuh"

// rows (and the sampled utilisation values, or NULL) folded into *acc; makespan = `delta` of the last row
extern "C" void emu_sum_rows(const gs_tick_row *rows, const double *util, long long n, gs_summary *acc) {
  GsSumPart p;
  gs_sum_zero(p);
  for (long long i = 0; i < n; ++i) gs_sum_row(p, rows[i], util ? util[i] : 0.0);
  gs_sum_add_rows(*acc, p);
  if (n > 0) acc->makespan = rows[n - 1].now;
}

// one window of fifo records folded into *acc from its watermark (acc->rows): what gs_sum_rows_kernel does
extern "C" void emu_sum_compact(const gs_evrow *ev, long long nev, const gs_qrow *qr, long long nq, long long row_first,
                                long long ticks, gs_summary *acc) {
  const long long wm = acc->rows;
  GsSumPart p;
  gs_sum_zero(p);
  long long qi = 0;
  for (long long k = 0; k < nev; ++k) {
    const gs_evrow &e = ev[k];
    const long long t_last = k + 1 < nev ? (long long)ev[k + 1].now - 1 : ticks;
    const long long v_lo = e.now > wm + 1 ? e.now : wm + 1;
    long long arrive_sum = 0;
    int oldest = 0;
    if (e.queued > 0) {
      while (qi < nq && qr[qi].now < e.now) ++qi;
      if (qi < nq && qr[qi].now == e.now) { arrive_sum = qr[qi].arrive_sum; oldest = qr[qi].oldest_arrive; }
    }
    gs_sum_record(p, e, arrive_sum, oldest, v_lo, t_last);
  }
  const long long lo = wm > row_first ? wm : row_first;
  if (ticks > lo) {
    gs_sum_add_rows(*acc, p);
    acc->makespan = ticks;
  }
}

// job part of k finished jobs (columns in finish order)
extern "C" void emu_sum_jobs(const int *arrive, const int *start, const int *end, const int *jct, const int *preempt,
                             const int *gpus, long long k, gs_summary *acc) {
  std::vector<GsSumJob> jobs((size_t)k);
  for (long long i = 0; i < k; ++i) jobs[(size_t)i] = gs_sum_job(arrive[i], start[i], end[i], jct[i], preempt[i], gpus[i]);
  gs_sum_jobs_serial(jobs.data(), k, *acc);
}

// fifo's job.csv run length for a job (max of the duration after network cost and the input duration)
extern "C" int emu_sum_run_length(double dur) { return gs_sum_run_length(dur); }

extern "C" void emu_sum_select(const int *v, long long k, int *out) { gs_sum_select_serial(v, k, out); }

extern "C" long long emu_sum_rank(int permille, long long k) { return gs_sum_rank(permille, k); }

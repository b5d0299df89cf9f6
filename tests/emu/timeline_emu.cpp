// TEST INFRASTRUCTURE -- host build of the timeline part of gpuschedule_b200/csrc/gs_summary.cuh.
//
// The bin key, the per-bin folds of rows and of the fifo engine's compact records (a record split at bin boundaries
// with gs_sum_record on each clipped range) and the serial row fold are compiled here with g++, exactly as the kernels
// use them.  The loops around them are serial restatements of gs_tl_fold_rows / gs_tl_fold_records: the same pass
// that finds each bin's first row (record) and queue-record count, then one partial per bin -- so that
// tests/test_timeline_cpu.py can check the kernels' range logic against a numpy binning on a box without a GPU.
// Built into a temporary directory by the test; the package never loads it.
#include <vector>

#include "gs_summary.cuh"

// rows lo .. hi - 1 into bins: the kernel's warp-per-bin ranges when `delta` never decreases, its serial fold otherwise
extern "C" int emu_tl_rows(const gs_tick_row *rows, const double *util, long long lo, long long hi, long long W, int B, gs_tbin *bins) {
  for (long long i = lo + 1; i < hi; ++i)
    if (rows[i].now < rows[i - 1].now) { gs_tl_fold_rows_serial(bins, B, W, rows, util, 0, lo, hi); return 1; }
  std::vector<long long> start((size_t)B + 1, hi);
  for (long long i = lo; i < hi; ++i) {
    const int k = gs_tl_bin(rows[i].now, W, B), kp = i > lo ? gs_tl_bin(rows[i - 1].now, W, B) : -1;
    for (int b = kp + 1; b <= k; ++b) start[(size_t)b] = i;
  }
  for (int b = 0; b < B; ++b) {
    if (start[(size_t)b] >= start[(size_t)b + 1]) continue;
    GsTlPart p;
    gs_tl_zero(p);
    for (long long i = start[(size_t)b]; i < start[(size_t)b + 1]; ++i) gs_tl_row(p, rows[i], util ? util[i] : 0.0, i);
    gs_tl_add(bins[b], p);
  }
  return 0;
}

// the serial fold alone (any order of `delta`)
extern "C" void emu_tl_rows_serial(const gs_tick_row *rows, const double *util, long long lo, long long hi, long long W, int B, gs_tbin *bins) {
  gs_tl_fold_rows_serial(bins, B, W, rows, util, 0, lo, hi);
}

// one window of fifo records with the rows up to `delta` = wm already folded: gs_tl_fold_records
extern "C" void emu_tl_compact(const gs_evrow *ev, int nev, const gs_qrow *qr, int nq, long long ticks, long long wm, long long W, int B,
                               gs_tbin *bins) {
  if (ticks <= wm || nev == 0) return;
  auto t_last = [&](int k) -> long long { return k + 1 < nev ? (long long)ev[k + 1].now - 1 : ticks; };
  int k0 = 0;
  while (k0 < nev - 1 && t_last(k0) <= wm) ++k0;
  std::vector<int> start((size_t)B + 1, nev), qstart((size_t)B + 1, 0);
  int qcount = 0;
  for (int k = 0; k < nev; ++k) {
    if (k >= k0) {
      const int kh = gs_tl_bin(t_last(k), W, B), kp = k > k0 ? gs_tl_bin(t_last(k - 1), W, B) : -1;
      for (int b = kp + 1; b <= kh; ++b) { start[(size_t)b] = k; qstart[(size_t)b] = qcount; }
    }
    qcount += ev[k].queued > 0;
  }
  for (int b = 0; b < B; ++b) {
    const int s = start[(size_t)b];
    if (s >= nev) continue;
    const int e = start[(size_t)b + 1] < nev - 1 ? start[(size_t)b + 1] : nev - 1;
    const long long b_lo = (long long)b * W, b_hi = b == B - 1 ? 0x7fffffffffffffffll : ((long long)b + 1) * W - 1;
    GsTlPart p;
    gs_tl_zero(p);
    int qi = qstart[(size_t)b];
    for (int k = s; k <= e; ++k) {
      const gs_evrow &rec = ev[k];
      long long v_lo = rec.now > wm + 1 ? (long long)rec.now : wm + 1;
      v_lo = v_lo > b_lo ? v_lo : b_lo;
      const long long tl = t_last(k), v_hi = tl < b_hi ? tl : b_hi;
      long long arrive_sum = 0; int oldest = 0;
      if (rec.queued > 0) {
        int q = qi;
        if (q >= nq || qr[q].now != rec.now) { q = 0; while (q < nq - 1 && qr[q].now < rec.now) ++q; }
        arrive_sum = qr[q].arrive_sum; oldest = qr[q].oldest_arrive;
        ++qi;
      }
      gs_tl_record(p, rec, arrive_sum, oldest, v_lo, v_hi);
    }
    gs_tl_add(bins[b], p);
  }
}

extern "C" int emu_tl_bin(long long delta, long long W, int B) { return gs_tl_bin(delta, W, B); }

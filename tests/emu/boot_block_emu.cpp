// TEST INFRASTRUCTURE -- host build of the blocked path of gpuschedule_b200/csrc/gs_boot.cuh (gs_boot_kernel<true>).
//
// The per-job helpers (gs_boot_pick_blocked, gs_boot_block_key, gs_boot_block_row, gs_boot_block_gap, gs_boot_arrive)
// are compiled here with g++, and the loop around them restates the kernel's chunked structure: chunks of
// GS_BOOT_THREADS jobs, each scanned as warps of 32 lanes (the shuffle-up steps, all lanes reading the previous step's
// values), then across the warp totals, with the packed max-key carry and the gap-sum carry between chunks.  So
// tests/test_boot_block_cpu.py can compare its traces with tracegen.bootstrap_packed(..., block_len=L) on a box
// without a GPU.  Built into a temporary directory by the test; the package never loads it.
#include <algorithm>
#include <vector>

#include "gs_boot.cuh"

namespace {

const int kThreads = GS_BOOT_THREADS, kWarps = GS_BOOT_THREADS / 32;

// inclusive scan of every warp of one chunk with __shfl_up_sync's steps; returns the warp totals (lane 31)
template <class Op>
std::vector<long long> warp_scan(std::vector<long long> &x, Op op) {
  for (int o = 1; o < 32; o <<= 1) {
    const std::vector<long long> y = x;                // every lane reads the values of the previous step
    for (int t = 0; t < kThreads; ++t)
      if ((t & 31) >= o) x[(size_t)t] = op(x[(size_t)t], y[(size_t)(t - o)]);
  }
  std::vector<long long> tot(kWarps);
  for (int w = 0; w < kWarps; ++w) tot[(size_t)w] = x[(size_t)(32 * w + 31)];
  return tot;
}

}  // namespace

// Blocked replica (seed, stream, mean block length L) of n jobs from the K population records into out[n], the
// source rows into rows_out[n]; spans_out / last_out receive the sum of min(tasks, M) and the last arrival tick.
// Returns -1 (and writes nothing) when the last arrival could reach 2^31 - 1.
extern "C" int emu_boot_block_trace(const gs_jobin *pop, long long K, unsigned long long seed, unsigned long long stream, long long n,
                                    int gap_num, int gap_den, unsigned L, int M, gs_jobin *out, long long *rows_out,
                                    long long *spans_out, long long *last_out) {
  std::vector<int> gaps((size_t)(K > 1 ? K - 1 : 1), 0);
  long long max_gap = 0;
  for (long long i = 0; i + 1 < K; ++i) {
    gaps[(size_t)i] = pop[i + 1].arrive_tick - pop[i].arrive_tick;
    max_gap = gaps[(size_t)i] > max_gap ? gaps[(size_t)i] : max_gap;
  }
  if (gs_boot_arrive_bound(n, max_gap, gap_num, gap_den) >= 0x7fffffffll) return -1;
  long long carry = 0, key_carry = 0, spans = 0, last = 0;
  std::vector<long long> key((size_t)kThreads), g((size_t)kThreads), row((size_t)kThreads);
  for (long long j0 = 0; j0 < n; j0 += kThreads) {
    std::vector<char> start((size_t)kThreads, 0);
    std::vector<long long> gi((size_t)kThreads, -1);
    for (int t = 0; t < kThreads; ++t) {
      const long long j = j0 + t;
      long long s = 0;
      if (j < n) start[(size_t)t] = gs_boot_pick_blocked(seed, stream, j, K, L, s, gi[(size_t)t]);
      key[(size_t)t] = gs_boot_block_key(start[(size_t)t] != 0, j, s);
    }
    const auto mx = [](long long a, long long b) { return std::max(a, b); };
    std::vector<long long> tot = warp_scan(key, mx);
    long long chunk_key = key_carry;
    for (int t = 0; t < kThreads; ++t) {
      long long before = key_carry;
      for (int w = 0; w < t / 32; ++w) before = std::max(before, tot[(size_t)w]);
      key[(size_t)t] = std::max(key[(size_t)t], before);
    }
    for (int w = 0; w < kWarps; ++w) chunk_key = std::max(chunk_key, tot[(size_t)w]);
    key_carry = chunk_key;
    for (int t = 0; t < kThreads; ++t) {
      const long long j = j0 + t;
      g[(size_t)t] = 0;
      if (j >= n) continue;
      row[(size_t)t] = gs_boot_block_row(key[(size_t)t], j, K);
      const long long gj = gs_boot_block_gap(start[(size_t)t] != 0, row[(size_t)t], gi[(size_t)t]);
      if (gj >= 0) g[(size_t)t] = gaps[(size_t)gj];
    }
    tot = warp_scan(g, [](long long a, long long b) { return a + b; });
    long long chunk = 0;
    for (int w = 0; w < kWarps; ++w) chunk += tot[(size_t)w];
    for (int t = 0; t < kThreads && j0 + t < n; ++t) {
      long long before = carry;
      for (int w = 0; w < t / 32; ++w) before += tot[(size_t)w];
      const gs_jobin &p = pop[row[(size_t)t]];
      gs_jobin r;
      r.arrive_tick = gs_boot_arrive(before + g[(size_t)t], gap_num, gap_den);
      r.gpus = p.gpus; r.gpu_per_task = p.gpu_per_task; r.ps_count = 0; r.mem_bytes = p.mem_bytes; r.duration = p.duration;
      out[j0 + t] = r;
      rows_out[j0 + t] = row[(size_t)t];
      const long long tasks = p.gpus / p.gpu_per_task;
      spans += tasks < M ? tasks : M;
      last = r.arrive_tick;
    }
    carry += chunk;
  }
  *spans_out = spans;
  *last_out = last;
  return 0;
}

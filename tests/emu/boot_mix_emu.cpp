// TEST INFRASTRUCTURE -- host build of the mixed paths of gpuschedule_b200/csrc/gs_boot.cuh (gs_boot_kernel<*, true>).
//
// The alias tables come from the library's own host builder (gs_boot_alias_build, what gs_boot_mixes runs), and the
// per-job helpers (gs_boot_pick_mixed, gs_boot_alias_pick, gs_boot_block_key, gs_boot_block_row, gs_boot_block_gap,
// gs_boot_arrive) are compiled here with g++.  The loop around them restates the kernel's chunked structure: chunks of
// GS_BOOT_THREADS jobs, each scanned as warps of 32 lanes (the shuffle-up steps, all lanes reading the previous step's
// values), then across the warp totals, with the packed max-key carry (blocked instantiation only) and the gap-sum carry
// between chunks.  So tests/test_boot_mix_cpu.py can compare its traces with tracegen.bootstrap_packed(..., weights=w)
// on a box without a GPU.  Built into a temporary directory by the test; the package never loads it.
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

// The alias table of K weights into U[K], A[K]; returns T (0: all weights 0, nothing written).
extern "C" unsigned long long emu_boot_alias_build(const unsigned *w, long long K, unsigned long long *U, long long *A) {
  std::vector<GsBootAlias> tab((size_t)K);
  const uint64_t T = gs_boot_alias_build(w, K, tab.data());
  if (T == 0) return 0;
  for (long long i = 0; i < K; ++i) { U[i] = tab[(size_t)i].u; A[i] = (long long)tab[(size_t)i].a; }
  return T;
}

// Mixed replica (seed, stream, mean block length L, weights w[K]; w NULL: the unweighted replica of a mixed launch,
// T = 0) of n jobs from the K population records into out[n], the source rows into rows_out[n]; spans_out / last_out
// receive the sum of min(tasks, M) and the last arrival tick.  blocked = 0 runs the iid instantiation (L must be 1),
// 1 the blocked one.  Returns -1 (and writes nothing) when the last arrival could reach 2^31 - 1 or the weights sum
// to 0.
extern "C" int emu_boot_mix_trace(const gs_jobin *pop, long long K, const unsigned *w, unsigned long long seed, unsigned long long stream,
                                  long long n, int gap_num, int gap_den, unsigned L, int blocked, int M, gs_jobin *out, long long *rows_out,
                                  long long *spans_out, long long *last_out) {
  std::vector<int> gaps((size_t)(K > 1 ? K - 1 : 1), 0);
  long long max_gap = 0;
  for (long long i = 0; i + 1 < K; ++i) {
    gaps[(size_t)i] = pop[i + 1].arrive_tick - pop[i].arrive_tick;
    max_gap = gaps[(size_t)i] > max_gap ? gaps[(size_t)i] : max_gap;
  }
  if (gs_boot_arrive_bound(n, max_gap, gap_num, gap_den) >= 0x7fffffffll) return -1;
  std::vector<GsBootAlias> tab((size_t)K);
  uint64_t T = 0;
  if (w && (T = gs_boot_alias_build(w, K, tab.data())) == 0) return -1;
  long long carry = 0, key_carry = 0, spans = 0, last = 0;
  std::vector<long long> key((size_t)kThreads), g((size_t)kThreads), row((size_t)kThreads);
  for (long long j0 = 0; j0 < n; j0 += kThreads) {
    std::vector<char> start((size_t)kThreads, 0);
    std::vector<long long> gi((size_t)kThreads, -1), s((size_t)kThreads, 0);
    for (int t = 0; t < kThreads; ++t) {
      const long long j = j0 + t;
      if (j < n) start[(size_t)t] = gs_boot_pick_mixed(seed, stream, j, K, blocked ? L : 1u, tab.data(), T, s[(size_t)t], gi[(size_t)t]);
      key[(size_t)t] = gs_boot_block_key(start[(size_t)t] != 0, j, s[(size_t)t]);
    }
    if (blocked) {
      const std::vector<long long> tot = warp_scan(key, [](long long a, long long b) { return std::max(a, b); });
      long long chunk_key = key_carry;
      for (int t = 0; t < kThreads; ++t) {
        long long before = key_carry;
        for (int wp = 0; wp < t / 32; ++wp) before = std::max(before, tot[(size_t)wp]);
        key[(size_t)t] = std::max(key[(size_t)t], before);
      }
      for (int wp = 0; wp < kWarps; ++wp) chunk_key = std::max(chunk_key, tot[(size_t)wp]);
      key_carry = chunk_key;
    }
    for (int t = 0; t < kThreads; ++t) {
      const long long j = j0 + t;
      g[(size_t)t] = 0;
      if (j >= n) continue;
      long long gj = gi[(size_t)t];
      row[(size_t)t] = s[(size_t)t];
      if (blocked) {
        row[(size_t)t] = gs_boot_block_row(key[(size_t)t], j, K);
        gj = gs_boot_block_gap(start[(size_t)t] != 0, row[(size_t)t], gi[(size_t)t]);
      }
      if (gj >= 0) g[(size_t)t] = gaps[(size_t)gj];
    }
    const std::vector<long long> tot = warp_scan(g, [](long long a, long long b) { return a + b; });
    long long chunk = 0;
    for (int wp = 0; wp < kWarps; ++wp) chunk += tot[(size_t)wp];
    for (int t = 0; t < kThreads && j0 + t < n; ++t) {
      long long before = carry;
      for (int wp = 0; wp < t / 32; ++wp) before += tot[(size_t)wp];
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

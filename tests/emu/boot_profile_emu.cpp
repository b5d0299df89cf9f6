// TEST INFRASTRUCTURE -- host build of the profiled paths of gpuschedule_b200/csrc/gs_boot.cuh (the profiled
// gs_boot_kernel instantiations).
//
// The host conversion (gs_boot_profile_invalid, gs_boot_profile_base), the arrival rule (gs_boot_profile_seg,
// gs_boot_profile_arrive) and the exact bound (gs_boot_profile_bound) are the library's own, compiled here with g++, as
// are the per-job helpers of the other instantiations.  The loop around them restates the kernel's chunked structure:
// chunks of GS_BOOT_THREADS jobs, each scanned as warps of 32 lanes (the shuffle-up steps, all lanes reading the
// previous step's values), then across the warp totals, with the packed max-key carry (blocked replicas only) and the
// gap-sum carry between chunks; a profiled job then looks up its segment in the replica's converted segments.  So
// tests/test_boot_profile_cpu.py can compare its traces with tracegen.bootstrap_packed(..., profile=...) on a box
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

// 0 when the profile (seg[m], period P) keeps the rules of gs_boot_profiles, else 1.
extern "C" int emu_boot_profile_invalid(const gs_boot_seg *seg, int m, int P) { return gs_boot_profile_invalid(seg, m, P) ? 1 : 0; }

// The device form of a valid profile: base starts s_out[m]; returns B (0 when P = 0).
extern "C" long long emu_boot_profile_base(const gs_boot_seg *seg, int m, int P, long long *s_out) {
  std::vector<GsBootProfSeg> d((size_t)m);
  const long long B = gs_boot_profile_base(seg, m, P, d.data());
  for (int k = 0; k < m; ++k) s_out[k] = d[(size_t)k].s;
  return B;
}

// Arrival ticks out[i] of the base times S[i] in int64 (the device's arithmetic).
extern "C" void emu_boot_profile_arrive(const gs_boot_seg *seg, int m, int P, const long long *S, long long cnt, long long *out) {
  std::vector<GsBootProfSeg> d((size_t)m);
  const long long B = gs_boot_profile_base(seg, m, P, d.data());
  for (long long i = 0; i < cnt; ++i) out[i] = gs_boot_profile_arrive<long long>(d.data(), m, P, B, S[i]);
}

// The exact bound arrive((n - 1) * max_gap), saturated at 2^63 - 1.
extern "C" long long emu_boot_profile_bound(const gs_boot_seg *seg, int m, int P, long long n, long long max_gap) {
  std::vector<GsBootProfSeg> d((size_t)m);
  const long long B = gs_boot_profile_base(seg, m, P, d.data());
  return gs_boot_profile_bound(d.data(), m, P, B, n, max_gap);
}

// Replica (seed, stream, mean block length L, weights w[K] or NULL, profile seg[m] with period P, or m = 0 for none)
// of n jobs from the K population records into out[n]; spans_out / last_out receive the sum of min(tasks, M) and
// the last arrival tick.  blocked = 0 runs the iid instantiation (L must be 1), 1 the blocked one.  A profiled
// replica uses the gap scale 1 / 1.  Returns -1 (and writes nothing) when the last arrival could reach 2^31 - 1 or
// the weights sum to 0.
extern "C" int emu_boot_profile_trace(const gs_jobin *pop, long long K, const unsigned *w, const gs_boot_seg *seg, int m, int P,
                                      unsigned long long seed, unsigned long long stream, long long n, int gap_num, int gap_den, unsigned L,
                                      int blocked, int M, gs_jobin *out, long long *spans_out, long long *last_out) {
  std::vector<int> gaps((size_t)(K > 1 ? K - 1 : 1), 0);
  long long max_gap = 0;
  for (long long i = 0; i + 1 < K; ++i) {
    gaps[(size_t)i] = pop[i + 1].arrive_tick - pop[i].arrive_tick;
    max_gap = gaps[(size_t)i] > max_gap ? gaps[(size_t)i] : max_gap;
  }
  std::vector<GsBootProfSeg> pseg((size_t)(m > 0 ? m : 1));
  long long B = 0;
  if (m > 0) {
    B = gs_boot_profile_base(seg, m, P, pseg.data());
    if (gs_boot_profile_bound(pseg.data(), m, P, B, n, max_gap) >= 0x7fffffffll) return -1;
  } else if (gs_boot_arrive_bound(n, max_gap, gap_num, gap_den) >= 0x7fffffffll) {
    return -1;
  }
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
      const long long S = before + g[(size_t)t];
      gs_jobin r;
      r.arrive_tick = m > 0 ? (int)gs_boot_profile_arrive<long long>(pseg.data(), m, P, B, S) : gs_boot_arrive(S, gap_num, gap_den);
      r.gpus = p.gpus; r.gpu_per_task = p.gpu_per_task; r.ps_count = 0; r.mem_bytes = p.mem_bytes; r.duration = p.duration;
      out[j0 + t] = r;
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

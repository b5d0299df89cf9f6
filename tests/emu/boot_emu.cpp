// TEST INFRASTRUCTURE -- host build of the __host__ __device__ part of gpuschedule_b200/csrc/gs_boot.cuh.
//
// The Philox4x64-10 generator, the high-word multiply, the per-job pick and the arrival arithmetic are compiled here
// with g++, exactly as gs_boot_kernel uses them, so that tests/test_bootstrap_cpu.py can compare the traces they make
// with tracegen.bootstrap_packed on a box without a GPU.  The loop around them is the serial counterpart of the
// kernel's block loop (a running sum instead of the chunked block scan).  Built into a temporary directory by the
// test; the package never loads it.
#include <vector>

#include "gs_boot.cuh"

extern "C" unsigned long long emu_boot_mulhi(unsigned long long a, unsigned long long b) { return gs_boot_mulhi(a, b); }

extern "C" void emu_boot_philox(unsigned long long k0, unsigned long long k1, const unsigned long long *ctr, unsigned long long *out) {
  const GsPhilox b = gs_boot_philox(k0, k1, ctr[0], ctr[1], ctr[2], ctr[3]);
  for (int i = 0; i < 4; ++i) out[i] = b.w[i];
}

extern "C" long long emu_boot_arrive_bound(long long n, long long max_gap, int gap_num, int gap_den) {
  return gs_boot_arrive_bound(n, max_gap, gap_num, gap_den);
}

// Replica (seed, stream) of n jobs from the K population records into out[n]; spans_out / last_out receive the sum of
// min(tasks, M) and the last arrival tick.  Returns -1 (and writes nothing) when the last arrival could reach 2^31 - 1.
extern "C" int emu_boot_trace(const gs_jobin *pop, long long K, unsigned long long seed, unsigned long long stream, long long n,
                              int gap_num, int gap_den, int M, gs_jobin *out, long long *spans_out, long long *last_out) {
  std::vector<int> gaps((size_t)(K > 1 ? K - 1 : 1), 0);
  long long max_gap = 0;
  for (long long i = 0; i + 1 < K; ++i) {
    gaps[(size_t)i] = pop[i + 1].arrive_tick - pop[i].arrive_tick;
    max_gap = gaps[(size_t)i] > max_gap ? gaps[(size_t)i] : max_gap;
  }
  if (gs_boot_arrive_bound(n, max_gap, gap_num, gap_den) >= 0x7fffffffll) return -1;
  long long S = 0, spans = 0, last = 0;
  for (long long j = 0; j < n; ++j) {
    long long row, gi;
    gs_boot_pick(seed, stream, j, K, row, gi);
    S += gi >= 0 ? gaps[(size_t)gi] : 0;
    const gs_jobin &p = pop[row];
    gs_jobin r;
    r.arrive_tick = gs_boot_arrive(S, gap_num, gap_den);
    r.gpus = p.gpus; r.gpu_per_task = p.gpu_per_task; r.ps_count = 0; r.mem_bytes = p.mem_bytes; r.duration = p.duration;
    out[j] = r;
    const long long tasks = p.gpus / p.gpu_per_task;
    spans += tasks < M ? tasks : M;
    last = r.arrive_tick;
  }
  *spans_out = spans;
  *last_out = last;
  return 0;
}

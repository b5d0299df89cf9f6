// TEST INFRASTRUCTURE -- host build of the interference part of gpuschedule_b200/csrc/gs_summary.cuh.
//
// The fixed-point rule gs_if_fp, the per-job values gs_if_value and gs_if_serial (the kernel's per-group jobdist
// records, sums and order statistics, serially) are compiled here with g++, exactly as the host-emulation build of
// gs_horus.cu uses them, so that tests/test_interference_cpu.py can check them against a Python-int restatement on
// job sets the engine would rarely produce (all degraded, saturated durations, lost GPU time past 2^64).  Built into
// a temporary directory by the test; the package never loads it.
#include <cstddef>
#include <vector>

#include "gs_summary.cuh"

// sizeof(gs_ifclass), then the offsets of its fields in declaration order
extern "C" void emu_if_layout(long long *out) {
  const size_t v[] = {sizeof(gs_ifclass), offsetof(gs_ifclass, degraded), offsetof(gs_ifclass, clean), offsetof(gs_ifclass, actual_sum),
                      offsetof(gs_ifclass, actual_sq_lo), offsetof(gs_ifclass, actual_sq_hi), offsetof(gs_ifclass, original_sum),
                      offsetof(gs_ifclass, excess_sum), offsetof(gs_ifclass, lost_gpu_time_lo), offsetof(gs_ifclass, lost_gpu_time_hi),
                      offsetof(gs_ifclass, preempted_jobs), offsetof(gs_ifclass, clamped), offsetof(gs_ifclass, degraded_jct_mid),
                      offsetof(gs_ifclass, actual_q), offsetof(gs_ifclass, actual_mid), offsetof(gs_ifclass, excess_max),
                      offsetof(gs_ifclass, preempt_max), offsetof(gs_ifclass, reserved)};
  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) out[i] = (long long)v[i];
}

// fp(x) and whether it saturated
extern "C" int emu_if_fp(double x, int *clamped) {
  int c = 0;
  const int v = gs_if_fp(x, c);
  *clamped = c;
  return v;
}

// interference statistics of k finished jobs (columns in finish order); 0, or -1 when the bounds are refused or
// nclasses is 0 (nothing written)
extern "C" int emu_if_jobs(const int *arrive, const int *start, const int *end, const int *jct, const int *preempt, const int *gpus,
                           const double *original, const double *actual, long long k, int nclasses, const int *bounds, gs_ifclass *out) {
  GsJdCfg cfg;
  const char *why = nullptr;
  if (nclasses < 1 || !gs_jd_make_cfg(nclasses, bounds, 0, nullptr, cfg, &why)) return -1;
  std::vector<GsSumJob> jobs((size_t)k);
  std::vector<GsIfDur> durs((size_t)k);
  for (long long i = 0; i < k; ++i) {
    jobs[(size_t)i] = gs_sum_job(arrive[i], start[i], end[i], jct[i], preempt[i], gpus[i]);
    durs[(size_t)i] = GsIfDur{gpus[i], original[i], actual[i]};
  }
  gs_if_serial(jobs.data(), durs.data(), k, cfg, out);
  return 0;
}

// TEST INFRASTRUCTURE -- host build of the arrivals part of gpuschedule_b200/csrc/gs_summary.cuh.
//
// The setting's validation and gs_arr_serial (each arrival bin's finished jobs as one class of gs_sd_serial, with the
// arrival ticks as the key) are compiled here with g++, exactly as the host-emulation build of gs_horus.cu uses them,
// so that tests/test_arrivals_cpu.py can check them against a Python-int restatement on a box without a GPU.  Built
// into a temporary directory by the test; the package never loads it.
#include <vector>

#include "gs_summary.cuh"

extern "C" int emu_arr_bin(long long a, long long width, int nbins) { return gs_tl_bin(a, width, nbins); }

// the setting's validation alone: 0, or -1 when gs_set_arrivals would refuse it
extern "C" int emu_arr_check(long long width, int nbins, long long tau) {
  GsArrCfg cfg;
  const char *why = nullptr;
  return gs_arr_make_cfg(width, nbins, tau, cfg, &why) ? 0 : -1;
}

// arrival-bin statistics of k finished jobs (columns in finish order) of a trace of n jobs arriving at trace_arrive;
// 0, or -1 when the setting is refused or off (nothing written)
extern "C" int emu_arr_jobs(const int *arrive, const int *start, const int *end, const int *jct, const int *preempt, const int *gpus,
                            long long k, const int *trace_arrive, long long n, long long width, int nbins, long long tau, gs_abin *out) {
  GsArrCfg cfg;
  const char *why = nullptr;
  if (!gs_arr_make_cfg(width, nbins, tau, cfg, &why) || cfg.nbins == 0) return -1;
  std::vector<GsSumJob> jobs((size_t)k);
  for (long long i = 0; i < k; ++i) jobs[(size_t)i] = gs_sum_job(arrive[i], start[i], end[i], jct[i], preempt[i], gpus[i]);
  gs_arr_serial(jobs.data(), arrive, k, trace_arrive, n, cfg, out);
  return 0;
}

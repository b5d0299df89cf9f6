// TEST INFRASTRUCTURE -- host build of the slowdown part of gpuschedule_b200/csrc/gs_summary.cuh.
//
// The key, the class, the bounded slowdown, the setting's validation and gs_sd_serial (the kernel's count / scatter /
// fold / select steps run serially, with the summary's gs_sum_select_serial) are compiled here with g++, exactly as the
// kernel and the host-emulation build of gs_horus.cu use them, so that tests/test_slowdown_cpu.py can check them
// against a Python-int restatement on a box without a GPU.  Built into a temporary directory by the test; the package
// never loads it.
#include <vector>

#include "gs_summary.cuh"

extern "C" long long emu_sd_key(int key, int gpus, int jct) { return gs_sd_key(key, gpus, jct); }

extern "C" int emu_sd_class(const long long *bounds, int nb, long long key) { return gs_sd_class(bounds, nb, key); }

extern "C" int emu_sd_value(int turn, int jct, long long tau) { return gs_sd_value(turn, jct, tau); }

// the setting's validation alone: 0, or -1 when gs_set_slowdown would refuse it
extern "C" int emu_sd_check(const gs_slowdown_cfg *in) {
  GsSdCfg cfg;
  const char *why = nullptr;
  return gs_sd_make_cfg(in, cfg, &why) ? 0 : -1;
}

// slowdown statistics of k finished jobs (columns in finish order); 0, or -1 when the setting is refused or off
// (nothing written)
extern "C" int emu_sd_jobs(const int *arrive, const int *start, const int *end, const int *jct, const int *preempt, const int *gpus,
                           long long k, const gs_slowdown_cfg *in, gs_sdclass *out, uint32_t *hist) {
  GsSdCfg cfg;
  const char *why = nullptr;
  if (!gs_sd_make_cfg(in, cfg, &why) || cfg.nclasses == 0) return -1;
  std::vector<GsSumJob> jobs((size_t)k);
  for (long long i = 0; i < k; ++i) jobs[(size_t)i] = gs_sum_job(arrive[i], start[i], end[i], jct[i], preempt[i], gpus[i]);
  gs_sd_serial(jobs.data(), k, cfg, out, hist);
  return 0;
}

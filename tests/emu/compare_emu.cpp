// TEST INFRASTRUCTURE -- host build of the paired comparison of gpuschedule_b200/csrc/gs_summary.cuh.
//
// gs_cmp_pair_serial (the kernel's membership / count / scatter / fold / select steps run serially, with the summary's
// gs_sum_select_serial) is compiled here with g++, exactly as the host-emulation build of gs_horus.cu uses it, so that
// tests/test_compare_cpu.py can check it against a numpy restatement of gs_jpair's definition on a box without a GPU.
// Built into a temporary directory by the test; the package never loads it.
#include <vector>

#include "gs_summary.cuh"

// One pair over n jobs: per run, start / end / jct / preempt by trace index and the finish order; arrive and gpus are
// the shared trace's.  0, or -1 when the setting is refused or C = 0 (nothing written).
extern "C" int emu_cmp_pair(const int *arrive, const int *gpus, long long n,
                            const int *start_a, const int *end_a, const int *jct_a, const int *fin_a, long long ka,
                            const int *start_b, const int *end_b, const int *jct_b, const int *fin_b, long long kb,
                            int nclasses, const int *bounds, int nedges, const int *edges, gs_jpair *out, uint32_t *hist) {
  GsJdCfg cfg;
  const char *why = nullptr;
  if (!gs_jd_make_cfg(nclasses, bounds, nedges, edges, cfg, &why) || nclasses == 0) return -1;
  std::vector<GsSumJob> ja((size_t)n), jb((size_t)n);
  for (long long j = 0; j < n; ++j) {
    ja[(size_t)j] = gs_sum_job(arrive[j], start_a[j], end_a[j], jct_a[j], 0, gpus[j]);
    jb[(size_t)j] = gs_sum_job(arrive[j], start_b[j], end_b[j], jct_b[j], 0, gpus[j]);
  }
  gs_cmp_pair_serial(ja.data(), jb.data(), n, fin_a, ka, fin_b, kb, cfg, out, hist);
  return 0;
}

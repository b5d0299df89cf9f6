// TEST INFRASTRUCTURE -- host build of the jobdist part of gpuschedule_b200/csrc/gs_summary.cuh.
//
// The class key, the CDF bin, the setting's validation and gs_jd_jobs_serial (the kernel's count / scatter / fold /
// select steps run serially, with the summary's gs_sum_select_serial) are compiled here with g++, exactly as the
// kernels and the host-emulation build of gs_horus.cu use them, so that tests/test_jobdist_cpu.py can check them
// against a numpy breakdown of job records on a box without a GPU.  Built into a temporary directory by the test;
// the package never loads it.
#include <vector>

#include "gs_summary.cuh"

extern "C" int emu_jd_class(const int *bounds, int nb, int gpus) { return gs_jd_class(bounds, nb, gpus); }

extern "C" int emu_jd_bin(const int *edges, int E, int v) { return gs_jd_bin(edges, E, v); }

// jobdist of k finished jobs (columns in finish order); 0, or -1 when the setting is refused (nothing written)
extern "C" int emu_jd_jobs(const int *arrive, const int *start, const int *end, const int *jct, const int *preempt, const int *gpus,
                           long long k, int nclasses, const int *bounds, int nedges, const int *edges, gs_jclass *classes, uint32_t *hist) {
  GsJdCfg cfg;
  const char *why = nullptr;
  if (!gs_jd_make_cfg(nclasses, bounds, nedges, edges, cfg, &why) || nclasses == 0) return -1;
  std::vector<GsSumJob> jobs((size_t)k);
  for (long long i = 0; i < k; ++i) jobs[(size_t)i] = gs_sum_job(arrive[i], start[i], end[i], jct[i], preempt[i], gpus[i]);
  gs_jd_jobs_serial(jobs.data(), k, cfg, classes, hist);
  return 0;
}

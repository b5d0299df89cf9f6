// TEST INFRASTRUCTURE -- host build of the occupancy part of gpuschedule_b200/csrc/gs_summary.cuh.
//
// The serial folds gs_occ_serial (rows, with the carry of an event-driven run or one tick per row) and
// gs_occ_records_serial (the fifo engine's compact records past a watermark), and the check of a queue edge setting,
// compiled with g++ exactly as the kernels' host forms use them, so that tests/test_occupancy_cpu.py can compare them
// with a Python-int restatement on a box without a GPU.  Built into a temporary directory by the test.
#include "gs_summary.cuh"

static_assert(sizeof(GsOccCarry) == 24, "the test passes the carry as 24 bytes");

// 1 when the setting is valid (and cfg receives it), 0 otherwise
extern "C" int emu_occ_cfg(int nedges, const int *edges) {
  GsOccCfg cfg;
  const char *why = nullptr;
  return gs_occ_make_cfg(nedges, edges, cfg, &why) ? 1 : 0;
}

static GsOccCfg cfg_of(int nedges, const int *edges) {
  GsOccCfg cfg{};
  cfg.nedges = nedges;
  for (int i = 0; i < nedges; ++i) cfg.edges[i] = edges[i];
  return cfg;
}

// rows lo .. hi - 1 of rows[] into the record, carry and histograms (hall: [H_all, H_wait] of G + 1 each)
extern "C" void emu_occ_rows(gs_occ *o, GsOccCarry *c, unsigned long long *hall, unsigned long long *hq, int nedges, const int *edges,
                             const gs_tick_row *rows, long long lo, long long hi, int done, int per_tick, int G) {
  o->total_gpus = G;
  const GsOccHist H{hall, hall + G + 1, hq};
  gs_occ_serial(*o, *c, H, cfg_of(nedges, edges), rows, 0, lo, hi, done, per_tick);
}

// one window of fifo records with the rows up to `delta` = wm already folded
extern "C" void emu_occ_records(gs_occ *o, unsigned long long *hall, unsigned long long *hq, int nedges, const int *edges,
                                const gs_evrow *ev, int nev, long long ticks, long long wm, int G) {
  o->total_gpus = G;
  const GsOccHist H{hall, hall + G + 1, hq};
  gs_occ_records_serial(*o, H, cfg_of(nedges, edges), ev, nev, ticks, wm);
}

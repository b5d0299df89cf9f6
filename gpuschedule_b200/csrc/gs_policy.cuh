// gs_policy.cuh -- part of libgsched.so (single translation unit, included from gsched.cu).
// Event-driven policies: sjf / dlas / dlas-gpu / gittins (warp-cooperative kernels + thread-per-replica fallback).
#pragma once

// ------------------------------------------------------------------ event-driven policies
// sjf / dlas / dlas-gpu / gittins: restated from the reference's dead Tiresias-style loops
// (run_sim.py:162-287, 664-947, 949-1203; SURVEY appendix A.2-A.5); the decisions taken where
// that code is undefined are listed in oracle/policy_oracle.c, which this kernel matches
// bit for bit.  First version: ONE THREAD per replica (a warp carries 32 replicas); every
// event re-evaluates all runnable jobs (counter update, ordering, emptied-cluster greedy
// re-admission), exactly as the specification does.  Lists live in global memory.
__device__ __forceinline__ double git_lookup(const SimDev &S, double a) {
  // attained service is a whole number of (GPU) ticks: when the table's range is small enough the host tabulates the
  // answer for every integer up to the largest sample (gs_config_sim) and the bisection below -- 17 dependent loads into
  // a 1.6 MB table for a 100k-job trace -- becomes one load
  if (a >= 0.0 && a < (double)S.git_direct_n) {
    const int k = (int)a;
    if ((double)k == a) return S.git_direct[k];
  }
  const int n = S.git_n;
  if (n < 2 || a > S.git_data[n - 2]) return 0.0;
  int lo = 0, hi = n - 1;
  while (lo < hi) { int mid = (lo + hi) >> 1; if (S.git_data[mid] > a) hi = mid; else lo = mid + 1; }
  return S.git_index[lo];
}

__device__ __forceinline__ void plist_remove(int *v, int &n, int x) {
  int w = 0;
  for (int i = 0; i < n; ++i) { int e = v[i]; if (e != x) v[w++] = e; }
  n = w;
}

__device__ bool pol_yarn_place(const SimDev &S, int gpus, int gpc, bool placeable) {
  if (!placeable) return false;
  const int M = S.M, G = S.G, tasks = gpus / gpc;
  int *idle = S.cidle, *kfree = S.ckfree;
  if (gpus <= G) {
    for (int nd = 0; nd < M; ++nd)
      if (idle[nd] >= gpus && kfree[nd] >= tasks) { idle[nd] -= gpus; kfree[nd] -= tasks; return true; }
    return false;
  }
  int cum = 0, last = -1;
  for (int nd = 0; nd < M; ++nd) {
    int cap = min(idle[nd] / gpc, kfree[nd]);
    if (cap <= 0) continue;
    cum += cap;
    if (cum >= tasks) { last = nd; break; }
  }
  if (last < 0) return false;
  int rem = tasks;
  for (int nd = 0; nd <= last; ++nd) {
    int cap = min(idle[nd] / gpc, kfree[nd]);
    if (cap <= 0) continue;
    int take = min(cap, rem);
    idle[nd] -= take * gpc; kfree[nd] -= take; rem -= take;
  }
  return true;
}

__global__ void __launch_bounds__(32) gs_policy_kernel(SimDev *sims, int nsims, long long max_ticks, int take_dlas) {
  const int sim = blockIdx.x * blockDim.x + threadIdx.x;
  if (sim >= nsims) return;
  SimDev &S = sims[sim];
  if (S.policy == GS_SCHED_FIFO || S.done || S.status != 0) return;
  if (!take_dlas) return;   // every event-driven policy has a warp-cooperative kernel; this one is the fallback (engine mode 2)
  const int policy = S.policy, n = S.n, M = S.M, G = S.G, K = S.K;
  const bool is_dlas = policy == GS_SCHED_DLAS || policy == GS_SCHED_DLAS_GPU;
  const bool gputime = policy == GS_SCHED_DLAS_GPU || policy == GS_SCHED_GITTINS;
  const int nq = is_dlas ? S.num_queue : 1;
  const JobIn *__restrict__ jobs = S.jobs;
  PJob *pj = S.pj;
  int *runnable = S.runnable, *endj = S.endj, *tmpl = S.tmpl;
  gs_job_rec *rec = S.rec;
  const long long cap_bytes = S.cap_bytes, fit_limit = S.fit_limit;
  const int total_gpus = M * G;
  int p = S.p, rn = S.rn, en = S.en, end_time = S.end_time, next_job_jump = S.next_job_jump, nfin = S.finished;
  int stale_n = S.stale_n;
  double next_git = S.next_gittins_unit;
  long long events = S.events, ticks = S.ticks;
  const long long row_first = ticks;
  long long budget = max_ticks > 0 ? max_ticks : 0x7fffffffffffffffLL;
  int status = 0;
  bool done = false;

  while (budget > 0 && (ticks - row_first) < S.rows_cap) {
    if (!((n - p) + rn > 0)) { done = true; break; }
    if (p >= n && end_time == 0x7fffffff) { done = true; break; }     // "cluster is not large enough"
    const int start_time = p < n ? jobs[p].arrive : 0x7fffffff;
    int event_time; bool has_start = false, has_end = false;
    const int *elist = endj; int ecount = en;
    if (end_time < start_time) { event_time = end_time; has_end = true; }
    else if (end_time > start_time) { event_time = start_time; has_start = true; }
    else {                      // tie: the start event inherits this end list (quirk Q25, run_sim.py:708-710)
      event_time = start_time; has_start = has_end = true;
      for (int i = 0; i < en; ++i) S.stalej[i] = endj[i];
      stale_n = en;
    }
    bool jumped = false;
    if (is_dlas && event_time > next_job_jump) { event_time = next_job_jump; jumped = true; }
    if (policy == GS_SCHED_GITTINS && (double)event_time > next_git) { event_time = (int)next_git; jumped = true; }
    if (jumped) has_start = has_end = false;       // the start event keeps the inherited list
    else if (has_start) {                          // the start event is consumed: an inherited list completes here
      if (stale_n > 0) { elist = S.stalej; ecount = stale_n; has_end = true; }
      stale_n = 0;
    }
    if (has_end) {
      for (int i = 0; i < ecount; ++i) {
        const int j = elist[i];
        PJob &r = pj[j];
        r.status = PST_END;
        gs_job_rec o; o.start = r.start; o.end = event_time;
        double cl = ceil(jobs[j].dur); o.jct = cl < 1.0 ? 1 : (int)cl; o.preempt = r.resume; o.duration = jobs[j].dur;
        rec[j] = o;
        S.fin[nfin++] = j; ++events;
        plist_remove(runnable, rn, j);
        plist_remove(S.queues + (size_t)r.q_id * n, S.qn[r.q_id], j);
      }
    }
    if (has_start) {
      while (p < n && jobs[p].arrive == event_time) {
        const int j = p++;
        PJob r; r.last_check = event_time; r.total_exec = 0; r.exec = 0; r.pending = 0; r.last_pending = 0; r.start = -1;
        r.resume = 0; r.status = PST_PENDING; r.q_id = 0; r.pad0 = 0; r.pad1 = 0;
        pj[j] = r;
        runnable[rn++] = j; S.queues[S.qn[0]++] = j; ++events;
      }
    }
    for (int i = 0; i < rn; ++i) {
      const int j = runnable[i];
      PJob &r = pj[j];
      const int dt = event_time - r.last_check;
      r.last_check = event_time;
      if (r.status == PST_RUNNING) {
        r.total_exec += dt; r.exec += dt;
        if (is_dlas) {
          const double j_gt = gputime ? (double)r.exec * jobs[j].gpus : (double)r.exec;
          if (r.q_id < nq - 1 && j_gt >= S.queue_limit[r.q_id]) {
            plist_remove(S.queues + (size_t)r.q_id * n, S.qn[r.q_id], j);
            r.q_id += 1;
            S.queues[(size_t)r.q_id * n + S.qn[r.q_id]++] = j;
          }
        }
      } else {
        r.pending += dt;
        if (r.exec > 0) r.last_pending += dt;
      }
    }
    // ---- order, empty the cluster, greedy re-admission
    int nrun = 0, npre = 0, busy = 0;
    long long mem_busy = 0;
    int *run_jobs = tmpl, *pre_jobs = tmpl + (n > 0 ? n - 1 : 0);
    if (policy == GS_SCHED_SJF) {
      for (int i = 1; i < rn; ++i) {          // stable insertion sort by num_gpu (list is nearly sorted)
        const int x = runnable[i]; const int kx = jobs[x].gpus; int k = i;
        while (k > 0 && jobs[runnable[k - 1]].gpus > kx) { runnable[k] = runnable[k - 1]; --k; }
        runnable[k] = x;
      }
      for (int nd = 0; nd < M; ++nd) { S.cidle[nd] = G; S.ckfree[nd] = K; }
      for (int i = 0; i < rn; ++i) {
        const int j = runnable[i];
        const JobIn jr = jobs[j];
        PJob &r = pj[j];
        if (pol_yarn_place(S, jr.gpus, jr.gpc, jr.memb < fit_limit)) {
          if (r.start < 0) r.start = event_time;
          if (r.status == PST_PENDING) run_jobs[nrun++] = j;
          busy += jr.gpus; mem_busy += (long long)jr.gpus * (jr.memb < cap_bytes ? jr.memb : cap_bytes);
        } else if (r.status == PST_RUNNING) { pre_jobs[-(npre++)] = j; }
      }
    } else {
      if (policy == GS_SCHED_GITTINS) {       // stable insertion sort by rank, ascending
        double *rk = reinterpret_cast<double *>(S.queues);     // gittins has no queues: reuse as rank scratch
        for (int i = 0; i < rn; ++i) {
          const int j = runnable[i]; const PJob &r = pj[j];
          rk[i] = git_lookup(S, r.status == PST_RUNNING ? (double)r.exec * jobs[j].gpus : (double)r.exec);
        }
        for (int i = 1; i < rn; ++i) {
          const int x = runnable[i]; const double kx = rk[i]; int k = i;
          while (k > 0 && rk[k - 1] > kx) { runnable[k] = runnable[k - 1]; rk[k] = rk[k - 1]; --k; }
          runnable[k] = x; rk[k] = kx;
        }
      }
      int free_gpu = total_gpus;
      const int nlists = policy == GS_SCHED_GITTINS ? 1 : nq;
      for (int q = 0; q < nlists; ++q) {
        const int *lst = policy == GS_SCHED_GITTINS ? runnable : S.queues + (size_t)q * n;
        const int ln = policy == GS_SCHED_GITTINS ? rn : S.qn[q];
        for (int i = 0; i < ln; ++i) {
          const int j = lst[i];
          const JobIn jr = jobs[j];
          PJob &r = pj[j];
          if (free_gpu >= jr.gpus) {
            if (r.status == PST_PENDING) run_jobs[nrun++] = j;
            free_gpu -= jr.gpus;
            busy += jr.gpus; mem_busy += (long long)jr.gpus * (jr.memb < cap_bytes ? jr.memb : cap_bytes);
          } else if (r.status == PST_RUNNING) { pre_jobs[-(npre++)] = j; }
        }
      }
    }
    for (int i = 0; i < npre; ++i) { pj[pre_jobs[-i]].status = PST_PENDING; ++events; }
    for (int i = 0; i < nrun; ++i) {
      PJob &r = pj[run_jobs[i]];
      r.status = PST_RUNNING; r.resume += 1; ++events;
      if (r.start < 0) r.start = event_time;
    }
    if (is_dlas) {
      for (int q = 0; q < nq; ++q) {
        int *qv = S.queues + (size_t)q * n;
        int w = 0, pn = 0;
        for (int i = 0; i < S.qn[q]; ++i) { const int j = qv[i]; if (pj[j].status == PST_PENDING) tmpl[pn++] = j; else qv[w++] = j; }
        for (int i = 0; i < pn; ++i) qv[w++] = tmpl[i];
      }
    }
    end_time = 0x7fffffff; en = 0;
    next_job_jump = 0x7fffffff;
    int running = 0, queued = 0, pmax = 0;
    long long psum = 0;
    for (int i = 0; i < rn; ++i) {
      const int j = runnable[i];
      const PJob r = pj[j];
      if (r.status != PST_RUNNING) { ++queued; psum += r.pending; pmax = max(pmax, r.pending); continue; }
      ++running;
      const JobIn jr = jobs[j];
      double cl = ceil(jr.dur);
      const int D = cl < 1.0 ? 1 : (int)cl;
      const int e = event_time + (D - r.total_exec);
      if (e < end_time) { end_time = e; en = 0; endj[en++] = j; }
      else if (e == end_time) endj[en++] = j;
      if (is_dlas && r.q_id < nq - 1) {
        const double lim = S.queue_limit[r.q_id];
        const double jt = gputime ? ceil((lim - (double)r.exec) / (double)jr.gpus) + event_time : lim - (double)r.exec + event_time;
        int jti = jt > 2.0e9 ? 0x7fffffff : (int)jt;
        next_job_jump = min(next_job_jump, jti);
      }
    }
    if (policy == GS_SCHED_GITTINS) next_git += (double)event_time;
    {
      int busy_nodes = 0;
      if (policy == GS_SCHED_SJF) for (int nd = 0; nd < M; ++nd) busy_nodes += (S.cidle[nd] < G);
      int4 *dst = reinterpret_cast<int4 *>(&S.rows[ticks - row_first]);
      dst[0] = make_int4(event_time, M - busy_nodes, busy_nodes, busy);
      dst[1] = make_int4(total_gpus - busy, running, queued, nfin);
      dst[2] = make_int4((int)(mem_busy & 0xffffffffLL), (int)(mem_busy >> 32), (int)(psum & 0xffffffffLL), (int)(psum >> 32));
      dst[3] = make_int4(pmax, 0, 0, 0);
    }
    ticks += 1; budget -= 1;
  }
  if (!done && !((n - p) + rn > 0)) done = true;
  if (!done && p >= n && end_time == 0x7fffffff) done = true;
  if (done) {   // jobs that started but never completed keep their start and restart count
    for (int j = 0; j < n; ++j) { const PJob r = pj[j]; if (r.status != PST_END && r.status != PST_NONE && r.start >= 0) { rec[j].start = r.start; rec[j].preempt = r.resume; } }
  }
  S.p = p; S.rn = rn; S.en = en; S.end_time = end_time; S.next_job_jump = next_job_jump; S.finished = nfin;
  S.stale_n = stale_n;
  S.next_gittins_unit = next_git; S.events = events; S.ticks = ticks; S.row_first = row_first;
  S.done = done ? 1 : 0; S.status = status; S.running = 0; S.top = 0; S.started = 0;
}

// ------------------------------------------------------------------ event-driven policies, warp cooperative
// dlas / dlas-gpu (MLFQ with GPU counting), one WARP per replica.  Same semantics as
// gs_policy_kernel / oracle/policy_oracle.c, but every O(runnable) loop of an event runs 32
// entries at a time: counter update + END compaction (ballot prefix), demotion list in runnable
// order, greedy admission as a warp prefix sum with skip, RUNNING-before-PENDING stable partition
// of each queue, min-reduction for the next completion / queue jump.
__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
  #pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(FULL, v, o); if (lane >= o) v += t; }
  return v;
}

// exact int64 sum of one int per lane: 32 pending times can add up past 2^31 - 1 (the thread kernel and the oracle sum
// into int64), so the warp sums the arithmetic high 16 bits and the low 16 bits apart; each partial sum stays below 2^21
// in magnitude, so the 32-bit reductions cannot wrap
__device__ __forceinline__ long long warp_sum_i64(int v) {
  const int hi = __reduce_add_sync(FULL, v >> 16);
  const unsigned lo = __reduce_add_sync(FULL, (unsigned)v & 0xffffu);
  return (long long)hi * 65536 + (long long)lo;
}

__global__ void __launch_bounds__(32, GS_POLICY_MINBLOCKS) gs_dlas_warp_kernel(SimDev *sims, int nsims, long long max_ticks) {
  const int sim = blockIdx.x;
  const int lane = threadIdx.x;
  if (sim >= nsims) return;
  SimDev &S = sims[sim];
  const int policy = S.policy;
  if (!(policy == GS_SCHED_DLAS || policy == GS_SCHED_DLAS_GPU) || S.done || S.status != 0) return;
  const int n = S.n, M = S.M, G = S.G;
  const bool gputime = policy == GS_SCHED_DLAS_GPU;
  const int nq = S.num_queue;
  const JobIn *__restrict__ jobs = S.jobs;
  PJob *pj = S.pj;
  int *runnable = S.runnable, *endj = S.endj, *tmpl = S.tmpl, *stalej = S.stalej;
  gs_job_rec *rec = S.rec;
  int *fin = S.fin, *queues = S.queues;
  gs_tick_row *rows = S.rows;
  const long long rows_cap = S.rows_cap;
  const long long cap_bytes = S.cap_bytes;
  const int total_gpus = M * G;
  const unsigned lt = (1u << lane) - 1u;
  int p = S.p, rn = S.rn, en = S.en, end_time = S.end_time, next_job_jump = S.next_job_jump, nfin = S.finished;
  int stale_n = S.stale_n;
  int qn[GS_MAX_QUEUES];
  #pragma unroll
  for (int q = 0; q < GS_MAX_QUEUES; ++q) qn[q] = S.qn[q];
  double qlim[GS_MAX_QUEUES];
  #pragma unroll
  for (int q = 0; q < GS_MAX_QUEUES; ++q) qlim[q] = S.queue_limit[q];
  long long events = S.events, ticks = S.ticks;
  const long long row_first = ticks;
  long long budget = max_ticks > 0 ? max_ticks : 0x7fffffffffffffffLL;
  bool done = false;

  while (budget > 0 && (ticks - row_first) < rows_cap) {
    if (!((n - p) + rn > 0)) { done = true; break; }
    if (p >= n && end_time == 0x7fffffff) { done = true; break; }
    const int start_time = p < n ? jobs[p].arrive : 0x7fffffff;
    int event_time; bool has_start = false, has_end = false;
    const int *elist = endj; int ecount = en;
    if (end_time < start_time) { event_time = end_time; has_end = true; }
    else if (end_time > start_time) { event_time = start_time; has_start = true; }
    else {                      // tie: the start event inherits this end list (quirk Q25, run_sim.py:708-710)
      event_time = start_time; has_start = has_end = true;
      for (int i = lane; i < en; i += 32) stalej[i] = endj[i];
      stale_n = en;
      __syncwarp();
    }
    if (event_time > next_job_jump) { event_time = next_job_jump; has_start = has_end = false; }   // keeps the inherited list
    else if (has_start) {       // the start event is consumed: an inherited list completes here, whatever the jobs' state
      if (stale_n > 0) { elist = stalej; ecount = stale_n; has_end = true; }
      stale_n = 0;
    }
    // ---- completions (an end list is in runnable order)
    if (has_end) {
      for (int i = lane; i < ecount; i += 32) {
        const int j = elist[i];
        PJob r = pj[j];
        r.status = PST_END;
        pj[j] = r;
        const double dur = jobs[j].dur;
        const double cl = ceil(dur);
        gs_job_rec o; o.start = r.start; o.end = event_time; o.jct = cl < 1.0 ? 1 : (int)cl; o.preempt = r.resume; o.duration = dur;
        rec[j] = o;
        fin[nfin + i] = j;
      }
      nfin += ecount; events += ecount;
    }
    // ---- arrivals: appended to runnable and to queue 0 in trace order
    if (has_start) {
      int cnt = 0;
      while (true) {
        const int idx = p + cnt + lane;
        const unsigned b = __ballot_sync(FULL, idx < n && jobs[idx].arrive == event_time);
        const int c = (b == FULL) ? 32 : __ffs(~b) - 1;       // run of arrivals from the front
        cnt += c;
        if (c < 32) break;
      }
      for (int i = lane; i < cnt; i += 32) {
        const int j = p + i;
        PJob r; r.last_check = event_time; r.total_exec = 0; r.exec = 0; r.pending = 0; r.last_pending = 0; r.start = -1;
        r.resume = 0; r.status = PST_PENDING; r.q_id = 0; r.pad0 = 0; r.pad1 = 0;
        pj[j] = r;
        runnable[rn + i] = j;
        queues[qn[0] + i] = j;
      }
      rn += cnt; qn[0] += cnt; events += cnt; p += cnt;
    }
    __syncwarp();
    // ---- pass 1 over runnable: drop END, age counters, detect demotions (kept in runnable order)
    int nd = 0;
    {
      int w = 0;
      for (int base = 0; base < rn; base += 32) {
        const int idx = base + lane;
        const bool valid = idx < rn;
        const int j = valid ? runnable[idx] : 0;
        PJob r;
        if (valid) r = pj[j]; else { r.status = PST_END; r.q_id = 0; r.last_check = 0; r.total_exec = 0; r.exec = 0; r.pending = 0; r.last_pending = 0; r.start = -1; r.resume = 0; }
        const bool keep = valid && r.status != PST_END;
        bool demote = false;
        if (keep) {
          const int dt = event_time - r.last_check;
          r.last_check = event_time;
          if (r.status == PST_RUNNING) {
            r.total_exec += dt; r.exec += dt;
            const double j_gt = gputime ? (double)r.exec * jobs[j].gpus : (double)r.exec;
            if (r.q_id < nq - 1 && j_gt >= qlim[r.q_id]) { demote = true; r.q_id += 1; }
          } else {
            r.pending += dt;
            if (r.exec > 0) r.last_pending += dt;
          }
          pj[j] = r;
        }
        const unsigned kb = __ballot_sync(FULL, keep), db = __ballot_sync(FULL, demote);
        if (keep) runnable[w + __popc(kb & lt)] = j;
        if (demote) tmpl[nd + __popc(db & lt)] = j;
        w += __popc(kb); nd += __popc(db);
      }
      rn = w;
    }
    __syncwarp();
    // ---- queues: drop END / demoted-away entries, then append this event's demotions
    for (int q = 0; q < nq; ++q) {
      int *qv = queues + (size_t)q * n;
      int w = 0;
      for (int base = 0; base < qn[q]; base += 32) {
        const int idx = base + lane;
        const bool valid = idx < qn[q];
        const int j = valid ? qv[idx] : 0;
        bool keep = false;
        if (valid) { const PJob r = pj[j]; keep = r.status != PST_END && r.q_id == q; }
        const unsigned kb = __ballot_sync(FULL, keep);
        if (keep) qv[w + __popc(kb & lt)] = j;
        w += __popc(kb);
      }
      qn[q] = w;
      __syncwarp();
      if (q > 0) {          // jobs demoted into q, in runnable order
        for (int base = 0; base < nd; base += 32) {
          const int idx = base + lane;
          const int j = idx < nd ? tmpl[idx] : 0;
          const bool mine = idx < nd && pj[j].q_id == q;
          const unsigned mb = __ballot_sync(FULL, mine);
          if (mine) qv[qn[q] + __popc(mb & lt)] = j;
          qn[q] += __popc(mb);
        }
      }
      __syncwarp();
    }
    // ---- greedy re-admission on the emptied cluster (GPU counting), queue by queue, and the
    //      RUNNING-before-PENDING stable partition of each queue
    int free_gpu = total_gpus, busy = 0;
    long long mem_busy = 0;
    for (int q = 0; q < nq; ++q) {
      int *qv = queues + (size_t)q * n;
      int w = 0, pn = 0;   // RUNNING entries written so far / PENDING entries parked in tmpl
      for (int base = 0; base < qn[q]; base += 32) {
        const int idx = base + lane;
        const bool valid = idx < qn[q];
        const int j = valid ? qv[idx] : 0;
        PJob r; JobIn jr;
        int g = 0;
        if (valid) { r = pj[j]; jr = jobs[j]; g = jr.gpus; } else { r.status = PST_NONE; r.start = -1; r.resume = 0; jr.memb = 0; }
        // sequential greedy over the 32 entries: admit while the prefix fits, skip the first that does not
        bool admitted = false, decided = !valid;
        while (true) {
          const unsigned ub = __ballot_sync(FULL, !decided);
          if (ub == 0) break;
          if (free_gpu == 0) { decided = true; continue; }
          const int inc = warp_incl_scan(decided ? 0 : g, lane);
          const bool fits = !decided && inc <= free_gpu;
          const unsigned fb = __ballot_sync(FULL, !decided && !fits);     // undecided entries that do not fit
          const int first_fail = fb ? __ffs(fb) - 1 : 32;
          if (!decided && lane < first_fail) { admitted = true; decided = true; }
          if (!decided && lane == first_fail) decided = true;            // rejected
          const int last_ok = first_fail - 1;
          const int used_now = last_ok >= 0 ? __shfl_sync(FULL, inc, last_ok < 0 ? 0 : last_ok) : 0;
          free_gpu -= used_now;
        }
        // status transitions (each one is an event): PENDING->RUNNING = resume, RUNNING->PENDING = preempt
        const bool flip_run = valid && admitted && r.status == PST_PENDING;
        const bool flip_pre = valid && !admitted && r.status == PST_RUNNING;
        if (flip_run) { r.status = PST_RUNNING; r.resume += 1; if (r.start < 0) r.start = event_time; pj[j] = r; }
        if (flip_pre) { r.status = PST_PENDING; pj[j] = r; }
        events += __popc(__ballot_sync(FULL, flip_run)) + __popc(__ballot_sync(FULL, flip_pre));
        // the admitted GPUs of a chunk come out of free_gpu <= M * G <= 2^26 (check_cluster), so this int sum cannot wrap
        busy += __reduce_add_sync(FULL, admitted ? g : 0);
        {
          long long mc = admitted ? (long long)g * (jr.memb < cap_bytes ? jr.memb : cap_bytes) : 0;
          #pragma unroll
          for (int o = 16; o > 0; o >>= 1) mc += __shfl_xor_sync(FULL, mc, o);
          mem_busy += mc;
        }
        // stable partition: RUNNING entries stay in place order, PENDING go behind
        const bool is_run = valid && admitted;
        const bool is_pen = valid && !admitted;
        const unsigned rb = __ballot_sync(FULL, is_run), pb = __ballot_sync(FULL, is_pen);
        if (is_run) qv[w + __popc(rb & lt)] = j;
        if (is_pen) tmpl[pn + __popc(pb & lt)] = j;
        w += __popc(rb); pn += __popc(pb);
      }
      __syncwarp();
      for (int i = lane; i < pn; i += 32) qv[w + i] = tmpl[i];
      __syncwarp();
    }
    // ---- final pass over runnable: transitions are counted, next completion / jump, statistics
    end_time = 0x7fffffff; en = 0; next_job_jump = 0x7fffffff;
    int running = 0, queued = 0, pmax = 0;
    long long psum = 0;
    for (int base = 0; base < rn; base += 32) {
      const int idx = base + lane;
      const bool valid = idx < rn;
      const int j = valid ? runnable[idx] : 0;
      int e = 0x7fffffff, jt = 0x7fffffff, pend = 0;
      bool isrun = false;
      if (valid) {
        const PJob r = pj[j];
        isrun = r.status == PST_RUNNING;
        if (isrun) {
          const JobIn jr = jobs[j];
          const double cl = ceil(jr.dur);
          const int D = cl < 1.0 ? 1 : (int)cl;
          e = event_time + (D - r.total_exec);
          if (r.q_id < nq - 1) {
            const double lim = qlim[r.q_id];
            const double t = gputime ? ceil((lim - (double)r.exec) / (double)jr.gpus) + event_time : lim - (double)r.exec + event_time;
            jt = t > 2.0e9 ? 0x7fffffff : (int)t;
          }
        } else pend = r.pending;
      }
      const int cmin = __reduce_min_sync(FULL, e);
      if (cmin < end_time) { end_time = cmin; en = 0; }
      const unsigned eb = __ballot_sync(FULL, valid && isrun && e == end_time);
      if (valid && isrun && e == end_time) endj[en + __popc(eb & lt)] = j;
      en += __popc(eb);
      next_job_jump = min(next_job_jump, __reduce_min_sync(FULL, jt));
      running += __popc(__ballot_sync(FULL, valid && isrun));
      queued += __popc(__ballot_sync(FULL, valid && !isrun));
      pmax = max(pmax, __reduce_max_sync(FULL, pend));
      psum += warp_sum_i64(pend);
    }
    __syncwarp();
    if (lane == 0) {
      int4 *dst = reinterpret_cast<int4 *>(&rows[ticks - row_first]);
      dst[0] = make_int4(event_time, M, 0, busy);
      dst[1] = make_int4(total_gpus - busy, running, queued, nfin);
      dst[2] = make_int4((int)(mem_busy & 0xffffffffLL), (int)(mem_busy >> 32), (int)(psum & 0xffffffffLL), (int)(psum >> 32));
      dst[3] = make_int4(pmax, 0, 0, 0);
    }
    ticks += 1; budget -= 1;
  }
  if (!done && !((n - p) + rn > 0)) done = true;
  if (!done && p >= n && end_time == 0x7fffffff) done = true;
  __syncwarp();
  if (done) {
    for (int j = lane; j < n; j += 32) { const PJob r = pj[j]; if (r.status != PST_END && r.status != PST_NONE && r.start >= 0) { rec[j].start = r.start; rec[j].preempt = r.resume; } }
  }
  if (lane == 0) {
    S.p = p; S.rn = rn; S.en = en; S.end_time = end_time; S.next_job_jump = next_job_jump; S.finished = nfin;
    S.stale_n = stale_n;
    #pragma unroll
    for (int q = 0; q < GS_MAX_QUEUES; ++q) S.qn[q] = qn[q];
    S.events = events; S.ticks = ticks; S.row_first = row_first;
    S.done = done ? 1 : 0; S.running = 0; S.top = 0; S.started = 0;
  }
}

// sjf (stable order by num_gpu + live-yarn placement on the emptied cluster) and gittins (stable
// order by gittins rank + GPU counting), one WARP per replica.  Same semantics as
// gs_policy_kernel / oracle/policy_oracle.c.  The runnable list stays sorted between events for
// sjf (keys never change), so new arrivals are INSERTED (count of keys <= k, warp-parallel shift);
// gittins ranks move a little every event, so the list is repaired with stable odd-even
// transposition rounds (adjacent swaps only when strictly greater == the unique stable order).
__global__ void __launch_bounds__(32, GS_POLICY_MINBLOCKS) gs_sortpol_warp_kernel(SimDev *sims, int nsims, long long max_ticks) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int sim = blockIdx.x;
  const int lane = threadIdx.x;
  if (sim >= nsims) return;
  SimDev &S = sims[sim];
  const int policy = S.policy;
  if (!(policy == GS_SCHED_SJF || policy == GS_SCHED_GITTINS) || S.done || S.status != 0) return;
  const bool sjf = policy == GS_SCHED_SJF;
  const int n = S.n, M = S.M, G = S.G, K = S.K;
  int *nidle = reinterpret_cast<int *>(smem_raw);        // sjf: (idle devices, free slots) per node
  int *nkfree = nidle + M;
  const JobIn *__restrict__ jobs = S.jobs;
  PJob *pj = S.pj;
  int *runnable = S.runnable, *endj = S.endj, *stalej = S.stalej;
  double *rk = reinterpret_cast<double *>(S.queues);     // gittins: rank of runnable[i] (no queues in these policies)
  gs_job_rec *rec = S.rec;
  int *fin = S.fin;
  gs_tick_row *rows = S.rows;
  const long long rows_cap = S.rows_cap;
  const long long cap_bytes = S.cap_bytes, fit_limit = S.fit_limit;
  const int total_gpus = M * G;
  const unsigned lt = (1u << lane) - 1u;
  int p = S.p, rn = S.rn, en = S.en, end_time = S.end_time, nfin = S.finished, stale_n = S.stale_n;
  double next_git = S.next_gittins_unit;
  long long events = S.events, ticks = S.ticks;
  const long long row_first = ticks;
  long long budget = max_ticks > 0 ? max_ticks : 0x7fffffffffffffffLL;
  bool done = false;
  // sharded mode (gs_comm_init): rank `me` of `nr` evaluates the gittins index for the chunks c of the runnable list
  // with c % nr == me and stores the values into every rank's receive buffer; one exchange per event
  const int nr_all = (!sjf && S.comm_n > 1) ? S.comm_n : 1, me = S.comm_rank;
  const int min_rn = S.comm_min_runnable;       // shorter runnable lists are not worth an exchange: every rank evaluates them itself
  const long long ccap = S.comm_cap;
  unsigned long long epoch = S.comm_epoch;
  long long wait_cycles = 0;
  int status = 0;
  const double rank_new = sjf ? 0.0 : git_lookup(S, 0.0);        // a new job: executed_time == 0

  while (budget > 0 && (ticks - row_first) < rows_cap) {
    if (!((n - p) + rn > 0)) { done = true; break; }
    if (p >= n && end_time == 0x7fffffff) { done = true; break; }
    const int start_time = p < n ? jobs[p].arrive : 0x7fffffff;
    int event_time; bool has_start = false, has_end = false;
    const int *elist = endj; int ecount = en;
    if (end_time < start_time) { event_time = end_time; has_end = true; }
    else if (end_time > start_time) { event_time = start_time; has_start = true; }
    else {                      // tie: the start event inherits this end list (quirk Q25, run_sim.py:994-996)
      event_time = start_time; has_start = has_end = true;
      if (!sjf) {               // sjf has no jump events, so nothing can come between the tie and the start
        for (int i = lane; i < en; i += 32) stalej[i] = endj[i];
        stale_n = en;
        __syncwarp();
      }
    }
    if (!sjf && (double)event_time > next_git) { event_time = (int)next_git; has_start = has_end = false; }   // keeps the inherited list
    else if (has_start) {       // the start event is consumed: an inherited list completes here
      if (stale_n > 0) { elist = stalej; ecount = stale_n; has_end = true; }
      stale_n = 0;
    }
    // ---- completions
    if (has_end) {
      for (int i = lane; i < ecount; i += 32) {
        const int j = elist[i];
        PJob r = pj[j];
        r.status = PST_END;
        pj[j] = r;
        const double dur = jobs[j].dur;
        const double cl = ceil(dur);
        gs_job_rec o; o.start = r.start; o.end = event_time; o.jct = cl < 1.0 ? 1 : (int)cl; o.preempt = r.resume; o.duration = dur;
        rec[j] = o;
        fin[nfin + i] = j;
      }
      nfin += ecount; events += ecount;
    }
    __syncwarp();
    // ---- pass 1: drop END, age counters, (gittins) rank of every survivor at its new position
    // (the list length is the same on every rank, so all of them take the same decision about the exchange)
    const int nr = (nr_all > 1 && rn > min_rn) ? nr_all : 1;
    {
      int w = 0;
      for (int base = 0; base < rn; base += 32) {
        const int idx = base + lane;
        const bool valid = idx < rn;
        const int j = valid ? runnable[idx] : 0;
        PJob r;
        r.status = PST_END; r.q_id = 0; r.last_check = 0; r.total_exec = 0; r.exec = 0; r.pending = 0; r.last_pending = 0; r.start = -1; r.resume = 0;
        if (valid) r = pj[j];
        const bool keep = valid && r.status != PST_END;
        const bool mine = nr == 1 || ((base >> 5) % nr) == me;     // sharded: whose chunk this is
        double rank = 0.0;
        if (keep) {
          const int dt = event_time - r.last_check;
          r.last_check = event_time;
          if (r.status == PST_RUNNING) { r.total_exec += dt; r.exec += dt; }
          else { r.pending += dt; if (r.exec > 0) r.last_pending += dt; }
          pj[j] = r;
          if (!sjf && mine) rank = git_lookup(S, r.status == PST_RUNNING ? (double)r.exec * jobs[j].gpus : (double)r.exec);
        }
        const unsigned kb = __ballot_sync(FULL, keep);
        if (keep) {
          const int pos = w + __popc(kb & lt);
          runnable[pos] = j;
          if (!sjf) {
            if (nr == 1) rk[pos] = rank;
            else if (mine) {
              const long long at = (long long)(epoch & 1ull) * ccap + pos;
              for (int q = 0; q < nr; ++q) S.comm_peer_rk[q][at] = rank;      // NVLink peer store (own buffer included)
            }
          }
        }
        w += __popc(kb);
      }
      rn = w;
    }
    __syncwarp();
    if (nr > 1) {
      // ---- the exchange: publish "my ranks of event `epoch` are in your buffer" to every rank, wait for theirs
      __threadfence_system();
      __syncwarp();
      const long long t0 = clock64();
      bool late = false;
      if (lane < nr) {
        *reinterpret_cast<volatile unsigned long long *>(&S.comm_peer_flags[lane][me]) = epoch + 1ull;
        const volatile unsigned long long *mine_f = reinterpret_cast<const volatile unsigned long long *>(&S.comm_flags[lane]);
        while (*mine_f < epoch + 1ull) {
          if (clock64() - t0 > 10000000000LL) { late = true; break; }       // ~5 s: a peer is gone
        }
      }
      late = __any_sync(FULL, late);
      wait_cycles += clock64() - t0;
      __threadfence_system();
      if (late) { status = GS_ERR_COMM; break; }
      const double *rin = S.comm_rk_in + (long long)(epoch & 1ull) * ccap;
      for (int i = lane; i < rn; i += 32) rk[i] = __ldcg(&rin[i]);
      epoch += 1ull;
      __syncwarp();
    }
    // ---- arrivals (after the survivors, like the list append of the specification)
    int cnt = 0;
    if (has_start) {
      while (true) {
        const int idx = p + cnt + lane;
        const unsigned b = __ballot_sync(FULL, idx < n && jobs[idx].arrive == event_time);
        const int c = (b == FULL) ? 32 : __ffs(~b) - 1;
        cnt += c;
        if (c < 32) break;
      }
      for (int i = lane; i < cnt; i += 32) {
        const int j = p + i;
        PJob r; r.last_check = event_time; r.total_exec = 0; r.exec = 0; r.pending = 0; r.last_pending = 0; r.start = -1;
        r.resume = 0; r.status = PST_PENDING; r.q_id = 0; r.pad0 = 0; r.pad1 = 0;
        pj[j] = r;
      }
      events += cnt;
      if (!sjf) {
        for (int i = lane; i < cnt; i += 32) { runnable[rn + i] = p + i; rk[rn + i] = rank_new; }
        rn += cnt;
      }
    }
    __syncwarp();
    if (sjf) {
      // stable insertion of each new job: position = number of runnable entries with num_gpu <= its own
      for (int i = 0; i < cnt; ++i) {
        const int j = p + i;
        const int kx = jobs[j].gpus;
        int pos = 0;
        for (int base = 0; base < rn; base += 32) {
          const int idx = base + lane;
          const bool le = idx < rn && jobs[runnable[idx]].gpus <= kx;
          pos += __popc(__ballot_sync(FULL, le));
        }
        for (int hi = rn; hi > pos; hi -= 32) {              // shift [pos, rn) right by one, from the tail
          const int idx = hi - 1 - lane;
          const int v = idx >= pos ? runnable[idx] : 0;
          __syncwarp();
          if (idx >= pos) runnable[idx + 1] = v;
          __syncwarp();
        }
        if (lane == 0) runnable[pos] = j;
        rn += 1;
        __syncwarp();
      }
    } else {
      // stable odd-even transposition until a full round makes no swap
      bool again = rn > 1;
      while (again) {
        unsigned any = 0;
        for (int phase = 0; phase < 2; ++phase) {
          for (int base = phase; base + 1 < rn; base += 64) {
            const int a = base + 2 * lane;
            bool sw = false;
            if (a + 1 < rn) {
              const double ka = rk[a], kb2 = rk[a + 1];
              if (ka > kb2) { const int ja = runnable[a], jb = runnable[a + 1]; runnable[a] = jb; runnable[a + 1] = ja; rk[a] = kb2; rk[a + 1] = ka; sw = true; }
            }
            any |= __ballot_sync(FULL, sw);
          }
          __syncwarp();
        }
        again = any != 0;
      }
    }
    p += cnt;
    __syncwarp();
    // ---- greedy re-admission on the emptied cluster, in list order; the chunk that has just been decided also feeds
    // the next completion (ties in list order) and the statistics, while its records are still in registers
    int busy = 0;
    long long mem_busy = 0;
    end_time = 0x7fffffff; en = 0;
    int running = 0, queued = 0, pmax = 0;
    long long psum = 0;
#define SORTPOL_ACCOUNT(valid_, j_, r_, dur_)                                                         \
    do {                                                                                              \
      int e_ = 0x7fffffff, pend_ = 0;                                                                 \
      const bool isrun_ = (valid_) && (r_).status == PST_RUNNING;                                     \
      if (isrun_) {                                                                                   \
        const double cl_ = ceil(dur_);                                                                \
        const int D_ = cl_ < 1.0 ? 1 : (int)cl_;                                                      \
        e_ = event_time + (D_ - (r_).total_exec);                                                     \
      } else if (valid_) pend_ = (r_).pending;                                                        \
      const int cmin_ = __reduce_min_sync(FULL, e_);                                                  \
      if (cmin_ < end_time) { end_time = cmin_; en = 0; }                                             \
      const unsigned eb_ = __ballot_sync(FULL, isrun_ && e_ == end_time);                             \
      if (isrun_ && e_ == end_time) endj[en + __popc(eb_ & lt)] = (j_);                               \
      en += __popc(eb_);                                                                              \
      running += __popc(__ballot_sync(FULL, isrun_));                                                 \
      queued += __popc(__ballot_sync(FULL, (valid_) && !isrun_));                                     \
      pmax = max(pmax, __reduce_max_sync(FULL, pend_));                                               \
      psum += warp_sum_i64(pend_);                                                                    \
    } while (0)
    if (sjf) {
      for (int nd = lane; nd < M; nd += 32) { nidle[nd] = G; nkfree[nd] = K; }
      __syncwarp();
      // The list is walked 32 entries at a time.  Consecutive entries that ask for the same thing (GPUs, GPUs per task,
      // fits a device) are placed together: identical jobs fill the nodes in id order -- each goes to the first node
      // that still holds one (single node) or takes the next tasks of the walk (cross node) -- so a run of r of them
      // is one prefix sum over the node capacities instead of r first-fit scans, and the first `placed` of the run are
      // the ones that start.  The list is ordered by GPU count, so runs are long.
      for (int base = 0; base < rn; base += 32) {
        const int idx = base + lane;
        const bool valid = idx < rn;
        const int j = valid ? runnable[idx] : 0;
        int hg = 0, hc = 1;
        long long memb = 0;
        PJob r;
        r.status = PST_NONE; r.start = -1; r.resume = 0;
        double dur = 0.0;
        r.total_exec = 0; r.pending = 0;
        if (valid) { const JobIn jr = jobs[j]; hg = jr.gpus; hc = jr.gpc; memb = jr.memb; dur = jr.dur; r = pj[j]; }
        const bool fit = valid && memb < fit_limit;
        const unsigned fb = __ballot_sync(FULL, fit);
        const int phg = __shfl_up_sync(FULL, hg, 1), phc = __shfl_up_sync(FULL, hc, 1);
        const bool pfit = lane > 0 && ((fb >> (lane - 1)) & 1u);
        const bool head = valid && (lane == 0 || hg != phg || hc != phc || fit != pfit);
        unsigned heads = __ballot_sync(FULL, head);
        const int nvalid = __popc(__ballot_sync(FULL, valid));
        bool ok = false;
        while (heads) {
          const int s0 = __ffs(heads) - 1;
          heads &= heads - 1;
          const int e0 = heads ? __ffs(heads) - 1 : nvalid;
          const int rcount = e0 - s0;
          const int rhg = __shfl_sync(FULL, hg, s0), rhc = __shfl_sync(FULL, hc, s0);
          int placed = 0;
          if ((fb >> s0) & 1u) {
            const int rtasks = rhc == 1 ? rhg : rhg / rhc;
            if (rhg <= G) {
              // capacity of a node in such jobs = min(idle / gpus, slots / tasks); divisions by the run's constants as
              // multiplications by 2^32 / d (exact below 65536; larger tables take the plain division)
              const bool small = G < 65536 && K < 65536;
              const unsigned mg = (small && rhg > 1) ? 0xffffffffu / (unsigned)rhg + 1u : 0u;
              const unsigned mt = (small && rtasks > 1) ? 0xffffffffu / (unsigned)rtasks + 1u : 0u;
              int left = rcount;
              for (int nb = 0; nb < M && left > 0; nb += 32) {
                const int nd = nb + lane;
                int c = 0, ni = 0, nk = 0;
                if (nd < M) {
                  ni = nidle[nd]; nk = nkfree[nd];
                  const int cg = rhg == 1 ? ni : (mg ? (int)__umulhi((unsigned)max(ni, 0), mg) : max(ni, 0) / rhg);
                  const int ct = rtasks == 1 ? nk : (mt ? (int)__umulhi((unsigned)max(nk, 0), mt) : max(nk, 0) / rtasks);
                  c = max(min(cg, ct), 0);
                }
                const int incl = warp_incl_scan(c, lane);
                const int take = min(c, max(left - (incl - c), 0));
                if (take > 0) { nidle[nd] = ni - take * rhg; nkfree[nd] = nk - take * rtasks; }
                left -= min(left, __shfl_sync(FULL, incl, 31));
              }
              placed = rcount - left;
            } else {
              // cross node: a job takes `rtasks` tasks from the nodes in id order, each node giving what it holds
              const long long want = (long long)rcount * rtasks;
              long long cap = 0;
              for (int nb = 0; nb < M && cap < want; nb += 32) {
                const int nd = nb + lane;
                const int c = nd < M ? max(min(nidle[nd] / rhc, nkfree[nd]), 0) : 0;
                cap += __reduce_add_sync(FULL, c);        // c <= G <= 64 per lane: the int sum cannot wrap
              }
              placed = (int)min((long long)rcount, cap / rtasks);
              long long todo = (long long)placed * rtasks;
              for (int nb = 0; nb < M && todo > 0; nb += 32) {
                const int nd = nb + lane;
                const int c = nd < M ? max(min(nidle[nd] / rhc, nkfree[nd]), 0) : 0;
                const int incl = warp_incl_scan(c, lane);
                const long long before = todo - (long long)(incl - c);
                const int take = before > 0 ? (int)min((long long)c, before) : 0;
                if (take > 0) { nidle[nd] -= take * rhc; nkfree[nd] -= take; }
                const int tot = __shfl_sync(FULL, incl, 31);
                todo -= min(todo, (long long)tot);
              }
            }
            __syncwarp();          // lanes updated different nodes
          }
          if (lane >= s0 && lane < e0) ok = (lane - s0) < placed;
        }
        const bool flip_run = valid && ok && r.status == PST_PENDING;
        const bool flip_pre = valid && !ok && r.status == PST_RUNNING;
        if (flip_run) { r.status = PST_RUNNING; r.resume += 1; if (r.start < 0) r.start = event_time; pj[j] = r; }
        else if (valid && ok && r.start < 0) { r.start = event_time; pj[j] = r; }
        if (flip_pre) { r.status = PST_PENDING; pj[j] = r; }
        events += __popc(__ballot_sync(FULL, flip_run)) + __popc(__ballot_sync(FULL, flip_pre));
        // placed jobs hold distinct devices, at most M * G <= 2^26 (check_cluster): this int sum cannot wrap
        busy += __reduce_add_sync(FULL, ok ? hg : 0);
        long long mc = ok ? (long long)hg * (memb < cap_bytes ? memb : cap_bytes) : 0;
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) mc += __shfl_xor_sync(FULL, mc, o);
        mem_busy += mc;
        SORTPOL_ACCOUNT(valid, j, r, dur);
      }
    } else {
      int free_gpu = total_gpus;
      for (int base = 0; base < rn; base += 32) {
        const int idx = base + lane;
        const bool valid = idx < rn;
        const int j = valid ? runnable[idx] : 0;
        PJob r; JobIn jr;
        r.status = PST_NONE; r.start = -1; r.resume = 0; r.total_exec = 0; r.pending = 0; jr.memb = 0; jr.gpus = 0; jr.dur = 0.0;
        int g = 0;
        if (valid) { r = pj[j]; jr = jobs[j]; g = jr.gpus; }
        bool admitted = false, decided = !valid;
        while (true) {
          const unsigned ub = __ballot_sync(FULL, !decided);
          if (ub == 0) break;
          if (free_gpu == 0) { decided = true; continue; }
          const int inc = warp_incl_scan(decided ? 0 : g, lane);
          const bool fits = !decided && inc <= free_gpu;
          const unsigned fb = __ballot_sync(FULL, !decided && !fits);
          const int first_fail = fb ? __ffs(fb) - 1 : 32;
          if (!decided && lane < first_fail) { admitted = true; decided = true; }
          if (!decided && lane == first_fail) decided = true;
          const int used_now = first_fail > 0 ? __shfl_sync(FULL, inc, first_fail - 1) : 0;
          free_gpu -= used_now;
        }
        const bool flip_run = valid && admitted && r.status == PST_PENDING;
        const bool flip_pre = valid && !admitted && r.status == PST_RUNNING;
        if (flip_run) { r.status = PST_RUNNING; r.resume += 1; if (r.start < 0) r.start = event_time; pj[j] = r; }
        if (flip_pre) { r.status = PST_PENDING; pj[j] = r; }
        events += __popc(__ballot_sync(FULL, flip_run)) + __popc(__ballot_sync(FULL, flip_pre));
        // the admitted GPUs of a chunk come out of free_gpu <= M * G <= 2^26 (check_cluster), so this int sum cannot wrap
        busy += __reduce_add_sync(FULL, admitted ? g : 0);
        long long mc = admitted ? (long long)g * (jr.memb < cap_bytes ? jr.memb : cap_bytes) : 0;
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) mc += __shfl_xor_sync(FULL, mc, o);
        mem_busy += mc;
        SORTPOL_ACCOUNT(valid, j, r, jr.dur);
      }
    }
#undef SORTPOL_ACCOUNT
    __syncwarp();
    // ---- next completion and statistics were accumulated chunk by chunk above
    if (!sjf) next_git += (double)event_time;
    int busy_nodes = 0;
    if (sjf) for (int base = 0; base < M; base += 32) { const int nd = base + lane; busy_nodes += __popc(__ballot_sync(FULL, nd < M && nidle[nd] < G)); }
    __syncwarp();
    if (lane == 0) {
      int4 *dst = reinterpret_cast<int4 *>(&rows[ticks - row_first]);
      dst[0] = make_int4(event_time, M - busy_nodes, busy_nodes, busy);
      dst[1] = make_int4(total_gpus - busy, running, queued, nfin);
      dst[2] = make_int4((int)(mem_busy & 0xffffffffLL), (int)(mem_busy >> 32), (int)(psum & 0xffffffffLL), (int)(psum >> 32));
      dst[3] = make_int4(pmax, 0, 0, 0);
    }
    ticks += 1; budget -= 1;
  }
  if (!done && !((n - p) + rn > 0)) done = true;
  if (!done && p >= n && end_time == 0x7fffffff) done = true;
  __syncwarp();
  if (done) {
    for (int j = lane; j < n; j += 32) { const PJob r = pj[j]; if (r.status != PST_END && r.status != PST_NONE && r.start >= 0) { rec[j].start = r.start; rec[j].preempt = r.resume; } }
  }
  if (lane == 0) {
    S.p = p; S.rn = rn; S.en = en; S.end_time = end_time; S.finished = nfin; S.next_gittins_unit = next_git; S.stale_n = stale_n;
    S.events = events; S.ticks = ticks; S.row_first = row_first;
    S.done = done ? 1 : 0; S.running = 0; S.top = 0; S.started = 0;
    S.comm_epoch = epoch; S.comm_wait_cycles += wait_cycles;
    if (status != 0) S.status = status;
  }
}


// gs_boot.cuh -- bootstrap replicas of a trace generated on the device (gs_boot_population / gs_boot_traces,
// include/gsched.h), included by gsched.cu.
//
// A replica is drawn from one base trace, the population P (K records in admission order) and its K - 1 inter-arrival
// gaps D.  Job j of replica (seed, stream) takes the four words w0..w3 of the Philox4x64-10 block with key
// (seed, stream) and counter (j + 1, 0, 0, 0) -- numpy.random.Philox(key=[seed, stream], counter=[j, 0, 0, 0])
// .random_raw(4), since numpy increments its counter before it generates -- and then
//   source row  r_j = floor(w0 * K / 2^64)
//   gap         g_0 = 0, g_j = D[floor(w1 * (K - 1) / 2^64)] (0 when K = 1)
//   arrival     arrive_j = floor((g_0 + ... + g_j) * gap_num / gap_den), exact integers
//   record      {arrive_j, P[r_j].gpus, P[r_j].gpu_per_task, 0, P[r_j].mem_bytes, P[r_j].duration}
// w3 is unused unless the replica is mixed, and w2 unless it is blocked.
//
// Blocked replicas (gs_boot_traces_blocked, the stationary bootstrap of Politis & Romano) resample runs of consecutive
// jobs of geometric length with mean L, so that a trace's bursts survive.  Job 0 starts a block; job j > 0 starts one
// iff floor(w2 * L / 2^64) == 0.  With b_j the last block start <= j and s_b = floor(w0_b * K / 2^64), job j copies
//   row  r_j = (s_{b_j} + (j - b_j)) mod K
//   gap  g_j = D[r_j - 1], the gap that preceded the row in the base trace, for a job that continues a block without
//        wrapping (r_j > 0); the iid gap above for a block start or a wrapped row
// With L = 1 every job starts a block, which is the iid bootstrap.  The generator, the picks and the arithmetic are
// __host__ __device__: tests/emu/boot_emu.cpp and tests/emu/boot_block_emu.cpp run them with g++, and
// tracegen.bootstrap_packed is their numpy mirror.
//
// Mixed replicas (gs_boot_mixes / gs_boot_traces_mixed) draw row i with probability w_i / T for integer weights w
// (T = sum w_i >= 1) through an exact integer alias table {U_i, A_i} (Walker / Vose; gs_boot_alias_build): with
// c = floor(w0 * K / 2^64), the row the unweighted bootstrap takes, and u = floor(w3 * T / 2^64), job j takes
//   row  c if u < U_c, else A_c
// Blocked mixed replicas apply this to s_b at block starts only; a block still continues through the base trace in
// order.  Equal weights give U_i = T everywhere, so every job keeps c: the unweighted replica byte for byte.
//
// gs_boot_kernel: one block per replica walks its jobs in chunks of the block size -- a Philox block per job, a gather
// of the population row, a block-wide inclusive int64 scan of the gaps with a carry between chunks -- and writes the
// chunk's 32-byte records through shared memory into the replica's slot of the trace arena with contiguous 16-byte
// stores.  The same pass reduces the replica's span-pool bound (sum of min(tasks, M)) and last arrival tick.  The
// blocked instantiation first runs a block-wide inclusive max-scan of the key (j << 32) | s_j of every block start
// (0 for other jobs), carried between chunks like the gap sum, so each job reads b_j and s_{b_j} from its scanned key
// however many chunks and wraps of the population its block spans.  The mixed instantiations (MIXED = true) read a
// replica's table offset and T from one extra per-replica record and load one 16-byte table entry per job.
//
// Profiled replicas (gs_boot_profiles / gs_boot_traces_profiled) keep every draw above and move only the arrivals: a
// profile of m segments {t_k, num_k, den_k} and period P becomes, on the host and exactly, base-time starts
//   s_0 = 0, s_(k+1) = s_k + ceil((t_(k+1) - t_k) * den_k / num_k), B = s_m with t_m := P (P > 0 only)
// and job j with gap sum S arrives at
//   a(S) = t_k + floor((S - s_k) * num_k / den_k), k the last segment with s_k <= S    (P = 0)
//   (S div B) * P + a(S mod B)                                                        (P > 0)
// The profiled instantiations load their replica's segments into shared memory once and find each job's segment by
// binary search after the gap scan (gs_boot_profile_seg / gs_boot_profile_arrive, which the host also uses for the
// arrival bound).
#pragma once

#include <stdint.h>

#include <vector>

#include "gsched.h"

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#endif
#ifndef __device__
#define __device__
#endif
#endif

#define GS_BOOT_HD static __host__ __device__ inline
#define GS_BOOT_THREADS 256

static_assert(sizeof(gs_boot_params) == 32, "gs_boot_params is 32 bytes");

// high 64 bits of the 128-bit product a * b
GS_BOOT_HD uint64_t gs_boot_mulhi(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

struct GsPhilox { uint64_t w[4]; };

// Philox4x64-10 (Salmon et al., SC'11; the constants of Random123 and numpy)
GS_BOOT_HD GsPhilox gs_boot_philox(uint64_t k0, uint64_t k1, uint64_t c0, uint64_t c1, uint64_t c2, uint64_t c3) {
  const uint64_t M0 = 0xD2E7470EE14C6C93ull, M1 = 0xCA5A826395121157ull;
  const uint64_t W0 = 0x9E3779B97F4A7C15ull, W1 = 0xBB67AE8584CAA73Bull;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int r = 0; r < 10; ++r) {
    if (r > 0) { k0 += W0; k1 += W1; }
    const uint64_t hi0 = gs_boot_mulhi(M0, c0), lo0 = M0 * c0;
    const uint64_t hi1 = gs_boot_mulhi(M1, c2), lo1 = M1 * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  GsPhilox b;
  b.w[0] = c0; b.w[1] = c1; b.w[2] = c2; b.w[3] = c3;
  return b;
}

// Source row and gap index (-1: no gap, g_j = 0) of job j of a population of K records.
GS_BOOT_HD void gs_boot_pick(uint64_t seed, uint64_t stream, long long j, long long K, long long &row, long long &gap) {
  const GsPhilox b = gs_boot_philox(seed, stream, (uint64_t)j + 1u, 0, 0, 0);
  row = (long long)gs_boot_mulhi(b.w[0], (uint64_t)K);
  gap = (j > 0 && K > 1) ? (long long)gs_boot_mulhi(b.w[1], (uint64_t)(K - 1)) : -1;
}

// gs_boot_pick for a replica with mean block length L >= 1: row is s_j (the row a block starting at j begins with),
// gap the iid gap index; returns whether job j starts a block.
GS_BOOT_HD bool gs_boot_pick_blocked(uint64_t seed, uint64_t stream, long long j, long long K, uint64_t L, long long &row, long long &gap) {
  const GsPhilox b = gs_boot_philox(seed, stream, (uint64_t)j + 1u, 0, 0, 0);
  row = (long long)gs_boot_mulhi(b.w[0], (uint64_t)K);
  gap = (j > 0 && K > 1) ? (long long)gs_boot_mulhi(b.w[1], (uint64_t)(K - 1)) : -1;
  return j == 0 || gs_boot_mulhi(b.w[2], L) == 0;
}

// Scan key of job j: (j << 32) | s_j for a block start, 0 otherwise.  j and s_j are below 2^31, so the maximum over
// jobs 0..j is the key of b_j (job 0's key is 0 when s_0 = 0, which decodes to the same b_j = 0, s = 0).
GS_BOOT_HD long long gs_boot_block_key(bool start, long long j, long long s) { return start ? (j << 32) | s : 0; }

// Row of job j from the scanned key of its block start: (s_b + (j - b)) mod K.  The sum stays below 2^32.
GS_BOOT_HD long long gs_boot_block_row(long long key, long long j, long long K) {
  const long long b = key >> 32, s = key & 0xffffffffll;
  return (long long)((uint32_t)(s + (j - b)) % (uint32_t)K);
}

// Gap index of job j (-1: g_j = 0): the iid pick for a block start or a wrapped row, else the row's own preceding gap.
GS_BOOT_HD long long gs_boot_block_gap(bool start, long long row, long long iid_gap) { return (start || row == 0) ? iid_gap : row - 1; }

// One column of an alias table: a job whose column is c keeps row c iff floor(w3 * T / 2^64) < u, else takes row a.
struct alignas(16) GsBootAlias { uint64_t u, a; };

// The alias table of the K integer weights w (Walker / Vose, exact integers): with T = sum w_i and q_i = w_i * K
// (both below 2^63 for K < 2^31), take FIFO worklists S = {i : q_i < T} and G = {i : q_i >= T} in ascending row order;
// while both are non-empty, take s from the front of S, let g be the front of G, set U_s = q_s, A_s = g and
// q_g -= T - q_s, and move g to the back of S once q_g < T.  Every row still in G gets U_i = T, A_i = i.  Returns T and
// fills tab[K]; T = 0 (all weights 0) writes nothing.  Row m is then drawn with probability w_m / T: U_m plus the
// T - U_i of every other column i that aliases m is w_m * K.
static inline uint64_t gs_boot_alias_build(const uint32_t *w, long long K, GsBootAlias *tab) {
  uint64_t T = 0;
  for (long long i = 0; i < K; ++i) T += w[i];
  if (T == 0) return 0;
  std::vector<uint64_t> q((size_t)K);
  std::vector<long long> S, G;
  S.reserve((size_t)K); G.reserve((size_t)K);
  for (long long i = 0; i < K; ++i) {
    q[(size_t)i] = (uint64_t)w[i] * (uint64_t)K;
    (q[(size_t)i] < T ? S : G).push_back(i);
  }
  size_t s0 = 0, g0 = 0;
  while (s0 < S.size() && g0 < G.size()) {
    const long long s = S[s0++], g = G[g0];
    tab[s].u = q[(size_t)s]; tab[s].a = (uint64_t)g;
    q[(size_t)g] -= T - q[(size_t)s];
    if (q[(size_t)g] < T) { ++g0; S.push_back(g); }
  }
  for (; g0 < G.size(); ++g0) { tab[G[g0]].u = T; tab[G[g0]].a = (uint64_t)G[g0]; }   // S is empty here
  return T;
}

// Row of a job whose unweighted row (column) is c under the alias table tab with weight sum T; T = 0 is the
// unweighted replica of a mixed launch (mix -1) and keeps c.
GS_BOOT_HD long long gs_boot_alias_pick(const GsBootAlias *tab, uint64_t T, long long c, uint64_t w3) {
  if (T == 0) return c;
#ifdef __CUDA_ARCH__
  const ulonglong2 e = __ldg(reinterpret_cast<const ulonglong2 *>(tab + c));
  return gs_boot_mulhi(w3, T) < e.x ? c : (long long)e.y;
#else
  return gs_boot_mulhi(w3, T) < tab[c].u ? c : (long long)tab[c].a;
#endif
}

// gs_boot_pick_blocked of a mixed replica: row is the weighted pick (s_j when blocked), gap the iid gap index; returns
// whether job j starts a block (always true for L = 1).
GS_BOOT_HD bool gs_boot_pick_mixed(uint64_t seed, uint64_t stream, long long j, long long K, uint64_t L, const GsBootAlias *tab, uint64_t T,
                                   long long &row, long long &gap) {
  const GsPhilox b = gs_boot_philox(seed, stream, (uint64_t)j + 1u, 0, 0, 0);
  row = gs_boot_alias_pick(tab, T, (long long)gs_boot_mulhi(b.w[0], (uint64_t)K), b.w[3]);
  gap = (j > 0 && K > 1) ? (long long)gs_boot_mulhi(b.w[1], (uint64_t)(K - 1)) : -1;
  return j == 0 || gs_boot_mulhi(b.w[2], L) == 0;
}

// arrive = floor(S * gap_num / gap_den) for a gap sum S >= 0.  The caller bounds S * gap_num below 2^62
// (gs_boot_arrive_bound), so the product fits in 64 bits.
GS_BOOT_HD int gs_boot_arrive(long long S, int gap_num, int gap_den) { return (int)(S * (long long)gap_num / gap_den); }

// Largest arrival tick any replica of n jobs can reach: floor((n - 1) * max_gap * gap_num / gap_den), exactly.
GS_BOOT_HD long long gs_boot_arrive_bound(long long n, long long max_gap, int gap_num, int gap_den) {
  if (n <= 1) return 0;
  const __int128 x = (__int128)(n - 1) * max_gap * gap_num / gap_den;
  return x > (__int128)0x7fffffffffffffffll ? 0x7fffffffffffffffll : (long long)x;
}

// One segment of a profile in device form: base-time start s, real start t and gap scale num / den.
struct GsBootProfSeg {
  long long s;
  int t, num, den, reserved;
};

// Why the profile of m segments seg[] with period P breaks the rules of gs_boot_profiles (include/gsched.h), or
// nullptr when it keeps them.
static inline const char *gs_boot_profile_invalid(const gs_boot_seg *seg, int m, int P) {
  if (m < 1 || m > GS_BOOT_MAX_SEGMENTS) return "nseg must be in 1..GS_BOOT_MAX_SEGMENTS";
  if (seg[0].start != 0) return "the first segment must start at tick 0";
  for (int k = 0; k < m; ++k) {
    if (k > 0 && seg[k].start <= seg[k - 1].start) return "segment starts must be strictly increasing";
    if (seg[k].start >= 0x7fffffff) return "segment starts must be below 2^31 - 1";
    if (seg[k].gap_num < 1 || seg[k].gap_den < 1) return "every gap scale needs gap_num >= 1 and gap_den >= 1";
  }
  if (P < 0) return "the period must be >= 0";
  if (P > 0 && P <= seg[m - 1].start) return "a period must exceed the last segment's start";
  return nullptr;
}

// The device form out[m] of a valid profile (seg[m], period P): s_0 = 0, s_(k+1) = s_k + ceil((t_(k+1) - t_k) *
// den_k / num_k).  Returns B = s_m with t_m := P, the base length of one period, or 0 when P = 0.  Every s_k and B
// stay below 2^62 + 64: the t_k differences add up to less than 2^31 and each den_k is below 2^31.
static inline long long gs_boot_profile_base(const gs_boot_seg *seg, int m, int P, GsBootProfSeg *out) {
  long long s = 0;
  for (int k = 0; k < m; ++k) {
    out[k].s = s; out[k].t = seg[k].start; out[k].num = seg[k].gap_num; out[k].den = seg[k].gap_den; out[k].reserved = 0;
    if (k + 1 < m || P > 0) {
      const long long d = (long long)((k + 1 < m ? seg[k + 1].start : P) - seg[k].start);
      s += (d * seg[k].gap_den + seg[k].gap_num - 1) / seg[k].gap_num;
    }
  }
  return P > 0 ? s : 0;
}

// The last of the m segments with s <= x (x >= 0; s_0 = 0), by binary search.
template <class I>
GS_BOOT_HD int gs_boot_profile_seg(const GsBootProfSeg *seg, int m, I x) {
  int lo = 0, hi = m;                                  // seg[lo].s <= x < seg[hi].s, seg[m].s = infinity
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if ((I)seg[mid].s <= x) lo = mid; else hi = mid;
  }
  return lo;
}

// Arrival tick of base time S >= 0 under a profile (seg[m], period P, base period B; P = 0: aperiodic).  I = long long
// on the device, where the caller's bound keeps (S - s_k) * num_k below 2^62; __int128 on the host for that bound.
template <class I>
GS_BOOT_HD I gs_boot_profile_arrive(const GsBootProfSeg *seg, int m, int P, long long B, I S) {
  I q = 0;
  if (P > 0) { q = S / (I)B; S -= q * (I)B; }
  const GsBootProfSeg &g = seg[gs_boot_profile_seg(seg, m, S)];
  return q * (I)P + (I)g.t + (S - (I)g.s) * (I)g.num / (I)g.den;
}

// Largest arrival tick any profiled replica of n jobs can reach: arrive((n - 1) * max_gap), exactly; saturated at
// 2^63 - 1.
static inline long long gs_boot_profile_bound(const GsBootProfSeg *seg, int m, int P, long long B, long long n, long long max_gap) {
  if (n <= 1) return 0;
  const __int128 x = gs_boot_profile_arrive<__int128>(seg, m, P, B, (__int128)(n - 1) * max_gap);
  return x > (__int128)0x7fffffffffffffffll ? 0x7fffffffffffffffll : (long long)x;
}

#ifdef __CUDACC__
namespace {

struct GsBootRep {        // one replica's parameters as the kernel reads them
  uint64_t seed, stream;
  long long n;
  int gap_num, gap_den, M;
  uint32_t block_len;     // mean block length L (read by the blocked instantiation only)
};

struct alignas(16) GsBootMix {   // one replica's alias table as the mixed instantiations read it
  uint64_t T;                    // weight sum; 0: unweighted (mix -1)
  long long off;                 // first entry of the replica's table in tabs
};

struct GsBootProf {              // one replica's profile as the profiled instantiations read it
  long long B;                   // base length of one period (0: aperiodic)
  int period, off, nseg;         // period P, first segment in segs, segments (0: unprofiled, profile -1)
  int reserved;
};

// The I-th argument of a pack.
template <int I, class T, class... Ts>
static __device__ __forceinline__ auto gs_boot_nth(T a, Ts... rest) {
  if constexpr (I == 0) return a; else return gs_boot_nth<I - 1>(rest...);
}

// gs_boot_pick_mixed of job j of this block's replica, whose table is {T, off} = mixes[blockIdx.x] (T = 0: mix -1).
static __device__ __forceinline__ bool gs_boot_pick_in_mix(const GsBootMix *mixes, const GsBootAlias *tabs, uint64_t seed, uint64_t stream,
                                                           long long j, long long K, uint64_t L, long long &row, long long &gap) {
  const ulonglong2 m = __ldg(reinterpret_cast<const ulonglong2 *>(mixes + blockIdx.x));
  return gs_boot_pick_mixed(seed, stream, j, K, L, tabs + m.y, m.x, row, gap);
}

// out[2 b] = sum over the jobs of min(tasks, M), out[2 b + 1] = last arrival tick (0 without jobs).
// BLOCKED = false is the iid bootstrap; BLOCKED = true draws blocks of mean length R.block_len (1 gives the iid trace).
// MIXED = true picks rows (block starts when blocked) through the alias table {T, off} = mixes[b] at tabs + off, two
// parameters appended as the pack `mix` = (const GsBootMix *mixes, const GsBootAlias *tabs).  The profiled
// instantiations append (const GsBootProf *profs, const GsBootProfSeg *segs) to the pack, after the mixed pair when MIXED:
// replica b's arrivals follow the profs[b].nseg segments at segs + profs[b].off (none: the gap scale as before).  The
// other instantiations have an empty pack: their parameter list, and so their code, is the one they had before mixes.
template <bool BLOCKED, bool MIXED, class... Mix>
__global__ void __launch_bounds__(GS_BOOT_THREADS) gs_boot_kernel(const GsBootRep *reps, const JobIn *pop, const int *gaps, long long K,
                                                                 JobIn *arena, long long stride_recs, long long *out, Mix... mix) {
  constexpr bool PROFILED = sizeof...(Mix) == (MIXED ? 4 : 2);
  static_assert(sizeof...(Mix) == (MIXED ? 2 : 0) + (PROFILED ? 2 : 0),
                "the mixed instantiations take (mixes, tabs), the profiled ones (profs, segs) after them");
  __shared__ int4 stage[2 * GS_BOOT_THREADS];
  __shared__ long long warp_tot[GS_BOOT_THREADS / 32];
  __shared__ long long warp_key[BLOCKED ? GS_BOOT_THREADS / 32 : 1];
  __shared__ long long red[2][GS_BOOT_THREADS / 32];
  __shared__ GsBootProfSeg pseg[PROFILED ? GS_BOOT_MAX_SEGMENTS : 1];
  const GsBootRep R = reps[blockIdx.x];
  int4 *dst = reinterpret_cast<int4 *>(arena + stride_recs * (long long)blockIdx.x);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  long long carry = 0, spans = 0, last = 0, key_carry = 0;
  [[maybe_unused]] GsBootProf prof{};
  if constexpr (PROFILED) {                            // the replica's segments, once
    prof = gs_boot_nth<MIXED ? 2 : 0>(mix...)[blockIdx.x];
    const GsBootProfSeg *segs = gs_boot_nth<MIXED ? 3 : 1>(mix...) + prof.off;
    for (int k = threadIdx.x; k < prof.nseg; k += blockDim.x) pseg[k] = segs[k];
    __syncthreads();
  }
  for (long long j0 = 0; j0 < R.n; j0 += blockDim.x) {
    const long long j = j0 + threadIdx.x;
    const bool in = j < R.n;
    long long g = 0;
    int4 lo = make_int4(0, 0, 0, 0), hi = make_int4(0, 0, 0, 0);
    if constexpr (BLOCKED) {
      long long s = 0, gi = -1;
      bool start = false;
      if (in) {
        if constexpr (MIXED) {
          start = gs_boot_pick_in_mix(gs_boot_nth<0>(mix...), gs_boot_nth<1>(mix...), R.seed, R.stream, j, K, R.block_len, s, gi);
        } else {
          start = gs_boot_pick_blocked(R.seed, R.stream, j, K, R.block_len, s, gi);
        }
      }
      long long key = gs_boot_block_key(start, j, s);   // inclusive max-scan: lanes, then warps, then the carry
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, key, o);
        if (lane >= o) key = max(key, y);
      }
      if (lane == 31) warp_key[warp] = key;
      __syncthreads();
      long long before = key_carry;
      for (int w = 0; w < nwarps; ++w) { const long long t = warp_key[w]; before = w < warp ? max(before, t) : before; key_carry = max(key_carry, t); }
      key = max(key, before);
      if (in) {                                        // warp_key is next written after the gap scan's barrier
        const long long row = gs_boot_block_row(key, j, K);
        const long long gj = gs_boot_block_gap(start, row, gi);
        const int4 *src = reinterpret_cast<const int4 *>(pop + row);
        lo = __ldg(src); hi = __ldg(src + 1);
        if (gj >= 0) g = __ldg(gaps + gj);
      }
    } else if (in) {
      long long row, gi;
      if constexpr (MIXED) {
        gs_boot_pick_in_mix(gs_boot_nth<0>(mix...), gs_boot_nth<1>(mix...), R.seed, R.stream, j, K, 1u, row, gi);
      } else {
        gs_boot_pick(R.seed, R.stream, j, K, row, gi);
      }
      const int4 *src = reinterpret_cast<const int4 *>(pop + row);
      lo = __ldg(src); hi = __ldg(src + 1);
      if (gi >= 0) g = __ldg(gaps + gi);
    }
    long long x = g;                                   // inclusive scan: lanes, then warps, then the carry
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_tot[warp] = x;
    __syncthreads();
    long long before = carry, chunk = 0;
    for (int w = 0; w < nwarps; ++w) { const long long t = warp_tot[w]; before += w < warp ? t : 0; chunk += t; }
    carry += chunk;
    if (in) {
      int arrive;
      if constexpr (PROFILED) {
        arrive = prof.nseg > 0 ? (int)gs_boot_profile_arrive<long long>(pseg, prof.nseg, prof.period, prof.B, before + x)
                               : gs_boot_arrive(before + x, R.gap_num, R.gap_den);
      } else {
        arrive = gs_boot_arrive(before + x, R.gap_num, R.gap_den);
      }
      const long long tasks = lo.y / lo.z;
      spans += tasks < R.M ? tasks : R.M;
      last = arrive;                                   // arrivals do not decrease: the thread's latest job is its largest
      stage[2 * threadIdx.x] = make_int4(arrive, lo.y, lo.z, 0);
      stage[2 * threadIdx.x + 1] = hi;
    }
    __syncthreads();
    const long long cnt = R.n - j0 < (long long)blockDim.x ? R.n - j0 : (long long)blockDim.x;
    for (int k = threadIdx.x; k < 2 * cnt; k += blockDim.x) dst[2 * j0 + k] = stage[k];
    __syncthreads();                                   // stage and warp_tot are rewritten by the next chunk
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    spans += __shfl_down_sync(0xffffffffu, spans, o);
    last = max(last, __shfl_down_sync(0xffffffffu, last, o));
  }
  if (lane == 0) { red[0][warp] = spans; red[1][warp] = last; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < nwarps; ++w) { spans += red[0][w]; last = max(last, red[1][w]); }
    out[2 * blockIdx.x] = spans;
    out[2 * blockIdx.x + 1] = last;
  }
}

}  // namespace
#endif  // __CUDACC__

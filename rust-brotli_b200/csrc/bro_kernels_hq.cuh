// bro_kernels_hq.cuh -- CUDA kernels (sm_90a) of the quality 10 / 11 path.
//
// Stage map (the specification of every stage is its sequential form in bro_hq.cuh / bro_bsplit.cuh, executed by the CPU model
// tools/gpu_model.cpp; the kernels must reproduce it bit for bit):
//   match   k_match_all      all matches of every position over the sorted bucket lists (replaces H10's binary tree,
//                            hash_to_binary_tree.rs:437-530, and FindAllMatchesH10, hq.rs:302-417)
//   parse   k_zopfli         literal cost estimate + shortest path per parse unit (hq.rs:644-1448)
//   split   k_bs_*           BrotliSplitBlock: entropy-code refinement, FindBlocks, ClusterBlocks (block_splitter.rs)
//   maps    k_cm_*           histograms with context + BrotliClusterHistograms -> literal / distance context maps
//                            (metablock.rs:133-301, cluster.rs)
#pragma once
#include "bro_kernels.cuh"
#include "bro_hq.cuh"
#include "bro_bsplit.cuh"

namespace bro {

// ---------------------------------------------------------------------------------------------------
// All matches.  One thread per sorted entry, like k_match; the bucket neighbours (position, key, first data word) of a CTA are
// staged in shared memory, lengths are measured against global memory (L2 resident: the window).
// ---------------------------------------------------------------------------------------------------
struct MatchAllArgs {
  MatchArgs m;      // sorted list, batch geometry, dictionary (m.best unused)
  HqMatch* hqm;     // indexed by absolute position (pre-shifted by the range start)
  uint8_t* hqn;
  int quality;
  int level;        // k_match_level: which long-prefix level this pass serves
  int last_pass;    // the pass that adds the static-dictionary matches (they come after every window match)
};

// First shared-memory index in [lo, i) that is in the bucket `key` and inside the window (position >= min_pos).  The slice is sorted
// by (key, position), so both bounds are binary searches and the scan loops below test nothing but their filter word.
__device__ __forceinline__ uint32_t bucket_scan_start(const uint32_t* s_key, const uint32_t* s_pos, uint32_t lo, uint32_t i, uint32_t key,
                                                     uint32_t min_pos) {
  uint32_t a = lo, b = i;
  while (a < b) {
    const uint32_t mid = (a + b) >> 1;
    if (s_key[mid] < key) a = mid + 1; else b = mid;
  }
  b = i;
  while (a < b) {
    const uint32_t mid = (a + b) >> 1;
    if (s_pos[mid] < min_pos) a = mid + 1; else b = mid;
  }
  return a;
}

template <int DEPTH>
__global__ void __launch_bounds__(MATCH_THREADS) k_match_all(MatchAllArgs A) {
  extern __shared__ __align__(16) uint32_t smem[];
  __shared__ __align__(8) uint64_t s_bar;
  const MatchArgs& a = A.m;
  constexpr uint32_t E = MATCH_THREADS + (uint32_t)DEPTH;
  uint32_t* s_pos = smem;
  uint32_t* s_key = smem + E;
  uint32_t* s_d0 = smem + 2 * E;
  const int64_t j0 = (int64_t)blockIdx.x * MATCH_THREADS - DEPTH;
  match_stage_positions(a, j0, E, s_pos, &s_bar);  // TMA bulk copy of the CTA's slice of the sorted list
  for (uint32_t i = threadIdx.x; i < E; i += MATCH_THREADS) {
    const uint32_t pos = s_pos[i];
    uint32_t key = 0xFFFFFFFFu, w0 = 0;
    if (pos != 0xFFFFFFFFu) {
      const uint8_t* p = a.data + a.origin + pos;
      w0 = ldu32(p);
      key = hash_key_from_words(a.hash_type, a.key_bits, w0, (uint32_t)p[4]);
    }
    s_key[i] = key; s_d0[i] = w0;
  }
  __syncthreads();
  const uint32_t i = threadIdx.x + (uint32_t)DEPTH;
  const uint32_t prel = s_pos[i];
  if (prel == 0xFFFFFFFFu || prel < a.payload_begin) return;
  const uint32_t p = a.origin + prel;
  const uint8_t* cur = a.data + p;
  const uint32_t maxl = bmin(a.lcap, a.n - p);
  const uint32_t max_backward = bmin(p, a.max_backward);
  HqMatchList L;
  hq_list_init(L);
  if (a.n - p >= 8) {
    hq_short_matches(cur, maxl, max_backward, hq_short_back(A.quality), L);
    if (L.best_len < maxl) {
      const uint32_t key = s_key[i], w0 = s_d0[i];
      const uint32_t lo = j0 < 0 ? bmax(i - (uint32_t)DEPTH, (uint32_t)(-j0)) : i - (uint32_t)DEPTH;  // (entries in front of the batch are void)
      const uint32_t start = bucket_scan_start(s_key, s_pos, lo, i, key, prel > max_backward ? prel - max_backward : 0u);
      for (uint32_t ci = i; ci-- > start;) {
        if (s_d0[ci] != w0) continue;
        if (!hq_bucket_candidate(cur, prel - s_pos[ci], maxl, L)) break;
      }
    }
    if (a.use_dict && A.last_pass) hq_dict_matches(a.dict, cur, a.n - p, L);
  }
  A.hqn[p] = (uint8_t)L.n;
  HqMatch* out = A.hqm + (size_t)p * HQ_MAXM;
  for (uint32_t k = 0; k < L.n; ++k) out[k] = L.m[k];
}

// One long-prefix level (bro_hq.cuh): the batch has been sorted by the 15-bit key of the level's hash; a thread scans the
// HQ_LEVEL_DEPTH entries in front of its own, keeps those whose 32 check bits agree, builds the level's Pareto front and merges
// it into the list the earlier passes left in hqm / hqn.
template <int DEPTH>
__global__ void __launch_bounds__(MATCH_THREADS) k_match_level(MatchAllArgs A) {
  extern __shared__ __align__(16) uint32_t smem[];
  __shared__ __align__(8) uint64_t s_bar;
  const MatchArgs& a = A.m;
  constexpr uint32_t E = MATCH_THREADS + (uint32_t)DEPTH;
  uint32_t* s_pos = smem;
  uint32_t* s_key = smem + E;
  uint32_t* s_chk = smem + 2 * E;
  const uint32_t nb8 = hq_level_bytes(A.level);
  const int64_t j0 = (int64_t)blockIdx.x * MATCH_THREADS - DEPTH;
  match_stage_positions(a, j0, E, s_pos, &s_bar);
  for (uint32_t i = threadIdx.x; i < E; i += MATCH_THREADS) {
    const uint32_t pos = s_pos[i];
    uint32_t key = 0xFFFFFFFFu, chk = 0;
    if (pos != 0xFFFFFFFFu) {
      const uint8_t* q = a.data + a.origin + pos;
      const uint64_t h = hq_level_hash_with([q](uint32_t k) { return ldu64(q + k); }, nb8);
      key = hq_level_key(h, a.key_bits);
      chk = (uint32_t)h;
    }
    s_key[i] = key; s_chk[i] = chk;
  }
  __syncthreads();
  const uint32_t i = threadIdx.x + (uint32_t)DEPTH;
  const uint32_t prel = s_pos[i];
  if (prel == 0xFFFFFFFFu || prel < a.payload_begin) return;
  const uint32_t p = a.origin + prel;
  const bool search = a.n - p >= nb8 + 8u;
  if (!search && !(A.last_pass && a.use_dict && a.n - p >= 8)) return;  // nothing to add to this position's list
  const uint8_t* cur = a.data + p;
  const uint32_t maxl = bmin(a.lcap, a.n - p);
  const uint32_t max_backward = bmin(p, a.max_backward);
  HqMatch* out = A.hqm + (size_t)p * HQ_MAXM;
  HqMatchList L;
  L.n = A.hqn[p];
  L.best_len = 1;
  for (uint32_t k = 0; k < L.n; ++k) L.m[k] = out[k];
  if (L.n) L.best_len = L.m[L.n - 1].lc & 0xFFFFu;
  if (search) {
    HqMatchList B;
    hq_list_init(B);
    const uint32_t key = s_key[i], chk = s_chk[i];
    const uint32_t lo = j0 < 0 ? bmax(i - (uint32_t)DEPTH, (uint32_t)(-j0)) : i - (uint32_t)DEPTH;
    const uint32_t start = bucket_scan_start(s_key, s_pos, lo, i, key, prel > max_backward ? prel - max_backward : 0u);
    for (uint32_t ci = i; ci-- > start;) {
      if (s_chk[ci] != chk) continue;
      if (!hq_bucket_candidate(cur, prel - s_pos[ci], maxl, B)) break;
    }
    hq_merge_lists(L, B);
  }
  if (a.use_dict && A.last_pass && a.n - p >= 8) hq_dict_matches(a.dict, cur, a.n - p, L);
  A.hqn[p] = (uint8_t)L.n;
  for (uint32_t k = 0; k < L.n; ++k) out[k] = L.m[k];
}

// ---------------------------------------------------------------------------------------------------
// Shortest-path parse: one unit per warp, lane 0 runs the sequential routine of bro_hq.cuh (the node array of a unit is a
// chain of dependent updates; the parallelism is across the units of a chunk).
// ---------------------------------------------------------------------------------------------------
#define BS_NONE_DEV 0xFFFFFFFFu
#define HQ_SCRATCH_WORDS 4096u  // per unit: HqCostModel (769) | literal-cost histograms (768) | pass-1 statistics (1024) | literal costs (256) | warm-up cache (4) | pooled statistics (1024)

struct ZopfliArgs {
  ZNode* nodes;       // [num_units][unit + 1]
  uint32_t* pre;      // [num_units][unit + 1]
  uint32_t* scratch;  // [num_units][HQ_SCRATCH_WORDS]
};

// One unit per warp (lane 0 runs the node sweep).  phase 1: warm-up cache, literal costs, shortest path with the initial cost
// model; at quality 11 the command statistics stay in the unit's scratch.  phase 2 (quality 11 only): the statistics of the unit's
// HQ_STATS_SPAN window are pooled (all lanes), costs from them, second shortest path.
__global__ void __launch_bounds__(32) k_zopfli(Workspace W, ZopfliArgs Z, int phase) {
  const uint32_t u = blockIdx.x;
  if (u >= W.num_units) return;
  const EncParams& P = W.P;
  const uint32_t s = u * P.unit, e = bmin(P.n, s + P.unit);
  uint32_t* scr = Z.scratch + (size_t)u * HQ_SCRATCH_WORDS;
  HqCostModel* model = reinterpret_cast<HqCostModel*>(scr);
  uint32_t* hist = scr + 769;
  uint32_t* stats = scr + 769 + 768;
  uint32_t* cost_literal = scr + 769 + 768 + 1024;
  int32_t* warm_dc = reinterpret_cast<int32_t*>(scr + 769 + 768 + 1024 + 256);
  uint32_t* pooled = scr + 769 + 768 + 1024 + 256 + 4;
  if (phase == 2) {  // pool the first-pass statistics of the window (they are complete: phase 1 was a kernel of its own)
    const uint32_t gu = bmax(1u, HQ_STATS_SPAN / P.unit);
    const uint32_t mb_u0 = u / P.mb_units * P.mb_units;
    const uint32_t g0 = mb_u0 + (u - mb_u0) / gu * gu, g1 = bmin(bmin(W.num_units, g0 + gu), mb_u0 + P.mb_units);
    for (uint32_t k = threadIdx.x; k < HQ_STATS_WORDS; k += 32u) {
      uint32_t acc = 0;
      for (uint32_t v = g0; v < g1; ++v) acc += Z.scratch[(size_t)v * HQ_SCRATCH_WORDS + 769 + 768 + k];
      pooled[k] = acc;
    }
    __syncwarp();
  }
  // every lane runs the node sweep on the same data (same loads, same stores: no more issue slots than one lane would take), so
  // that the 16 distance-cache probes of UpdateNodes can be spread over the lanes (hq_update_nodes)
  uint32_t* pre = Z.pre + (size_t)u * (P.unit + 1);
  HqUnit U;
  U.data = W.data; U.ustart = s; U.len = e - s; U.abs_base = P.abs_base; U.max_backward = P.max_backward; U.quality = P.quality;
  U.model = model; U.lit_pre = pre; U.start_dc = warm_dc; U.nodes = Z.nodes + (size_t)u * (P.unit + 1);
  hq_model_initial(model, W.lut);
  RawCmd* out = W.raw + (size_t)u * (P.unit / 2 + 1);
  const bool two = P.quality >= 11;
  uint32_t tail, ncopy, ncmd;
  if (phase == 1) {
    const uint32_t mb_span = P.unit * P.mb_units, mb_lo = s / mb_span * mb_span, mb_hi = bmin(P.n, mb_lo + mb_span);
    warm_dc[0] = warm_dc[1] = warm_dc[2] = warm_dc[3] = 0x3fffffff;
    if ((u % P.mb_units) != 0 && s >= HQ_WARMUP_BYTES) {  // incoming distance cache (bro_hq.cuh:hq_warm_start_cache)
      const int32_t unknown[4] = {0x3fffffff, 0x3fffffff, 0x3fffffff, 0x3fffffff};
      HqUnit V = U;
      V.ustart = s - HQ_WARMUP_BYTES; V.len = HQ_WARMUP_BYTES; V.start_dc = unknown;
      hq_literal_costs_unit(W.data + V.ustart, V.len, V.ustart - mb_lo, mb_hi - s, W.lut, hist, pre);
      hq_warm_start_cache(V, W.hqm, W.hqn, out, warm_dc);
    }
    hq_literal_costs_unit(W.data + s, U.len, s - mb_lo, mb_hi - e, W.lut, hist, pre);
    if (two) for (uint32_t i = 0; i < HQ_STATS_WORDS; ++i) stats[i] = 0;
    ncmd = hq_zopfli_unit(U, W.hqm, W.hqn, out, &tail, &ncopy, two ? stats : nullptr);
  } else {
    hq_model_from_stats(model, pooled, W.lut, W.data + s, U.len, cost_literal, pre);
    ncmd = hq_zopfli_unit(U, W.hqm, W.hqn, out, &tail, &ncopy, nullptr);
  }
  W.unit_ncmd[u] = ncmd;
  W.unit_tail[u] = tail;
  W.unit_ncopy[u] = ncopy;
}

}  // namespace bro

namespace bro {

// ===================================================================================================
// Histogram clustering on the device (specification: bs_combine / bs_best_cluster in bro_bsplit.cuh).
// One warp runs the greedy control flow of a problem with warp-uniform scalars; the population costs -- the only heavy
// part -- are computed by all 32 lanes.  Problems (batches of 64 histograms, then the survivors of all batches) run in
// parallel on different warps.
// ===================================================================================================
#define FULLMASK 0xffffffffu

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULLMASK, v, o);
  return v;
}
__device__ __forceinline__ uint32_t warp_sum_u32(uint32_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULLMASK, v, o);
  return v;
}
__device__ __forceinline__ uint32_t warp_max_u32(uint32_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(FULLMASK, v, o));
  return v;
}

// bs_pop_cost_q16(h, g, A) by a whole warp (A is a multiple of 32).  s_dh: 18 words of shared memory owned by the warp.
// Every lane returns the result.
__device__ uint64_t warp_pop_cost(const uint32_t* h, const uint32_t* g, uint32_t A, const uint32_t* lut, uint32_t* s_dh) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t total = 0, count = 0, s4[5] = {0, 0, 0, 0, 0};
  for (uint32_t base = 0; base < A; base += 32) {
    const uint32_t v = h[base + lane] + (g ? g[base + lane] : 0u);
    total += v;
    uint32_t nz = __ballot_sync(FULLMASK, v != 0);
    while (nz && count < 5) {
      const int src = __ffs((int)nz) - 1;
      s4[count++] = __shfl_sync(FULLMASK, v, src);
      nz &= nz - 1;
    }
  }
  total = warp_sum_u32(total);
  if (total == 0 || count == 1) return 12ull << 16;
  if (count == 2) return (20ull + total) << 16;
  if (count == 3) {
    const uint32_t mx = bmax(s4[0], bmax(s4[1], s4[2]));
    return (28ull + 2ull * total - mx) << 16;
  }
  if (count == 4) {
    for (int i = 0; i < 4; ++i)
      for (int j = i + 1; j < 4; ++j)
        if (s4[j] > s4[i]) { const uint32_t t = s4[j]; s4[j] = s4[i]; s4[i] = t; }
    const uint32_t h23 = s4[2] + s4[3];
    const uint32_t mx = bmax(h23, s4[0]);
    return (37ull + 3ull * h23 + 2ull * (s4[0] + s4[1]) - mx) << 16;
  }
  __syncwarp();
  if (lane < 18) s_dh[lane] = 0;
  __syncwarp();
  const uint32_t log2total = log2_q16(lut, total);
  uint64_t bits = 0, run_bits = 0;
  uint32_t max_depth = 1, run = 0, dh0 = 0, dh17 = 0;
  for (uint32_t base = 0; base < A; base += 32) {
    const uint32_t v = h[base + lane] + (g ? g[base + lane] : 0u);
    if (v) {
      const uint32_t log2p = log2total - log2_q16(lut, v);
      uint32_t depth = (log2p + 32768u) >> 16;
      bits += (uint64_t)v * log2p;
      if (depth > 15) depth = 15;
      max_depth = bmax(max_depth, depth);
      atomicAdd(&s_dh[depth], 1u);
    }
    // zero runs, in index order (warp-uniform walk over the zero mask of this group)
    const uint32_t zm = __ballot_sync(FULLMASK, v == 0);
    uint32_t pos = 0;
    while (pos < 32) {
      const uint32_t rest = zm >> pos;
      if (rest & 1u) {
        const uint32_t inv = ~rest;
        const uint32_t streak = inv ? bmin((uint32_t)(__ffs((int)inv) - 1), 32u - pos) : 32u - pos;
        run += streak;
        pos += streak;
        if (pos < 32) {  // the run ended inside the group
          if (run < 3) dh0 += run;
          else { uint32_t r = run - 2; while (r > 0) { ++dh17; run_bits += 3ull << 16; r >>= 3; } }
          run = 0;
        }
      } else {
        if (run) {  // a run carried from the previous group ends at this group's first symbol
          if (run < 3) dh0 += run;
          else { uint32_t r = run - 2; while (r > 0) { ++dh17; run_bits += 3ull << 16; r >>= 3; } }
          run = 0;
        }
        const uint32_t streak = rest ? bmin((uint32_t)(__ffs((int)rest) - 1), 32u - pos) : 32u - pos;
        pos += streak;
      }
    }
  }
  // a run still open here is the tail of the histogram: not coded
  bits = warp_sum_u64(bits) + run_bits;
  max_depth = warp_max_u32(max_depth);
  __syncwarp();
  if (lane == 0) { s_dh[0] += dh0; s_dh[17] += dh17; }
  __syncwarp();
  bits += (uint64_t)(18 + 2 * max_depth) << 16;
  const uint32_t c = lane < 18 ? s_dh[lane] : 0u;
  const uint64_t sx = warp_sum_u64(c ? xlog2x_q16(lut, c) : 0ull);
  const uint32_t t = warp_sum_u32(c);
  __syncwarp();
  return bits + bits_entropy_q16(sx, t, lut);
}

struct ClProblem {   // one clustering problem
  uint32_t A, n;           // alphabet, number of input histograms
  const uint32_t* in;      // [n][A] inputs (kept intact)
  uint32_t* work;          // [n][A] clusters, merged in place (slot = id)
  uint64_t* cost;          // [n]
  uint32_t* size;          // [n]
  uint32_t* sym;           // [n] cluster of every input
  uint32_t* clusters;      // [n] survivor lists (batch b at [64 b ..)), then the final list at [0 ..)
  uint32_t* bj;            // [n] best partner of row id
  int64_t* bd;             // [n] its cost_diff
  uint32_t* nsurv;         // [ceil(n / 64)] survivors per batch ; nsurv[-1] (one word in front) = final cluster count
  uint32_t batch_max, final_max;
};

__device__ __forceinline__ int64_t warp_pair_diff(const ClProblem& C, uint32_t a, uint32_t b, const uint32_t* lut, uint32_t* s_dh) {
  return (int64_t)warp_pop_cost(C.work + (size_t)a * C.A, C.work + (size_t)b * C.A, C.A, lut, s_dh) - (int64_t)C.cost[a] - (int64_t)C.cost[b] +
         bs_half_cluster_cost_diff_q16(C.size[a], C.size[b], lut);
}
__device__ void warp_recompute_row(const ClProblem& C, const uint32_t* clusters, uint32_t n, uint32_t a, const uint32_t* lut, uint32_t* s_dh) {
  uint32_t bj = BS_NONE_DEV;
  int64_t bd = 0;
  for (uint32_t q = 0; q < n; ++q) {
    const uint32_t b = clusters[q];
    if (b <= a) continue;
    const int64_t d = warp_pair_diff(C, a, b, lut, s_dh);
    if (bj == BS_NONE_DEV || d < bd) { bd = d; bj = b; }
  }
  if ((threadIdx.x & 31) == 0) { C.bj[a] = bj; C.bd[a] = bd; }
  __syncwarp();
}
// bs_combine by one CTA of CLB_WARPS warps.  clusters[0..n) ascending ids; symbols[0..nsym) relabelled.  Returns the new count
// (every thread).  The control flow is CTA uniform; what is spread over the warps is the one expensive thing, the population cost
// of candidate pairs (a launch list of q10 had this stage, then run by a single warp per problem, at 41 % of all kernel time):
//   * first fill: row q belongs to warp q % CLB_WARPS,
//   * after a merge: the rows that only have to look at the new cluster are spread the same way, the rows whose best partner
//     disappeared are marked and then recomputed one after the other with their partners spread over the warps.
// A row's best partner is "smallest diff, smallest id on ties" in every variant, so the result does not depend on the mapping.
#define CLB_WARPS 8
#define CL_DIRTY 0xFFFFFFFEu
struct ClbShared {
  uint32_t dh[CLB_WARPS][18];
  int64_t red_d[CLB_WARPS];
  uint32_t red_j[CLB_WARPS];
};
__device__ void cta_recompute_row(const ClProblem& C, const uint32_t* clusters, uint32_t n, uint32_t a, const uint32_t* lut, ClbShared& S) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t bj = BS_NONE_DEV;
  int64_t bd = 0;
  for (uint32_t q = wid; q < n; q += CLB_WARPS) {
    const uint32_t b = clusters[q];
    if (b <= a) continue;
    const int64_t d = warp_pair_diff(C, a, b, lut, S.dh[wid]);
    if (bj == BS_NONE_DEV || d < bd) { bd = d; bj = b; }
  }
  if (lane == 0) { S.red_d[wid] = bd; S.red_j[wid] = bj; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (uint32_t w = 0; w < CLB_WARPS; ++w) {
      const uint32_t oj = S.red_j[w];
      if (oj == BS_NONE_DEV) continue;
      const int64_t od = S.red_d[w];
      if (bj == BS_NONE_DEV || od < bd || (od == bd && oj < bj)) { bd = od; bj = oj; }
    }
    C.bj[a] = bj; C.bd[a] = bd;
  }
  __syncthreads();
}
__device__ uint32_t cta_combine(const ClProblem& C, uint32_t* clusters, uint32_t n, uint32_t* symbols, uint32_t nsym, uint32_t max_clusters,
                                const uint32_t* lut, ClbShared& S) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (n <= 1) return n;
  __syncthreads();
  for (uint32_t q = wid; q < n; q += CLB_WARPS) warp_recompute_row(C, clusters, n, clusters[q], lut, S.dh[wid]);
  bool forced = false;
  while (n > 1) {
    __syncthreads();
    // best row: smallest diff, then smallest partner distance, then smallest id (every warp finds the same one)
    uint32_t a = BS_NONE_DEV, ad = 0;
    int64_t abd = 0;
    for (uint32_t q = lane; q < n; q += 32) {
      const uint32_t r = clusters[q];
      const uint32_t j = C.bj[r];
      if (j == BS_NONE_DEV) continue;
      const int64_t d = C.bd[r];
      if (a == BS_NONE_DEV || d < abd || (d == abd && j - r < ad)) { a = r; abd = d; ad = j - r; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint32_t oa = __shfl_xor_sync(FULLMASK, a, o), oad = __shfl_xor_sync(FULLMASK, ad, o);
      const int64_t obd = __shfl_xor_sync(FULLMASK, abd, o);
      if (oa != BS_NONE_DEV && (a == BS_NONE_DEV || obd < abd || (obd == abd && (oad < ad || (oad == ad && oa < a))))) { a = oa; abd = obd; ad = oad; }
    }
    if (a == BS_NONE_DEV) break;
    if (!forced && abd >= 0) forced = true;
    if (forced && n <= max_clusters) break;
    const uint32_t b = C.bj[a];
    __syncthreads();
    for (uint32_t s = threadIdx.x; s < C.A; s += CLB_WARPS * 32) C.work[(size_t)a * C.A + s] += C.work[(size_t)b * C.A + s];
    for (uint32_t i = threadIdx.x; i < nsym; i += CLB_WARPS * 32) if (symbols[i] == b) symbols[i] = a;
    __syncthreads();
    const uint64_t nc = warp_pop_cost(C.work + (size_t)a * C.A, nullptr, C.A, lut, S.dh[wid]);  // (every warp, same value)
    if (wid == 0) {
      if (lane == 0) { C.cost[a] = nc; C.size[a] += C.size[b]; }
      // remove b from the list (order preserved)
      uint32_t pos = 0;
      for (uint32_t q0 = 0; q0 < n; q0 += 32) {
        const uint32_t q = q0 + lane;
        const uint32_t hit = __ballot_sync(FULLMASK, q < n && clusters[q] == b);
        if (hit) { pos = q0 + (uint32_t)__ffs((int)hit) - 1u; break; }
      }
      for (uint32_t q0 = pos; q0 + 1 < n; q0 += 32) {
        const uint32_t q = q0 + lane;
        uint32_t v = 0;
        if (q + 1 < n) v = clusters[q + 1];
        __syncwarp();
        if (q + 1 < n) clusters[q] = v;
        __syncwarp();
      }
    }
    --n;
    __syncthreads();
    for (uint32_t q = wid; q < n; q += CLB_WARPS) {
      const uint32_t r = clusters[q];
      if (r < a) {
        const uint32_t j = C.bj[r];
        if (j == a || j == b) { if (lane == 0) C.bj[r] = CL_DIRTY; }
        else {
          const int64_t d = warp_pair_diff(C, r, a, lut, S.dh[wid]);
          if (lane == 0 && (j == BS_NONE_DEV || d < C.bd[r] || (d == C.bd[r] && a < j))) { C.bd[r] = d; C.bj[r] = a; }
        }
      } else if (r > a && r < b) {
        if (C.bj[r] == b && lane == 0) C.bj[r] = CL_DIRTY;
      }
    }
    __syncthreads();
    for (uint32_t q = 0; q < n; ++q) {
      const uint32_t r = clusters[q];
      if (r != a && C.bj[r] == CL_DIRTY) cta_recompute_row(C, clusters, n, r, lut, S);
    }
    cta_recompute_row(C, clusters, n, a, lut, S);
  }
  __syncthreads();
  return n;
}

#define CL_WARPS 4
// work = in, cost = pop cost, size = 1, sym = id: one warp per histogram
__device__ __forceinline__ void cl_prepare_one(const ClProblem& C, uint32_t i, const uint32_t* lut, uint32_t* s_dh) {
  const uint32_t lane = threadIdx.x & 31;
  for (uint32_t s = lane; s < C.A; s += 32) C.work[(size_t)i * C.A + s] = C.in[(size_t)i * C.A + s];
  __syncwarp();
  const uint64_t c = warp_pop_cost(C.in + (size_t)i * C.A, nullptr, C.A, lut, s_dh);
  if (lane == 0) { C.cost[i] = c; C.size[i] = 1; C.sym[i] = i; }
}
// one batch of <= 64 histograms (whole CTA)
__device__ __forceinline__ void cl_batch_one(const ClProblem& C, uint32_t batch, const uint32_t* lut, ClbShared& S) {
  const uint32_t i0 = batch * 64u, k = bmin(64u, C.n - i0);
  for (uint32_t j = threadIdx.x; j < k; j += CLB_WARPS * 32) C.clusters[i0 + j] = i0 + j;
  __syncthreads();
  const uint32_t nn = cta_combine(C, C.clusters + i0, k, C.sym + i0, k, C.batch_max, lut, S);
  if (threadIdx.x == 0) C.nsurv[batch] = nn;
}
// survivors of all batches -> one list, final combine (whole CTA)
__device__ __forceinline__ void cl_final_one(const ClProblem& C, const uint32_t* lut, ClbShared& S) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nbatch = (C.n + 63) / 64;
  uint32_t nc = 0;
  for (uint32_t b = 0; b < nbatch; ++b) {  // compaction towards the front never overtakes its source (warp 0 moves, everyone counts)
    const uint32_t k = C.nsurv[b];
    if (threadIdx.x < 32) {
      uint32_t v0 = 0, v1 = 0;
      if (lane < k) v0 = C.clusters[b * 64u + lane];
      if (lane + 32 < k) v1 = C.clusters[b * 64u + lane + 32];
      __syncwarp();
      if (lane < k) C.clusters[nc + lane] = v0;
      if (lane + 32 < k) C.clusters[nc + lane + 32] = v1;
      __syncwarp();
    }
    nc += k;
  }
  __syncthreads();
  nc = cta_combine(C, C.clusters, nc, C.sym, C.n, C.final_max, lut, S);
  if (threadIdx.x == 0) C.nsurv[-1] = nc;
}
// bs_best_cluster for input i: nearest of the final clusters, first in list order on ties
__device__ __forceinline__ void cl_assign_one(const ClProblem& C, uint32_t i, const uint32_t* lut, uint32_t* s_dh) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nc = C.nsurv[-1];
  const uint32_t* histo = C.in + (size_t)i * C.A;
  uint32_t total = 0;
  for (uint32_t s = lane; s < C.A; s += 32) total += histo[s];
  total = warp_sum_u32(total);
  uint32_t best = C.clusters[0];
  if (total != 0) {
    int64_t best_bits = 0;
    for (uint32_t j = 0; j < nc; ++j) {
      const uint32_t c = C.clusters[j];
      const int64_t bits = (int64_t)warp_pop_cost(histo, C.work + (size_t)c * C.A, C.A, lut, s_dh) - (int64_t)C.cost[c];
      if (j == 0 || bits < best_bits) { best_bits = bits; best = c; }
    }
  }
  if (lane == 0) C.sym[i] = best;
}

}  // namespace bro

namespace bro {

// ===================================================================================================
// BrotliSplitBlock on the device.  Per (metablock m, category cat): literals / commands / distance symbols.
// ===================================================================================================
struct BsMeta {
  uint32_t count;     // symbols
  uint32_t nh;        // entropy codes (histograms) in use
  uint32_t nseg;      // FindBlocks segments
  uint32_t nb;        // blocks (runs of equal ids)
  uint32_t simple;    // fewer than 128 symbols: one block, nothing to do
  uint32_t pad_[3];
};
struct BsWs {  // device view of one lane's block-split workspace; every array is [num_mb][...] with the three categories side by side
  uint32_t cap[3], maxb[3], segc[3];   // per-category capacities: symbols, blocks, segments
  uint32_t cap_sum, maxb_sum, segc_sum, bh_sum;  // bh_sum = maxb0 * 256 + maxb1 * 704 + maxb2 * dist_A
  uint32_t dist_A, hist_stride;                  // hist_stride = 100 * (256 + 704 + dist_A)
  BsMeta* meta;          // [num_mb][3]
  uint8_t* blockid;      // [num_mb][cap_sum]
  uint32_t* signal;      // [num_mb][cap_sum][4]
  uint32_t* hist;        // [num_mb][100 * 1024]
  uint32_t* icost;       // [num_mb][100 * 1024]
  uint32_t* firstpos;    // [num_mb][3][128]
  uint8_t* fmap;         // [num_mb][segc_sum][128]  backward map of every segment
  uint8_t* enter;        // [num_mb][segc_sum]       id at the first symbol behind the segment
  uint32_t* bstart;      // [num_mb][maxb_sum]  first symbol of each block (+ nb: count)
  uint32_t* bh_in;       // [num_mb][bh_sum]    block histograms
  uint32_t* bh_work;     // [num_mb][bh_sum]
  uint64_t* ccost;       // [num_mb][maxb_sum]
  uint32_t *csize, *hsym, *clusters, *bj;   // [num_mb][maxb_sum]
  int64_t* bd;           // [num_mb][maxb_sum]
  uint32_t* nsurv;       // [num_mb][3][maxb_max / 64 + 2]   (slot 0 = final count)
  uint32_t nsurv_stride;
};
__device__ __forceinline__ uint32_t bs_off(const uint32_t* v, int cat) { return cat == 0 ? 0u : (cat == 1 ? v[0] : v[0] + v[1]); }
__device__ __forceinline__ uint32_t bs_bh_off(const BsWs& B, int cat) { return cat == 0 ? 0u : (cat == 1 ? B.maxb[0] * 256u : B.maxb[0] * 256u + B.maxb[1] * 704u); }  // (the distance part is last)
__device__ __forceinline__ uint32_t bs_hist_off(int cat) { return cat == 0 ? 0u : (cat == 1 ? 100u * 256u : 100u * 256u + 100u * 704u); }  // (the distance part is last)

struct BsCat {  // one (metablock, category) problem
  const uint16_t* syms;
  uint32_t mask;
  BsParams p;
  BsMeta* meta;
  uint8_t* blockid;
  uint32_t* signal;
  uint32_t *hist, *icost;
  uint32_t* firstpos;
  uint32_t* bstart;
  uint32_t maxb;
};
__device__ __forceinline__ BsCat bs_cat(const Workspace& W, const BsWs& B, uint32_t m, int cat) {
  BsCat c;
  const MBDesc& mb = W.mb[m];
  c.p = bs_params(cat, B.dist_A);
  if (cat == 0) { c.syms = W.lit_syms + mb.start; c.mask = 0xFFu; }
  else if (cat == 1) { c.syms = W.cmd_syms + (size_t)m * W.cmd_cap; c.mask = 0x3FFu; }
  else { c.syms = W.dist_syms + (size_t)m * W.cmd_cap; c.mask = 0x3FFu; }
  c.meta = B.meta + (size_t)m * 3 + cat;
  c.blockid = B.blockid + (size_t)m * B.cap_sum + bs_off(B.cap, cat);
  c.signal = B.signal + ((size_t)m * B.cap_sum + bs_off(B.cap, cat)) * 4;
  c.hist = B.hist + (size_t)m * B.hist_stride + bs_hist_off(cat);
  c.icost = B.icost + (size_t)m * B.hist_stride + bs_hist_off(cat);
  c.firstpos = B.firstpos + ((size_t)m * 3 + cat) * 128;
  c.bstart = B.bstart + (size_t)m * B.maxb_sum + bs_off(B.maxb, cat);
  c.maxb = B.maxb[cat];
  return c;
}
__device__ __forceinline__ ClProblem bs_cluster_problem(const Workspace& W, const BsWs& B, uint32_t m, int cat) {
  ClProblem C;
  const size_t bo = (size_t)m * B.maxb_sum + bs_off(B.maxb, cat);
  C.A = bs_params(cat, B.dist_A).A;
  C.n = B.meta[(size_t)m * 3 + cat].nb;
  C.in = B.bh_in + (size_t)m * B.bh_sum + bs_bh_off(B, cat);
  C.work = B.bh_work + (size_t)m * B.bh_sum + bs_bh_off(B, cat);
  C.cost = B.ccost + bo; C.size = B.csize + bo; C.sym = B.hsym + bo; C.clusters = B.clusters + bo; C.bj = B.bj + bo; C.bd = B.bd + bo;
  C.nsurv = B.nsurv + ((size_t)m * 3 + cat) * B.nsurv_stride + 1;
  C.batch_max = 64;
  C.final_max = 256;
  return C;
}

// grid (num_mb, 3), 128 threads: symbol count, number of entropy codes, histograms cleared
__global__ void __launch_bounds__(128) k_bs_setup(Workspace W, BsWs B) {
  const uint32_t m = blockIdx.x;
  const int cat = (int)blockIdx.y;
  const BsCat c = bs_cat(W, B, m, cat);
  const MBDesc& mb = W.mb[m];
  const uint32_t count = cat == 0 ? mb.nlit : (cat == 1 ? mb.ncmd : mb.ndist);
  const uint32_t nh = count < 128 ? 1u : bs_num_histograms(count, c.p);
  for (uint32_t i = threadIdx.x; i < nh * c.p.A; i += blockDim.x) c.hist[i] = 0;
  if (threadIdx.x == 0) {
    BsMeta t;
    t.count = count; t.nh = nh; t.nseg = (count + BS_SEG - 1) / BS_SEG; t.nb = 1; t.simple = count < 128 ? 1u : 0u;
    t.pad_[0] = t.pad_[1] = t.pad_[2] = 0;
    *c.meta = t;
  }
}
// InitialEntropyCodes + RefineEntropyCodes: one thread per sample stride; grid (x, num_mb, 3)
__global__ void __launch_bounds__(256) k_bs_sample(Workspace W, BsWs B) {
  const uint32_t m = blockIdx.y;
  const int cat = (int)blockIdx.z;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  if (t.simple) return;
  const uint32_t iters = bs_refine_iters(t.count, t.nh, c.p.stride);
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < t.nh + iters; k += gridDim.x * blockDim.x) {
    uint32_t pos, h;
    if (k < t.nh) { h = k; pos = bs_initial_pos(k, t.nh, t.count, c.p.stride); }
    else { h = (k - t.nh) % t.nh; pos = bs_refine_pos(k - t.nh, t.count, c.p.stride); }
    uint32_t* hh = c.hist + (size_t)h * c.p.A;
    for (uint32_t j = 0; j < c.p.stride; ++j) atomicAdd(&hh[c.syms[pos + j] & c.mask], 1u);
  }
}
// insert-cost table of the current codes: grid (num_mb, 3), 256 threads
__global__ void __launch_bounds__(256) k_bs_icost(Workspace W, BsWs B) {
  __shared__ uint32_t s_lt[BS_MAX_HIST];
  const uint32_t m = blockIdx.x;
  const int cat = (int)blockIdx.y;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  if (t.simple || t.nh <= 1) return;
  const uint32_t A = c.p.A, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (uint32_t k = wid; k < t.nh; k += 8) {
    uint32_t tot = 0;
    for (uint32_t s = lane; s < A; s += 32) tot += c.hist[(size_t)k * A + s];
    tot = warp_sum_u32(tot);
    if (lane == 0) s_lt[k] = log2_q16(W.lut, tot);
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < A * t.nh; i += blockDim.x) {
    const uint32_t s = i / t.nh, k = i % t.nh;
    c.icost[i] = bs_insert_cost(s_lt[k], c.hist[(size_t)k * A + s], W.lut);
  }
}
// FindBlocks forward pass: one warp per segment, lane l owns codes l, l + 32, l + 64, l + 96.  grid (segments, num_mb, 3)
__global__ void __launch_bounds__(32) k_bs_forward(Workspace W, BsWs B) {
  const uint32_t m = blockIdx.y;
  const int cat = (int)blockIdx.z;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  if (t.simple || t.nh <= 1 || blockIdx.x >= t.nseg) return;
  const uint32_t lane = threadIdx.x, nh = t.nh;
  const uint32_t s = blockIdx.x * BS_SEG, e = bmin(t.count, s + BS_SEG);
  const uint32_t w = s == 0 ? 0u : (s > BS_WARM ? s - BS_WARM : 0u);
  uint32_t cost[4] = {0, 0, 0, 0};
  const bool act0 = lane < nh, act1 = lane + 32 < nh, act2 = lane + 64 < nh, act3 = lane + 96 < nh;
  for (uint32_t i = w; i < e; ++i) {
    const uint32_t* ic = c.icost + (size_t)(c.syms[i] & c.mask) * nh;
    uint32_t mn = 0xFFFFFFFFu, arg = 0;
    if (act0) { cost[0] += ic[lane]; mn = cost[0]; arg = lane; }
    if (act1) { cost[1] += ic[lane + 32]; if (cost[1] < mn) { mn = cost[1]; arg = lane + 32; } }
    if (act2) { cost[2] += ic[lane + 64]; if (cost[2] < mn) { mn = cost[2]; arg = lane + 64; } }
    if (act3) { cost[3] += ic[lane + 96]; if (cost[3] < mn) { mn = cost[3]; arg = lane + 96; } }
    // warp argmin: smallest cost, smallest code index on ties (the sequential scan keeps the first strict minimum)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint32_t om = __shfl_xor_sync(FULLMASK, mn, o), oa = __shfl_xor_sync(FULLMASK, arg, o);
      if (om < mn || (om == mn && oa < arg)) { mn = om; arg = oa; }
    }
    const uint32_t sc = bs_switch_cost_at(c.p.switch_cost_q16, i);
    uint32_t sig[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const bool act = lane + 32 * q < nh;
      bool hit = false;
      if (act) {
        cost[q] -= mn;
        if (cost[q] >= sc) { cost[q] = sc; hit = true; }
      }
      sig[q] = __ballot_sync(FULLMASK, hit);
    }
    if (i >= s && lane == 0) {
      c.blockid[i] = (uint8_t)arg;
      *reinterpret_cast<uint4*>(c.signal + (size_t)i * 4) = make_uint4(sig[0], sig[1], sig[2], sig[3]);
    }
  }
}
// Backward pass of FindBlocks (block_splitter.rs:323-347), exact but segment parallel.  The id at symbol i is a function of the id
// at i + 1 (keep it, or jump to the cheapest code of i when the switch bit of the kept id is set), so a segment is a map
// "id at the first symbol behind the segment -> id at its first symbol":
//   k_bs_bfunc   one warp per segment walks all 128 hypotheses at once (4 per lane); they usually coalesce after a few hundred
//                symbols, from where on a single walk is enough;
//   k_bs_bchain  one thread per (metablock, category) chains the maps from the last segment to the first;
//   k_bs_bwrite  one lane per segment repeats its walk with the now known incoming id and writes the ids.
__global__ void __launch_bounds__(32) k_bs_bfunc(Workspace W, BsWs B) {
  const uint32_t m = blockIdx.y;
  const int cat = (int)blockIdx.z;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  if (t.simple || t.nh <= 1 || blockIdx.x >= t.nseg) return;
  const uint32_t lane = threadIdx.x;
  const uint32_t s = blockIdx.x * BS_SEG, e = bmin(t.count, s + BS_SEG);
  uint32_t cur[4] = {lane, lane + 32, lane + 64, lane + 96};
  uint32_t hi = e;
  bool uniform = false;
  if (e == t.count) {  // the last symbol keeps its own cheapest code whatever comes in
    const uint32_t last = c.blockid[t.count - 1];
    cur[0] = cur[1] = cur[2] = cur[3] = last;
    hi = t.count - 1;
    uniform = true;
  }
  for (uint32_t i = hi; i > s;) {
    --i;
    const uint4 sg = *reinterpret_cast<const uint4*>(c.signal + (size_t)i * 4);
    const uint32_t bid = c.blockid[i];
    if (uniform) {
      const uint32_t x = cur[0];
      const uint32_t word = (x >> 5) == 0 ? sg.x : ((x >> 5) == 1 ? sg.y : ((x >> 5) == 2 ? sg.z : sg.w));
      if (((word >> (x & 31)) & 1u) && x != bid) cur[0] = bid;
      continue;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t x = cur[q];
      const uint32_t word = (x >> 5) == 0 ? sg.x : ((x >> 5) == 1 ? sg.y : ((x >> 5) == 2 ? sg.z : sg.w));
      if (((word >> (x & 31)) & 1u) && x != bid) cur[q] = bid;
    }
    if ((i & 15u) == 0) {  // all hypotheses below nh agree: one walk from here on
      const uint32_t c0 = __shfl_sync(FULLMASK, cur[0], 0);
      const bool same = (lane >= t.nh || cur[0] == c0) && (lane + 32 >= t.nh || cur[1] == c0) && (lane + 64 >= t.nh || cur[2] == c0) &&
                        (lane + 96 >= t.nh || cur[3] == c0);
      if (__all_sync(FULLMASK, same)) { uniform = true; cur[0] = c0; }
    }
  }
  uint8_t* f = B.fmap + ((size_t)m * B.segc_sum + bs_off(B.segc, cat) + blockIdx.x) * 128;
  if (uniform) { const uint8_t v = (uint8_t)cur[0]; f[lane] = v; f[lane + 32] = v; f[lane + 64] = v; f[lane + 96] = v; }
  else { f[lane] = (uint8_t)cur[0]; f[lane + 32] = (uint8_t)cur[1]; f[lane + 64] = (uint8_t)cur[2]; f[lane + 96] = (uint8_t)cur[3]; }
}
// grid (num_mb, 3), 32 threads
__global__ void __launch_bounds__(32) k_bs_bchain(Workspace W, BsWs B) {
  const uint32_t m = blockIdx.x;
  const int cat = (int)blockIdx.y;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  if (t.simple) return;
  if (t.nh <= 1) {  // a single code: every symbol belongs to it
    for (uint32_t i = threadIdx.x; i < t.count; i += 32) c.blockid[i] = 0;
    return;
  }
  if (threadIdx.x != 0) return;
  const uint8_t* fmap = B.fmap + ((size_t)m * B.segc_sum + bs_off(B.segc, cat)) * 128;
  uint8_t* enter = B.enter + (size_t)m * B.segc_sum + bs_off(B.segc, cat);
  uint32_t id = 0;  // the last segment ignores its incoming id
  for (uint32_t sgm = t.nseg; sgm-- > 0;) {
    enter[sgm] = (uint8_t)id;
    id = fmap[(size_t)sgm * 128 + id];
  }
}
// grid (segments, num_mb, 3), 32 threads (lane 0 works)
__global__ void __launch_bounds__(32) k_bs_bwrite(Workspace W, BsWs B) {
  const uint32_t m = blockIdx.y;
  const int cat = (int)blockIdx.z;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  if (t.simple || t.nh <= 1 || blockIdx.x >= t.nseg || threadIdx.x != 0) return;
  const uint32_t s = blockIdx.x * BS_SEG, e = bmin(t.count, s + BS_SEG);
  uint32_t cur = B.enter[(size_t)m * B.segc_sum + bs_off(B.segc, cat) + blockIdx.x];
  uint32_t hi = e;
  if (e == t.count) { cur = c.blockid[t.count - 1]; hi = t.count - 1; }
  for (uint32_t i = hi; i > s;) {
    --i;
    const uint32_t word = c.signal[(size_t)i * 4 + (cur >> 5)];
    const uint32_t bid = c.blockid[i];
    if (((word >> (cur & 31)) & 1u) && cur != bid) cur = bid;
    c.blockid[i] = (uint8_t)cur;
  }
}

// RemapBlockIds: first position of every id -> dense ids in order of first use; histograms cleared.  grid (num_mb, 3), 256 threads
__global__ void __launch_bounds__(256) k_bs_remap(Workspace W, BsWs B) {
  __shared__ uint32_t s_first[128];
  __shared__ uint32_t s_new[128];
  __shared__ uint32_t s_n;
  const uint32_t m = blockIdx.x;
  const int cat = (int)blockIdx.y;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  if (t.simple) return;
  if (threadIdx.x < 128) s_first[threadIdx.x] = 0xFFFFFFFFu;
  __syncthreads();
  if (t.nh > 1) {
    for (uint32_t i = threadIdx.x; i < t.count; i += blockDim.x) {
      const uint32_t id = c.blockid[i];
      if (i == 0 || c.blockid[i - 1] != id) atomicMin(&s_first[id], i);
    }
  } else if (threadIdx.x == 0) s_first[0] = 0;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t next = 0;
    for (;;) {  // ids by ascending first position
      uint32_t best = 0xFFFFFFFFu, bi = 0;
      for (uint32_t k = 0; k < 128; ++k) if (s_first[k] < best) { best = s_first[k]; bi = k; }
      if (best == 0xFFFFFFFFu) break;
      s_new[bi] = next++;
      s_first[bi] = 0xFFFFFFFFu;
    }
    s_n = next;
  }
  __syncthreads();
  if (threadIdx.x < 128) c.firstpos[threadIdx.x] = s_new[threadIdx.x];
  for (uint32_t i = threadIdx.x; i < s_n * c.p.A; i += blockDim.x) c.hist[i] = 0;
  if (threadIdx.x == 0) c.meta->nh = s_n;
}
// BuildBlockHistograms: relabel + count.  grid (x, num_mb, 3)
__global__ void __launch_bounds__(256) k_bs_rehist(Workspace W, BsWs B) {
  const uint32_t m = blockIdx.y;
  const int cat = (int)blockIdx.z;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  if (t.simple) return;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < t.count; i += gridDim.x * blockDim.x) {
    const uint32_t id = c.firstpos[c.blockid[i]];
    c.blockid[i] = (uint8_t)id;
    atomicAdd(&c.hist[(size_t)id * c.p.A + (c.syms[i] & c.mask)], 1u);
  }
}
// Blocks = runs of equal ids (at most maxb: later switches are ignored).  grid (num_mb, 3), 1024 threads
__global__ void __launch_bounds__(1024) k_bs_blocks(Workspace W, BsWs B) {
  __shared__ uint32_t s_warp[33];
  const uint32_t m = blockIdx.x;
  const int cat = (int)blockIdx.y;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  if (t.simple) {
    if (threadIdx.x == 0) { c.bstart[0] = 0; c.bstart[1] = t.count; c.meta->nb = 1; }
    return;
  }
  uint32_t run = 0;
  for (uint32_t base = 0; base < t.count; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t flag = (i < t.count && (i == 0 || c.blockid[i] != c.blockid[i - 1])) ? 1u : 0u;
    uint32_t tot;
    const uint32_t ex = block_excl_scan_1024(flag, s_warp, &tot);
    if (flag) {
      const uint32_t b = run + ex;
      if (b + 1u < c.maxb) c.bstart[b] = i;  // (bstart has maxb words per category and needs one for the end marker)
    }
    run += tot;
  }
  if (threadIdx.x == 0) {
    // more blocks than the workspace holds (never seen: the switch cost keeps blocks hundreds of symbols long): the tail is one block
    const uint32_t nb = bmin(run, c.maxb - 1u);
    c.bstart[nb] = t.count;
    c.meta->nb = nb;
  }
}
// per-block histograms: grid (x, num_mb, 3)
__global__ void __launch_bounds__(256) k_bs_bhist(Workspace W, BsWs B) {
  const uint32_t m = blockIdx.y;
  const int cat = (int)blockIdx.z;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  if (t.simple) return;
  uint32_t* bh = B.bh_in + (size_t)m * B.bh_sum + bs_bh_off(B, cat);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < t.count; i += gridDim.x * blockDim.x) {
    const uint32_t b = find_block(c.bstart, t.nb, i);
    atomicAdd(&bh[(size_t)b * c.p.A + (c.syms[i] & c.mask)], 1u);
  }
}

// ---- clustering drivers: kind 0 = ClusterBlocks of (m, cat), kind 1 = context maps (defined further down) ----
struct CmWs;
__device__ ClProblem cm_cluster_problem(const Workspace& W, const CmWs& M, uint32_t m, int which);

// grid (x, num_mb, 3): one warp per block histogram
__global__ void __launch_bounds__(CL_WARPS * 32) k_bs_cl_prepare(Workspace W, BsWs B) {
  __shared__ uint32_t s_dh[CL_WARPS][18];
  const uint32_t m = blockIdx.y;
  const int cat = (int)blockIdx.z;
  if (B.meta[(size_t)m * 3 + cat].simple) return;
  const ClProblem C = bs_cluster_problem(W, B, m, cat);
  const uint32_t wid = threadIdx.x >> 5;
  for (uint32_t i = blockIdx.x * CL_WARPS + wid; i < C.n; i += gridDim.x * CL_WARPS) cl_prepare_one(C, i, W.lut, s_dh[wid]);
}
// grid (x, num_mb, 3): one CTA per batch of 64 block histograms
__global__ void __launch_bounds__(CLB_WARPS * 32) k_bs_cl_batch(Workspace W, BsWs B) {
  __shared__ ClbShared S;
  const uint32_t m = blockIdx.y;
  const int cat = (int)blockIdx.z;
  if (B.meta[(size_t)m * 3 + cat].simple) return;
  const ClProblem C = bs_cluster_problem(W, B, m, cat);
  const uint32_t nbatch = (C.n + 63) / 64;
  for (uint32_t b = blockIdx.x; b < nbatch; b += gridDim.x) cl_batch_one(C, b, W.lut, S);
}
// grid (num_mb, 3), one CTA
__global__ void __launch_bounds__(CLB_WARPS * 32) k_bs_cl_final(Workspace W, BsWs B) {
  __shared__ ClbShared S;
  const uint32_t m = blockIdx.x;
  const int cat = (int)blockIdx.y;
  if (B.meta[(size_t)m * 3 + cat].simple) return;
  const ClProblem C = bs_cluster_problem(W, B, m, cat);
  cl_final_one(C, W.lut, S);
}
__global__ void __launch_bounds__(CL_WARPS * 32) k_bs_cl_assign(Workspace W, BsWs B) {
  __shared__ uint32_t s_dh[CL_WARPS][18];
  const uint32_t m = blockIdx.y;
  const int cat = (int)blockIdx.z;
  if (B.meta[(size_t)m * 3 + cat].simple) return;
  const ClProblem C = bs_cluster_problem(W, B, m, cat);
  const uint32_t wid = threadIdx.x >> 5;
  for (uint32_t i = blockIdx.x * CL_WARPS + wid; i < C.n; i += gridDim.x * CL_WARPS) cl_assign_one(C, i, W.lut, s_dh[wid]);
}
// Block types by first use, equal neighbours merged -> the split arrays the header / emission stages read.
// grid (num_mb, 3), one thread.
__global__ void __launch_bounds__(32) k_bs_types(Workspace W, BsWs B) {
  if (threadIdx.x != 0) return;
  const uint32_t m = blockIdx.x;
  const int cat = (int)blockIdx.y;
  const BsCat c = bs_cat(W, B, m, cat);
  const BsMeta t = *c.meta;
  const CatInfo ci = cat_info(W, m, cat);
  if (t.simple) {
    ci.types[0] = 0;
    ci.lengths[0] = t.count ? t.count : 1u;
    ci.starts[0] = 0;
    ci.counts[0] = 1;
    ci.counts[1] = 1;
    return;
  }
  const ClProblem C = bs_cluster_problem(W, B, m, cat);
  uint32_t* new_index = C.bj;  // free now: reused as the id map (indexed by cluster id < nb)
  for (uint32_t i = 0; i < t.nb; ++i) new_index[i] = 0xFFFFFFFFu;
  uint32_t next_index = 0;
  for (uint32_t i = 0; i < t.nb; ++i)
    if (new_index[C.sym[i]] == 0xFFFFFFFFu) new_index[C.sym[i]] = next_index++;
  uint32_t cur_length = 0, max_type = 0, nblk = 0, acc = 0;
  for (uint32_t i = 0; i < t.nb; ++i) {
    cur_length += c.bstart[i + 1] - c.bstart[i];
    if (i + 1 == t.nb || C.sym[i] != C.sym[i + 1]) {
      const uint32_t id = new_index[C.sym[i]];
      ci.types[nblk] = (uint8_t)id;
      ci.lengths[nblk] = cur_length;
      ci.starts[nblk] = acc;
      acc += cur_length;
      max_type = bmax(max_type, id);
      cur_length = 0;
      ++nblk;
    }
  }
  ci.counts[0] = nblk;
  ci.counts[1] = max_type + 1;
}

}  // namespace bro

namespace bro {

// ===================================================================================================
// Distance alphabet parameters (BrotliBuildMetaBlock + ComputeDistanceCost, metablock.rs:88-207): the cost of all 64 (NPOSTFIX,
// NDIRECT) combinations in parallel -- one CTA per combination and metablock re-codes every distance, histograms the symbols in
// shared memory and sums the extra bits -- then the reference's greedy walk over the table, then the commands are re-coded.
// ===================================================================================================
__global__ void __launch_bounds__(256) k_dist_cost(Workspace W, uint64_t* cost /* [num_mb][64] */) {
  __shared__ uint32_t s_h[BRO_DIST_A_MAX];
  __shared__ uint32_t s_dh[18];
  __shared__ unsigned long long s_extra;
  const uint32_t m = blockIdx.y, np = blockIdx.x >> 4, nd = (blockIdx.x & 15u) << np;
  const MBDesc& mb = W.mb[m];
  for (uint32_t i = threadIdx.x; i < BRO_DIST_A_MAX; i += blockDim.x) s_h[i] = 0;
  if (threadIdx.x == 0) s_extra = 0;
  __syncthreads();
  uint32_t extra_bits = 0;
  const GCmd* cmds = W.cmds + (size_t)m * W.cmd_cap;
  for (uint32_t i = threadIdx.x; i < mb.ncmd; i += blockDim.x) {
    const GCmd g = cmds[i];
    if (g.copy_len == 0 || g.cmd_prefix < 128) continue;
    uint32_t sn, ex;
    prefix_encode_copy_distance_params(restore_distance_code00(g.dist_prefix, g.dist_extra), np, nd, &sn, &ex);
    atomicAdd(&s_h[sn & 0x3ffu], 1u);
    extra_bits += sn >> 10;
  }
  extra_bits = warp_sum_u32(extra_bits);
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_extra, (unsigned long long)extra_bits);
  __syncthreads();
  if (threadIdx.x < 32) {
    const uint64_t pc = warp_pop_cost(s_h, nullptr, BRO_DIST_A_MAX, W.lut, s_dh);
    if (threadIdx.x == 0) cost[(size_t)m * 64 + blockIdx.x] = pc + ((uint64_t)s_extra << 16);
  }
}
// grid (x, num_mb): every CTA repeats the (tiny) decision, CTA 0 records it, all re-code their share of the commands
__global__ void __launch_bounds__(256) k_dist_apply(Workspace W, const uint64_t* cost) {
  const uint32_t m = blockIdx.y;
  MBDesc& mb = W.mb[m];
  const uint32_t ch = choose_distance_params(cost + (size_t)m * 64);
  const uint32_t np = ch & 0xFFu, nd = ch >> 8;
  if (blockIdx.x == 0 && threadIdx.x == 0) mb.dist_params = ch;
  if (ch == 0) return;
  GCmd* cmds = W.cmds + (size_t)m * W.cmd_cap;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < mb.ncmd; i += gridDim.x * blockDim.x) {
    GCmd& g = cmds[i];
    if (g.copy_len == 0 || g.cmd_prefix < 128) continue;
    uint32_t sn, ex;
    prefix_encode_copy_distance_params(restore_distance_code00(g.dist_prefix, g.dist_extra), np, nd, &sn, &ex);
    g.dist_prefix = (uint16_t)sn;
    g.dist_extra = ex;
  }
}

// ===================================================================================================
// Context maps (BrotliBuildMetaBlock, metablock.rs:133-301): histograms per (block type, context), clustered to at most 256
// prefix codes per category; the clusters' histograms are the coding histograms, the assignment is the context map.
// ===================================================================================================
#define CM_LIT_MAX (256u * 64u)
#define CM_DIST_MAX (256u * 4u)
struct CmWs {
  uint32_t *in_lit, *work_lit;     // [num_mb][CM_LIT_MAX * 256]
  uint32_t *in_dist, *work_dist;   // [num_mb][CM_DIST_MAX * 64]
  uint64_t* cost;                  // [num_mb][CM_LIT_MAX + CM_DIST_MAX]  (literal part first)
  uint32_t *size, *sym, *clusters, *bj;
  int64_t* bd;
  uint32_t* nsurv;                 // [num_mb][2][CM_LIT_MAX / 64 + 2]
  uint32_t* counts;                // [num_mb][2] number of literal / distance prefix codes
  uint8_t* lit_cmap;               // [num_mb][CM_LIT_MAX]
  uint8_t* dist_cmap;              // [num_mb][CM_DIST_MAX]
};
#define CM_NSURV_STRIDE (CM_LIT_MAX / 64u + 2u)
__device__ ClProblem cm_cluster_problem(const Workspace& W, const CmWs& M, uint32_t m, int which) {
  ClProblem C;
  const uint32_t* cnt = W.split_counts + (size_t)m * 6;
  const size_t po = (size_t)m * (CM_LIT_MAX + CM_DIST_MAX) + (which ? CM_LIT_MAX : 0u);
  if (which == 0) { C.A = 256; C.n = cnt[1] * 64u; C.in = M.in_lit + (size_t)m * CM_LIT_MAX * 256; C.work = M.work_lit + (size_t)m * CM_LIT_MAX * 256; }
  else { C.A = W.dist_A; C.n = cnt[5] * 4u; C.in = M.in_dist + (size_t)m * CM_DIST_MAX * W.dist_A; C.work = M.work_dist + (size_t)m * CM_DIST_MAX * W.dist_A; }
  C.cost = M.cost + po; C.size = M.size + po; C.sym = M.sym + po; C.clusters = M.clusters + po; C.bj = M.bj + po; C.bd = M.bd + po;
  C.nsurv = M.nsurv + ((size_t)m * 2 + which) * CM_NSURV_STRIDE + 1;
  C.batch_max = 256;
  C.final_max = 256;
  return C;
}
// grid (x, num_mb): clears the context histograms of the block types in use and the command histograms
__global__ void __launch_bounds__(256) k_cm_zero(Workspace W, CmWs M) {
  const uint32_t m = blockIdx.y;
  const uint32_t* cnt = W.split_counts + (size_t)m * 6;
  const size_t nl = (size_t)cnt[1] * 64 * 256, nd = (size_t)cnt[5] * 4 * W.dist_A, nc = (size_t)cnt[3] * 704;
  uint32_t* il = M.in_lit + (size_t)m * CM_LIT_MAX * 256;
  uint32_t* id = M.in_dist + (size_t)m * CM_DIST_MAX * W.dist_A;
  uint32_t* ch = W.cmd_hist + (size_t)m * (W.max_cmd_types + 1) * 704;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nl + nd + nc; i += (size_t)gridDim.x * blockDim.x) {
    if (i < nl) il[i] = 0;
    else if (i < nl + nd) id[i - nl] = 0;
    else ch[i - nl - nd] = 0;
  }
}
// BrotliBuildHistogramsWithContext (histogram.rs:465-553): grid (x, num_mb, 3)
__global__ void __launch_bounds__(256) k_cm_hist(Workspace W, CmWs M) {
  const uint32_t m = blockIdx.y;
  const int cat = (int)blockIdx.z;
  const MBDesc& mb = W.mb[m];
  const SplitView v = make_view(W, m, cat);
  const uint32_t count = cat == 0 ? mb.nlit : (cat == 1 ? mb.ncmd : mb.ndist);
  const uint16_t* syms = cat == 0 ? W.lit_syms + mb.start : (cat == 1 ? W.cmd_syms + (size_t)m * W.cmd_cap : W.dist_syms + (size_t)m * W.cmd_cap);
  uint32_t* il = M.in_lit + (size_t)m * CM_LIT_MAX * 256;
  uint32_t* id = M.in_dist + (size_t)m * CM_DIST_MAX * W.dist_A;
  uint32_t* ch = W.cmd_hist + (size_t)m * (W.max_cmd_types + 1) * 704;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
    const uint32_t t = v.types[v.num_blocks > 1 ? find_block(v.starts, v.num_blocks, i) : 0u];
    const uint32_t s = syms[i];
    if (cat == 0) atomicAdd(&il[((size_t)t * 64 + (s >> 8)) * 256 + (s & 0xFFu)], 1u);
    else if (cat == 1) atomicAdd(&ch[(size_t)t * 704 + s], 1u);
    else atomicAdd(&id[((size_t)t * 4 + (s >> 10)) * W.dist_A + (s & 0x3FFu)], 1u);
  }
}
__global__ void __launch_bounds__(CL_WARPS * 32) k_cm_cl_prepare(Workspace W, CmWs M) {
  __shared__ uint32_t s_dh[CL_WARPS][18];
  const ClProblem C = cm_cluster_problem(W, M, blockIdx.y, (int)blockIdx.z);
  const uint32_t wid = threadIdx.x >> 5;
  for (uint32_t i = blockIdx.x * CL_WARPS + wid; i < C.n; i += gridDim.x * CL_WARPS) cl_prepare_one(C, i, W.lut, s_dh[wid]);
}
__global__ void __launch_bounds__(CLB_WARPS * 32) k_cm_cl_batch(Workspace W, CmWs M) {
  __shared__ ClbShared S;
  const ClProblem C = cm_cluster_problem(W, M, blockIdx.y, (int)blockIdx.z);
  const uint32_t nbatch = (C.n + 63) / 64;
  for (uint32_t b = blockIdx.x; b < nbatch; b += gridDim.x) cl_batch_one(C, b, W.lut, S);
}
__global__ void __launch_bounds__(CLB_WARPS * 32) k_cm_cl_final(Workspace W, CmWs M) {
  __shared__ ClbShared S;
  const ClProblem C = cm_cluster_problem(W, M, blockIdx.x, (int)blockIdx.y);
  cl_final_one(C, W.lut, S);
}
__global__ void __launch_bounds__(CL_WARPS * 32) k_cm_cl_assign(Workspace W, CmWs M) {
  __shared__ uint32_t s_dh[CL_WARPS][18];
  const ClProblem C = cm_cluster_problem(W, M, blockIdx.y, (int)blockIdx.z);
  const uint32_t wid = threadIdx.x >> 5;
  for (uint32_t i = blockIdx.x * CL_WARPS + wid; i < C.n; i += gridDim.x * CL_WARPS) cl_assign_one(C, i, W.lut, s_dh[wid]);
}
// HistogramReindex (cluster.rs:316-358): dense code ids by first use -> context map; output histograms cleared.
// grid (num_mb, 2), 256 threads
__global__ void __launch_bounds__(256) k_cm_reindex(Workspace W, CmWs M) {
  __shared__ uint32_t s_next;
  const uint32_t m = blockIdx.x;
  const int which = (int)blockIdx.y;
  const ClProblem C = cm_cluster_problem(W, M, m, which);
  uint32_t* new_index = C.bj;  // free now
  for (uint32_t i = threadIdx.x; i < C.n; i += blockDim.x) new_index[i] = 0xFFFFFFFFu;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t next = 0;
    for (uint32_t i = 0; i < C.n; ++i)
      if (new_index[C.sym[i]] == 0xFFFFFFFFu) new_index[C.sym[i]] = next++;
    s_next = next;
    M.counts[(size_t)m * 2 + which] = next;
  }
  __syncthreads();
  uint8_t* cmap = which == 0 ? M.lit_cmap + (size_t)m * CM_LIT_MAX : M.dist_cmap + (size_t)m * CM_DIST_MAX;
  const bool replicate = which == 0 && !W.P.ctx_model;  // literal context modelling off: every context uses the code of context 0
  for (uint32_t i = threadIdx.x; i < C.n; i += blockDim.x) cmap[i] = (uint8_t)new_index[C.sym[replicate ? (i & ~63u) : i]];
  uint32_t* out = which == 0 ? W.lit_hist + (size_t)m * (W.max_lit_trees + 13) * 256 : W.dist_hist + (size_t)m * (W.max_dist_types + 1) * W.dist_A;
  for (uint32_t i = threadIdx.x; i < s_next * C.A; i += blockDim.x) out[i] = 0;
}
// output histogram of a code = sum of the inputs mapped to it.  grid (x, num_mb, 2)
__global__ void __launch_bounds__(256) k_cm_rebuild(Workspace W, CmWs M) {
  const uint32_t m = blockIdx.y;
  const int which = (int)blockIdx.z;
  const ClProblem C = cm_cluster_problem(W, M, m, which);
  const uint8_t* cmap = which == 0 ? M.lit_cmap + (size_t)m * CM_LIT_MAX : M.dist_cmap + (size_t)m * CM_DIST_MAX;
  uint32_t* out = which == 0 ? W.lit_hist + (size_t)m * (W.max_lit_trees + 13) * 256 : W.dist_hist + (size_t)m * (W.max_dist_types + 1) * W.dist_A;
  const size_t total = (size_t)C.n * C.A;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t v = C.in[i];
    if (v) atomicAdd(&out[(size_t)cmap[i / C.A] * C.A + (i % C.A)], v);
  }
}

}  // namespace bro

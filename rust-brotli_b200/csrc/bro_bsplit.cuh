// bro_bsplit.cuh -- quality 10 / 11 histogram stage: population cost, block splitting by entropy codes, histogram
// clustering (block types, literal / distance context maps).
//
// Reference semantics: BrotliPopulationCost (bit_cost.rs:76-211), BrotliSplitBlock -> SplitByteVector ->
// InitialEntropyCodes / RefineEntropyCodes / FindBlocks / RemapBlockIds / BuildBlockHistograms / ClusterBlocks
// (block_splitter.rs:133-929), BrotliHistogramCombine / BrotliCompareAndPushToQueue / BrotliHistogramBitCostDistance /
// BrotliHistogramRemap / BrotliHistogramReindex / BrotliClusterHistograms (cluster.rs:52-420), BrotliBuildMetaBlock
// (metablock.rs:133-301).
//
// GPU re-design (what the kernels in bro_kernels_hq.cuh parallelise, and what the sequential forms below specify):
//  * all costs are Q16 integers, so reductions are order independent and the CPU model equals the GPU bit for bit;
//  * RefineEntropyCodes: sample k of the LCG sequence is seed * 16807^(k+1) mod 2^32, so the samples are independent;
//  * FindBlocks: the symbol vector is cut into segments of BS_SEG symbols; a segment's cost vector is warmed up over the
//    BS_WARM symbols in front of it (costs are clamped to [0, switch cost], so the start state is forgotten quickly) instead
//    of being carried through the whole vector; the backward pass is exact over the recorded switch bits;
//  * the pair queue of the clustering (2048 entries, partial) is replaced by one "best partner" per cluster (exact greedy
//    on the full pair set, O(n) memory), recomputed only for the rows a merge invalidates;
//  * ties in the remap step go to the first cluster of the list instead of the previous block's cluster (sequential tie rule).
#pragma once
#include "bro_common.cuh"
#include "bro_split.cuh"

namespace bro {

#define BS_SEG 8192u
#define BS_WARM 1024u
#define BS_MAX_HIST 100u

struct BsParams {
  uint32_t A, per_hist, max_hist, stride, switch_cost_q16;
};
BRO_HD BsParams bs_params(int cat, uint32_t dist_A = 64) {  // block_splitter.rs:21-45
  BsParams p;
  if (cat == 0) { p.A = 256; p.per_hist = 544; p.max_hist = 100; p.stride = 70; p.switch_cost_q16 = 1841562u; }       // 28.1
  else if (cat == 1) { p.A = 704; p.per_hist = 530; p.max_hist = 50; p.stride = 40; p.switch_cost_q16 = 884736u; }    // 13.5
  else { p.A = dist_A; p.per_hist = 544; p.max_hist = 50; p.stride = 40; p.switch_cost_q16 = 956826u; }                   // 14.6
  return p;
}

// ---------------------------------------------------------------------------------------------------
// BrotliPopulationCost of h (+ g, if not null) in Q16 bits.
// ---------------------------------------------------------------------------------------------------
BRO_HD_NOINLINE uint64_t bs_pop_cost_q16(const uint32_t* h, const uint32_t* g, uint32_t size, const uint32_t* lut) {
  uint32_t total = 0, count = 0, s4[5] = {0, 0, 0, 0, 0};
  for (uint32_t i = 0; i < size; ++i) {
    const uint32_t v = h[i] + (g ? g[i] : 0u);
    total += v;
    if (v && count < 5) s4[count++] = v;
  }
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
  uint32_t depth_histo[18];
  for (int i = 0; i < 18; ++i) depth_histo[i] = 0;
  uint64_t bits = 0;
  uint32_t max_depth = 1;
  const uint32_t log2total = log2_q16(lut, total);
  for (uint32_t i = 0; i < size;) {
    const uint32_t v = h[i] + (g ? g[i] : 0u);
    if (v) {
      const uint32_t log2p = log2total - log2_q16(lut, v);
      uint32_t depth = (log2p + 32768u) >> 16;
      bits += (uint64_t)v * log2p;
      if (depth > 15) depth = 15;
      if (depth > max_depth) max_depth = depth;
      ++depth_histo[depth];
      ++i;
    } else {
      uint32_t reps = 1;
      for (uint32_t k = i + 1; k < size && (h[k] + (g ? g[k] : 0u)) == 0; ++k) ++reps;
      i += reps;
      if (i == size) break;  // trailing zeros are not coded
      if (reps < 3) depth_histo[0] += reps;
      else {
        reps -= 2;
        while (reps > 0) { ++depth_histo[17]; bits += 3ull << 16; reps >>= 3; }
      }
    }
  }
  bits += (uint64_t)(18 + 2 * max_depth) << 16;
  uint64_t sx; uint32_t t;
  hist_sums(depth_histo, 18, lut, &sx, &t);
  return bits + bits_entropy_q16(sx, t, lut);
}
// 0.5 * ClusterCostDiff(a, b) of cluster.rs:37-50 in Q16 (<= 0)
BRO_HD int64_t bs_half_cluster_cost_diff_q16(uint32_t a, uint32_t b, const uint32_t* lut) {
  const int64_t d = (int64_t)xlog2x_q16(lut, a) + (int64_t)xlog2x_q16(lut, b) - (int64_t)xlog2x_q16(lut, a + b);
  return d / 2;
}
// cost_diff of merging clusters a and b (cluster.rs:52-121): cost(a+b) - cost(a) - cost(b) + 0.5 * ClusterCostDiff
BRO_HD int64_t bs_pair_diff_q16(const uint32_t* ha, const uint32_t* hb, uint32_t A, uint64_t cost_a, uint64_t cost_b, uint32_t size_a,
                                uint32_t size_b, const uint32_t* lut) {
  return (int64_t)bs_pop_cost_q16(ha, hb, A, lut) - (int64_t)cost_a - (int64_t)cost_b + bs_half_cluster_cost_diff_q16(size_a, size_b, lut);
}

// ---------------------------------------------------------------------------------------------------
// LCG of the block splitter: MyRand step k (k >= 1) from seed 7 (block_splitter.rs:125-131).
// ---------------------------------------------------------------------------------------------------
BRO_HD uint32_t bs_rand_at(uint32_t k) {  // 7 * 16807^k mod 2^32 (odd, hence never 0)
  uint32_t r = 7, b = 16807u;
  while (k) {
    if (k & 1u) r *= b;
    b *= b;
    k >>= 1;
  }
  return r;
}
BRO_HD uint32_t bs_num_histograms(uint32_t count, const BsParams& p) { return bmin(count / p.per_hist + 1u, p.max_hist); }
// start of the initial stride of histogram i (InitialEntropyCodes, block_splitter.rs:133-158)
BRO_HD uint32_t bs_initial_pos(uint32_t i, uint32_t nh, uint32_t count, uint32_t stride) {
  const uint32_t block_length = count / nh;
  uint32_t pos = (uint32_t)((uint64_t)count * i / nh);
  if (i != 0) pos += bs_rand_at(i) % block_length;
  if (pos + stride >= count) pos = count - stride - 1;
  return pos;
}
BRO_HD uint32_t bs_refine_iters(uint32_t count, uint32_t nh, uint32_t stride) {  // :182-201
  uint32_t iters = 2u * count / stride + 100u;
  return (iters + nh - 1) / nh * nh;
}
BRO_HD uint32_t bs_refine_pos(uint32_t iter, uint32_t count, uint32_t stride) {  // RandomSample, :160-180 (stride < count)
  return bs_rand_at(iter + 1) % (count - stride + 1);
}
// block switch cost at symbol index i (FindBlocks, :314-316): * (0.77 + 0.07 * i / 2000) for i < 2000
BRO_HD uint32_t bs_switch_cost_at(uint32_t bsc, uint32_t i) {
  if (i >= 2000) return bsc;
  return (uint32_t)(((uint64_t)bsc * (50463u + (4588u * i) / 2000u)) >> 16);
}
// insert cost of a symbol with count c in a histogram whose log2(total) is lt (BitCost(0) = -2; :207-213, :255-266)
BRO_HD uint32_t bs_insert_cost(uint32_t lt, uint32_t c, const uint32_t* lut) { return c == 0 ? lt + (2u << 16) : lt - log2_q16(lut, c); }

#ifndef __CUDACC__
}  // namespace bro
#include <algorithm>
#include <vector>
namespace bro {
// ===================================================================================================
// Sequential forms (CPU model; the specification of the kernels).
// ===================================================================================================

// Greedy agglomerative clustering of the clusters listed in `clusters` (ascending ids into hist / cost / size).
// symbols[0..nsym) are relabelled when their cluster is merged away.  Returns the new cluster count; `clusters` keeps the
// survivors in order.  Row a = best partner b > a: smallest cost_diff, smallest b on ties; the pair merged next is the best
// row: smallest diff, then smallest b - a, then smallest a.  Merging stops when no pair has a negative diff, unless more than
// max_clusters are left -- then the best pair is merged whatever its sign (cluster.rs:123-243).
#define BS_NONE 0xFFFFFFFFu
inline uint32_t bs_combine(std::vector<uint32_t>& hist, uint32_t A, std::vector<uint64_t>& cost, std::vector<uint32_t>& size,
                           uint32_t* clusters, uint32_t n, uint32_t* symbols, uint32_t nsym, uint32_t max_clusters, const uint32_t* lut) {
  if (n <= 1) return n;
  const uint32_t top = clusters[n - 1] + 1;
  std::vector<int64_t> bd(top, 0);
  std::vector<uint32_t> bj(top, BS_NONE);
  auto diff = [&](uint32_t a, uint32_t b) {
    return bs_pair_diff_q16(&hist[(size_t)a * A], &hist[(size_t)b * A], A, cost[a], cost[b], size[a], size[b], lut);
  };
  auto recompute_row = [&](uint32_t a) {
    bj[a] = BS_NONE;
    for (uint32_t q = 0; q < n; ++q) {
      const uint32_t b = clusters[q];
      if (b <= a) continue;
      const int64_t d = diff(a, b);
      if (bj[a] == BS_NONE || d < bd[a]) { bd[a] = d; bj[a] = b; }
    }
  };
  for (uint32_t q = 0; q < n; ++q) recompute_row(clusters[q]);
  bool forced = false;
  while (n > 1) {
    uint32_t a = BS_NONE;
    for (uint32_t q = 0; q < n; ++q) {
      const uint32_t r = clusters[q];
      if (bj[r] == BS_NONE) continue;
      if (a == BS_NONE || bd[r] < bd[a] || (bd[r] == bd[a] && bj[r] - r < bj[a] - a)) a = r;
    }
    if (a == BS_NONE) break;
    if (!forced && bd[a] >= 0) forced = true;  // from here on only the cluster limit drives merging
    if (forced && n <= max_clusters) break;
    const uint32_t b = bj[a];
    for (uint32_t s = 0; s < A; ++s) hist[(size_t)a * A + s] += hist[(size_t)b * A + s];
    cost[a] = bs_pop_cost_q16(&hist[(size_t)a * A], nullptr, A, lut);
    size[a] += size[b];
    for (uint32_t i = 0; i < nsym; ++i) if (symbols[i] == b) symbols[i] = a;
    {
      uint32_t w = 0;
      for (uint32_t q = 0; q < n; ++q) if (clusters[q] != b) clusters[w++] = clusters[q];
      n = w;
    }
    for (uint32_t q = 0; q < n; ++q) {
      const uint32_t r = clusters[q];
      if (r < a) {
        if (bj[r] == a || bj[r] == b) recompute_row(r);
        else {
          const int64_t d = diff(r, a);
          if (bj[r] == BS_NONE || d < bd[r] || (d == bd[r] && a < bj[r])) { bd[r] = d; bj[r] = a; }
        }
      } else if (r > a && r < b) {
        if (bj[r] == b) recompute_row(r);
      }
    }
    recompute_row(a);
  }
  return n;
}

// best cluster of `histo` among clusters[0..n): smallest BrotliHistogramBitCostDistance, first in list order on ties
inline uint32_t bs_best_cluster(const uint32_t* histo, uint32_t A, const std::vector<uint32_t>& hist, const std::vector<uint64_t>& cost,
                                const uint32_t* clusters, uint32_t n, const uint32_t* lut) {
  uint32_t total = 0;
  for (uint32_t s = 0; s < A; ++s) total += histo[s];
  if (total == 0) return clusters[0];
  uint32_t best = clusters[0];
  int64_t best_bits = 0;
  for (uint32_t j = 0; j < n; ++j) {
    const uint32_t c = clusters[j];
    const int64_t bits = (int64_t)bs_pop_cost_q16(histo, &hist[(size_t)c * A], A, lut) - (int64_t)cost[c];
    if (j == 0 || bits < best_bits) { best_bits = bits; best = c; }
  }
  return best;
}

// BrotliClusterHistograms: in[n][A] -> out histograms (dense, reindexed by first use) and symbols[n].  Returns the number of
// output histograms.
inline uint32_t bs_cluster_histograms(const uint32_t* in, uint32_t n, uint32_t A, uint32_t max_clusters, const uint32_t* lut,
                                      std::vector<uint32_t>& out, std::vector<uint32_t>& symbols) {
  std::vector<uint32_t> hist(in, in + (size_t)n * A), size(n, 1), clusters(n);
  std::vector<uint64_t> cost(n);
  symbols.resize(n);
  for (uint32_t i = 0; i < n; ++i) { cost[i] = bs_pop_cost_q16(&hist[(size_t)i * A], nullptr, A, lut); symbols[i] = i; }
  uint32_t nc = 0;
  for (uint32_t i = 0; i < n; i += 64) {
    const uint32_t k = std::min(64u, n - i);
    for (uint32_t j = 0; j < k; ++j) clusters[nc + j] = i + j;
    nc += bs_combine(hist, A, cost, size, &clusters[nc], k, &symbols[i], k, max_clusters, lut);
  }
  nc = bs_combine(hist, A, cost, size, clusters.data(), nc, symbols.data(), n, max_clusters, lut);
  // HistogramRemap: every input to its nearest cluster, then the clusters are rebuilt from their members
  for (uint32_t i = 0; i < n; ++i) symbols[i] = bs_best_cluster(in + (size_t)i * A, A, hist, cost, clusters.data(), nc, lut);
  // HistogramReindex: dense ids in order of first use
  std::vector<uint32_t> new_index(n, 0xFFFFFFFFu);
  uint32_t next = 0;
  for (uint32_t i = 0; i < n; ++i) if (new_index[symbols[i]] == 0xFFFFFFFFu) new_index[symbols[i]] = next++;
  out.assign((size_t)next * A, 0);
  for (uint32_t i = 0; i < n; ++i) {
    symbols[i] = new_index[symbols[i]];
    for (uint32_t s = 0; s < A; ++s) out[(size_t)symbols[i] * A + s] += in[(size_t)i * A + s];
  }
  return next;
}

// FindBlocks forward pass over segment [s, e) of the symbol vector: block_id[i] = cheapest histogram at i, signal = one bit
// per (symbol, histogram) "would switch here".  insert_cost[sym * nh + k].
inline void bs_find_blocks_forward(const uint16_t* syms, uint32_t mask, uint32_t s, uint32_t e, uint32_t nh, const uint32_t* insert_cost,
                                   uint32_t bsc, uint8_t* block_id, uint32_t* signal /* [count][4] */) {
  uint32_t cost[BS_MAX_HIST];
  for (uint32_t k = 0; k < nh; ++k) cost[k] = 0;
  const uint32_t w = s == 0 ? 0u : (s > BS_WARM ? s - BS_WARM : 0u);
  for (uint32_t i = w; i < e; ++i) {
    const uint32_t* ic = insert_cost + (size_t)(syms[i] & mask) * nh;
    uint32_t mn = 0xFFFFFFFFu, arg = 0;
    for (uint32_t k = 0; k < nh; ++k) {
      cost[k] += ic[k];
      if (cost[k] < mn) { mn = cost[k]; arg = k; }
    }
    const uint32_t sc = bs_switch_cost_at(bsc, i);
    uint32_t sig[4] = {0, 0, 0, 0};
    for (uint32_t k = 0; k < nh; ++k) {
      cost[k] -= mn;
      if (cost[k] >= sc) { cost[k] = sc; sig[k >> 5] |= 1u << (k & 31); }
    }
    if (i >= s) {
      block_id[i] = (uint8_t)arg;
      for (int q = 0; q < 4; ++q) signal[(size_t)i * 4 + q] = sig[q];
    }
  }
}

struct BsSplit {
  uint32_t num_types;
  std::vector<uint8_t> types;
  std::vector<uint32_t> lengths;
};

// SplitByteVector (block_splitter.rs:692-837) + ClusterBlocks (:399-690).  syms[i] & mask is the symbol.
inline void bs_split_vector(const uint16_t* syms, uint32_t mask, uint32_t count, int cat, uint32_t max_blocks, const uint32_t* lut, BsSplit* out,
                            uint32_t dist_A = 64) {
  const BsParams p = bs_params(cat, dist_A);
  const uint32_t A = p.A;
  out->types.clear();
  out->lengths.clear();
  if (count < 128) {  // kMinLengthForBlockSplitting (an empty category gets one block too: the header needs a length)
    out->num_types = 1;
    out->types.push_back(0);
    out->lengths.push_back(count ? count : 1u);
    return;
  }
  uint32_t nh = bs_num_histograms(count, p);
  std::vector<uint32_t> hist((size_t)nh * A, 0);
  for (uint32_t i = 0; i < nh; ++i) {
    const uint32_t pos = bs_initial_pos(i, nh, count, p.stride);
    for (uint32_t j = 0; j < p.stride; ++j) ++hist[(size_t)i * A + (syms[pos + j] & mask)];
  }
  {
    const uint32_t iters = bs_refine_iters(count, nh, p.stride);
    for (uint32_t it = 0; it < iters; ++it) {
      const uint32_t pos = bs_refine_pos(it, count, p.stride);
      for (uint32_t j = 0; j < p.stride; ++j) ++hist[(size_t)(it % nh) * A + (syms[pos + j] & mask)];
    }
  }
  std::vector<uint8_t> block_id(count, 0);
  std::vector<uint32_t> signal((size_t)count * 4), insert_cost;
  for (int iter = 0; iter < 3; ++iter) {
    if (nh > 1) {
      insert_cost.assign((size_t)A * nh, 0);
      for (uint32_t k = 0; k < nh; ++k) {
        uint32_t total = 0;
        for (uint32_t s = 0; s < A; ++s) total += hist[(size_t)k * A + s];
        const uint32_t lt = log2_q16(lut, total);
        for (uint32_t s = 0; s < A; ++s) insert_cost[(size_t)s * nh + k] = bs_insert_cost(lt, hist[(size_t)k * A + s], lut);
      }
      for (uint32_t s = 0; s < count; s += BS_SEG)
        bs_find_blocks_forward(syms, mask, s, std::min(count, s + BS_SEG), nh, insert_cost.data(), p.switch_cost_q16, block_id.data(), signal.data());
      // backward pass (:323-347)
      uint32_t cur = block_id[count - 1];
      for (uint32_t i = count - 1; i > 0;) {
        --i;
        if (((signal[(size_t)i * 4 + (cur >> 5)] >> (cur & 31)) & 1u) && cur != block_id[i]) cur = block_id[i];
        block_id[i] = (uint8_t)cur;
      }
    } else {
      std::fill(block_id.begin(), block_id.end(), 0);
    }
    // RemapBlockIds (:352-376) + BuildBlockHistograms (:378-397)
    uint32_t new_id[256], next = 0;
    for (uint32_t k = 0; k < 256; ++k) new_id[k] = 256;
    for (uint32_t i = 0; i < count; ++i) if (new_id[block_id[i]] == 256) new_id[block_id[i]] = next++;
    nh = next;
    hist.assign((size_t)nh * A, 0);
    for (uint32_t i = 0; i < count; ++i) {
      block_id[i] = (uint8_t)new_id[block_id[i]];
      ++hist[(size_t)block_id[i] * A + (syms[i] & mask)];
    }
  }
  // blocks = runs of equal ids (at most max_blocks: later switches are ignored)
  std::vector<uint32_t> bl;
  for (uint32_t i = 0; i < count; ++i) {
    if (i == 0 || (block_id[i] != block_id[i - 1] && bl.size() < max_blocks)) bl.push_back(0);
    ++bl.back();
  }
  const uint32_t nb = (uint32_t)bl.size();
  // ClusterBlocks: batches of 64 block histograms are clustered in place (cluster id = slot of its first block), then all
  // batch survivors together (<= 256 types)
  std::vector<uint32_t> all_hist((size_t)nb * A, 0), all_size(nb, 1), hsym(nb), clusters(nb);
  std::vector<uint64_t> all_cost(nb);
  {
    uint32_t pos = 0;
    for (uint32_t i = 0; i < nb; ++i) {
      for (uint32_t q = 0; q < bl[i]; ++q) ++all_hist[(size_t)i * A + (syms[pos++] & mask)];
      all_cost[i] = bs_pop_cost_q16(&all_hist[(size_t)i * A], nullptr, A, lut);
      hsym[i] = i;
    }
  }
  uint32_t nc = 0;
  for (uint32_t i = 0; i < nb; i += 64) {
    const uint32_t k = std::min(64u, nb - i);
    for (uint32_t j = 0; j < k; ++j) clusters[nc + j] = i + j;
    nc += bs_combine(all_hist, A, all_cost, all_size, &clusters[nc], k, &hsym[i], k, 64, lut);
  }
  nc = bs_combine(all_hist, A, all_cost, all_size, clusters.data(), nc, hsym.data(), nb, 256, lut);
  // every block to its nearest final cluster; types numbered by first use; equal neighbours merged
  std::vector<uint32_t> new_index(nb, 0xFFFFFFFFu);
  uint32_t next_index = 0, pos = 0;
  std::vector<uint32_t> histo(A);
  for (uint32_t i = 0; i < nb; ++i) {
    std::fill(histo.begin(), histo.end(), 0u);
    for (uint32_t q = 0; q < bl[i]; ++q) ++histo[syms[pos++] & mask];
    hsym[i] = bs_best_cluster(histo.data(), A, all_hist, all_cost, clusters.data(), nc, lut);
    if (new_index[hsym[i]] == 0xFFFFFFFFu) new_index[hsym[i]] = next_index++;
  }
  uint32_t cur_length = 0, max_type = 0;
  for (uint32_t i = 0; i < nb; ++i) {
    cur_length += bl[i];
    if (i + 1 == nb || hsym[i] != hsym[i + 1]) {
      const uint32_t id = new_index[hsym[i]];
      out->types.push_back((uint8_t)id);
      out->lengths.push_back(cur_length);
      max_type = std::max(max_type, id);
      cur_length = 0;
    }
  }
  out->num_types = max_type + 1;
}
#endif

}  // namespace bro

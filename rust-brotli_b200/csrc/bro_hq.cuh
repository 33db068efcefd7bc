// bro_hq.cuh -- quality 10 / 11: all matches per position, literal cost estimate, shortest-path ("Zopfli") parse.
//
// Reference semantics: FindAllMatchesH10 (backward_references/hq.rs:302-417) on top of the H10 binary tree
// (hash_to_binary_tree.rs:437-530), BrotliEstimateBitCostsForLiterals (literal_cost.rs), ZopfliCostModel (hq.rs:167-252,
// :1046-1154), UpdateNodes / EvaluateNode / StartPosQueue (hq.rs:419-821), ZopfliIterate (:1157),
// BrotliCreateHqZopfliBackwardReferences (:1237), BrotliZopfliCreateCommands (:97).
//
// GPU re-design:
//  * The mutating binary tree is replaced by the position-ordered bucket lists the sort stage already builds: a position's
//    matches are the Pareto front (longer => farther) over the short-range scan, the `depth` nearest earlier positions of
//    its bucket that share its first four bytes, and the static-dictionary candidate.  Every position is independent.
//  * The shortest-path parse runs per parse unit (32 / 64 KiB instead of the reference's 256 KiB input block), units are
//    independent: each starts from an unknown distance cache and its copies stop at its end; the finalise stage assigns the
//    real short codes from the true distance sequence and merges copies that continue across a seam (bro_finalize.cuh).
//  * Costs are Q10 fixed point (u32) instead of f32, so the result does not depend on evaluation order or on the machine.
// Everything in this header is a per-position or per-unit sequential routine (one GPU thread, or the CPU model).
#pragma once
#include "bro_common.cuh"
#include "bro_parse.cuh"

namespace bro {

#ifndef HQ_MAXW
#define HQ_MAXW 8u           // window matches kept per position (the longest ones)
#endif
#ifndef HQ_MAXD
#define HQ_MAXD 8u           // dictionary matches kept per position (the longest ones)
#endif
#define HQ_MAXM (HQ_MAXW + HQ_MAXD)
#define HQ_LCAP 384u         // match length cap of the all-matches stage (> MaxZopfliLen = 325); longer copies are extended by the parse
#define HQ_QBITS 10          // cost fixed point
#define HQ_ONE (1u << HQ_QBITS)
#define HQ_INF 0xFFFFFFFFu

struct HqMatch {
  uint32_t dist;  // backward distance; for a dictionary match: word_id (index + (transform << NDBITS[len]))
  uint32_t lc;    // bits 0..15 bytes produced, bits 16..20 word length (dictionary), bit 31 dictionary
};
BRO_HD uint32_t hqm_len(const HqMatch& m) { return m.lc & 0xFFFFu; }
BRO_HD bool hqm_is_dict(const HqMatch& m) { return (m.lc >> 31) != 0; }
BRO_HD uint32_t hqm_len_code(const HqMatch& m) { return hqm_is_dict(m) ? ((m.lc >> 16) & 31u) : (m.lc & 0xFFFFu); }

BRO_HD int hq_max_candidates(int quality) { return quality <= 10 ? 1 : 5; }          // hq.rs:417-419
BRO_HD uint32_t hq_max_zopfli_len(int quality) { return quality <= 10 ? 150u : 325u; }  // hq.rs:159-165
BRO_HD uint32_t hq_short_back(int quality) { return quality != 11 ? 16u : 64u; }      // hq.rs:325-329

// common-prefix length of a[..] and b[..], at most max_len (device: 8 bytes at a time; the input has >= 512 B of padding)
BRO_HD uint32_t hq_lcp(const uint8_t* a, const uint8_t* b, uint32_t max_len) {
#ifdef __CUDA_ARCH__
  uint32_t i = 0;
  while (i + 8 <= max_len) {
    uint64_t x, y;
    memcpy(&x, a + i, 8);
    memcpy(&y, b + i, 8);
    x ^= y;
    if (x) return i + ((uint32_t)(__ffsll((long long)x) - 1) >> 3);
    i += 8;
  }
  while (i < max_len && a[i] == b[i]) ++i;
  return i;
#else
  return lcp_bytes(a, b, max_len);
#endif
}

// ---------------------------------------------------------------------------------------------------
// All matches of one position.
// ---------------------------------------------------------------------------------------------------
struct HqMatchList {
  HqMatch m[HQ_MAXM];
  uint32_t n;
  uint32_t best_len;
};
BRO_HD void hq_list_init(HqMatchList& L) { L.n = 0; L.best_len = 1; }
BRO_HD void hq_push(HqMatchList& L, uint32_t dist, uint32_t lc) {
  if (L.n == HQ_MAXW) {  // full: drop the shortest
    for (uint32_t k = 0; k + 1 < HQ_MAXW; ++k) L.m[k] = L.m[k + 1];
    L.n = HQ_MAXW - 1;
  }
  L.m[L.n].dist = dist;
  L.m[L.n].lc = lc;
  ++L.n;
}
// 2- and 3-byte matches at very short distances, which no 4-byte hash can find (hq.rs:325-356)
BRO_HD void hq_short_matches(const uint8_t* cur, uint32_t max_len, uint32_t max_backward, uint32_t short_back, HqMatchList& L) {
  for (uint32_t back = 1; back < short_back && L.best_len <= 2; ++back) {
    if (back > max_backward) break;
    const uint8_t* prev = cur - back;
    if (cur[0] == prev[0] && cur[1] == prev[1]) {
      const uint32_t len = hq_lcp(prev, cur, max_len);
      if (len > L.best_len) {
        L.best_len = len;
        hq_push(L, back, len);
      }
    }
  }
}
// One bucket candidate at distance `backward` that is known to share the first four bytes.  Returns false when the walk can
// stop (a full-length match: nothing farther can be longer).
BRO_HD bool hq_bucket_candidate(const uint8_t* cur, uint32_t backward, uint32_t max_len, HqMatchList& L) {
  const uint8_t* prev = cur - backward;
  if (L.best_len < max_len && prev[L.best_len] != cur[L.best_len]) return true;  // cannot be strictly longer
  const uint32_t len = hq_lcp(prev, cur, max_len);
  if (len > L.best_len) {
    L.best_len = len;
    hq_push(L, backward, len);
  }
  return len < max_len;
}
// ---------------------------------------------------------------------------------------------------
// Long-prefix candidate levels.  The 1024 nearest entries of a 4-byte bucket are the neighbourhood H10's tree walks for short and
// medium matches, but a long match far away hides behind thousands of nearer 4-byte look-alikes (the tree finds it because it is
// ordered by content).  So the positions are bucketed again by a hash of their first 8, 16 and 32 bytes; in each of these lists
// the entries in front of a position whose whole 64-bit hash agrees (32 bits are compared) are candidates, nearest first, and
// form a Pareto front B (strictly longer with growing distance).  The final list is the Pareto front of everything, the HQ_MAXW
// longest kept.  6 MB of text, q10: +1.2 % -> +0.3 % of libbrotlienc's size; JSON logs +2.0 % -> +0.7 %.
// ---------------------------------------------------------------------------------------------------
#define HQ_MAX_LEVELS 3
#define HQ_LEVEL_DEPTH 1024
BRO_HD uint32_t hq_level_bytes(int level) { return 8u << level; }  // 8, 16, 32
template <typename Load64>
BRO_HD uint64_t hq_level_hash_with(Load64 load64, uint32_t nbytes) {
  uint64_t h = 0x9E3779B97F4A7C15ull * nbytes;
  for (uint32_t k = 0; k < nbytes; k += 8) {
    h = (h ^ load64(k)) * 0xff51afd7ed558ccdull;
    h ^= h >> 32;
  }
  return h;
}
BRO_HD uint64_t hq_load64_bytes(const uint8_t* p) {
  uint64_t v = 0;
  for (int i = 7; i >= 0; --i) v = (v << 8) | p[i];
  return v;
}
BRO_HD uint64_t hq_level_hash(const uint8_t* p, uint32_t nbytes) {
  return hq_level_hash_with([p](uint32_t k) { return hq_load64_bytes(p + k); }, nbytes);
}
BRO_HD uint32_t hq_level_key(uint64_t h, int key_bits) { return (uint32_t)(h >> (64 - key_bits)); }
BRO_HD void hq_merge_lists(HqMatchList& L, const HqMatchList& B) {
  HqMatch m[2 * HQ_MAXW];
  uint32_t n = 0, ia = 0, ib = 0, best = 1;
  while (ia < L.n || ib < B.n) {
    const bool take_a = ib >= B.n || (ia < L.n && L.m[ia].dist <= B.m[ib].dist);
    const HqMatch c = take_a ? L.m[ia++] : B.m[ib++];
    if ((c.lc & 0xFFFFu) > best) { best = c.lc & 0xFFFFu; m[n++] = c; }
  }
  const uint32_t drop = n > HQ_MAXW ? n - HQ_MAXW : 0u;  // the shortest go
  for (uint32_t k = drop; k < n; ++k) L.m[k - drop] = m[k];
  L.n = n - drop;
  L.best_len = best;
}

// static-dictionary matches (hq.rs:372-404): every produced length above the longest window match, the HQ_MAXD longest kept
BRO_HD void hq_dict_matches(const DictView& D, const uint8_t* cur, uint32_t max_len, HqMatchList& L) {
  uint32_t dm[DICT_MAX_MATCH_LEN + 1];
  const uint32_t minlen = bmax(4u, L.best_len + 1u);
  if (!dict_all_matches(D, cur, minlen, max_len, dm)) return;
  const uint32_t maxlen = bmin(DICT_MAX_MATCH_LEN, max_len);
  uint32_t cnt = 0;
  for (uint32_t l = minlen; l <= maxlen; ++l) cnt += dm[l] < DICT_NO_MATCH;
  for (uint32_t l = minlen; l <= maxlen; ++l) {
    if (dm[l] >= DICT_NO_MATCH) continue;
    if (cnt-- > HQ_MAXD) continue;  // more than HQ_MAXD lengths: the shortest are dropped
    L.m[L.n].dist = dm[l] >> 5;
    L.m[L.n].lc = l | ((dm[l] & 31u) << 16) | 0x80000000u;
    ++L.n;
  }
}

// ---------------------------------------------------------------------------------------------------
// Literal cost estimate of one unit (BrotliEstimateBitCostsForLiterals, literal_cost.rs: a sliding-window histogram around every
// position): Q10 bits per position as exclusive prefix sums pre[0..len], pre[0] = 0.  hist: scratch of 3 * 256 u32.
// ---------------------------------------------------------------------------------------------------
BRO_HD uint32_t hq_utf8_position(uint32_t last, uint32_t c, uint32_t clamp) {  // literal_cost.rs:8-19
  if (c < 128) return 0;
  if (c >= 192) return bmin(1u, clamp);
  if (last < 0xe0) return 0;
  return bmin(2u, clamp);
}
BRO_HD bool hq_is_mostly_utf8(const uint8_t* d, uint32_t len) {  // utf8_util.rs:4-73, min_fraction 0.75
  uint32_t size_utf8 = 0, i = 0;
  while (i < len) {
    const uint32_t left = len - i;
    const uint8_t c0 = d[i];
    uint32_t n = 1;
    bool ok = false;
    if ((c0 & 0x80) == 0) { ok = c0 > 0; }
    if (!ok && left > 1 && (c0 & 0xe0) == 0xc0 && (d[i + 1] & 0xc0) == 0x80) {
      const uint32_t s = ((uint32_t)(c0 & 0x1f) << 6) | (d[i + 1] & 0x3f);
      if (s > 0x7f) { ok = true; n = 2; }
    }
    if (!ok && left > 2 && (c0 & 0xf0) == 0xe0 && (d[i + 1] & 0xc0) == 0x80 && (d[i + 2] & 0xc0) == 0x80) {
      const uint32_t s = ((uint32_t)(c0 & 0x0f) << 12) | ((uint32_t)(d[i + 1] & 0x3f) << 6) | (d[i + 2] & 0x3f);
      if (s > 0x7ff) { ok = true; n = 3; }
    }
    if (!ok && left > 3 && (c0 & 0xf8) == 0xf0 && (d[i + 1] & 0xc0) == 0x80 && (d[i + 2] & 0xc0) == 0x80 && (d[i + 3] & 0xc0) == 0x80) {
      const uint32_t s = ((uint32_t)(c0 & 0x07) << 18) | ((uint32_t)(d[i + 1] & 0x3f) << 12) | ((uint32_t)(d[i + 2] & 0x3f) << 6) | (d[i + 3] & 0x3f);
      if (s > 0xffff && s <= 0x10ffff) { ok = true; n = 4; }
    }
    if (ok) size_utf8 += n;
    i += n;
  }
  return (uint64_t)size_utf8 * 4 > (uint64_t)len * 3;
}
BRO_HD uint32_t hq_lit_cost_q(const uint32_t* lut, uint32_t in_window, uint32_t histo, uint32_t i, bool ramp) {
  if (histo == 0) histo = 1;
  uint32_t c = ((log2_q16(lut, in_window) - log2_q16(lut, histo)) >> (16 - HQ_QBITS)) + 30u;  // + 0.02905
  if (c < HQ_ONE) c = (c >> 1) + (HQ_ONE >> 1);
  if (ramp && i < 2000) c += 717u - ((2000u - i) * 358u) / 2000u;  // + 0.7 - (2000 - i) / 2000 * 0.35
  return c;
}
// d = the unit's first byte; the unit is [0, len) inside the metablock span [-before, len + after): the sliding windows reach
// into the neighbouring units (not across the metablock: its ends are where the reference's block ends are), and the start-up
// surcharge of literal_cost.rs:173-175 applies to the first 2000 bytes of the metablock only.
BRO_HD_NOINLINE void hq_literal_costs_unit(const uint8_t* d, uint32_t len, uint32_t before, uint32_t after, const uint32_t* lut, uint32_t* hist,
                                           uint32_t* pre) {
  pre[0] = 0;
  if (len == 0) return;
  const int64_t lo = -(int64_t)before, hi = (int64_t)len + after;  // metablock span relative to d
  if (hq_is_mostly_utf8(d, len)) {
    // DecideMultiByteStatsLevel, literal_cost.rs:21-48 (on the unit)
    uint32_t counts[3] = {0, 0, 0}, max_utf8 = 1, last_c = 0;
    for (uint32_t i = 0; i < len; ++i) {
      const uint32_t c = d[i];
      ++counts[hq_utf8_position(last_c, c, 2)];
      last_c = c;
    }
    if (counts[2] < 500) max_utf8 = 1;
    if (counts[1] + counts[2] < 25) max_utf8 = 0;
    const int64_t W = 495;
    uint32_t in_window_utf8[3] = {0, 0, 0};
    for (uint32_t i = 0; i < 3 * 256; ++i) hist[i] = 0;
    auto cls = [&](int64_t p) -> uint32_t {  // class of the byte at p from its two predecessors (0 outside the metablock)
      const uint32_t c = p - 1 >= lo ? d[p - 1] : 0u, lc = p - 2 >= lo ? d[p - 2] : 0u;
      return hq_utf8_position(lc, c, max_utf8);
    };
    // window of position 0: [max(lo, -W), min(hi, W))
    for (int64_t p = (-W > lo ? -W : lo); p < (W < hi ? W : hi); ++p) { const uint32_t k = cls(p); ++hist[k * 256 + d[p]]; ++in_window_utf8[k]; }
    for (uint32_t i = 0; i < len; ++i) {
      const int64_t out = (int64_t)i - W - 1, in = (int64_t)i + W - 1;  // window of i: [i - W, i + W)
      if (i > 0) {
        if (out >= lo) { const uint32_t k = cls(out); --hist[k * 256 + d[out]]; --in_window_utf8[k]; }
        if (in < hi) { const uint32_t k = cls(in); ++hist[k * 256 + d[in]]; ++in_window_utf8[k]; }
      }
      const uint32_t up = cls((int64_t)i);
      pre[i + 1] = pre[i] + hq_lit_cost_q(lut, in_window_utf8[up], hist[up * 256 + d[i]], before + i, true);
    }
  } else {
    const int64_t W = 2000;
    uint32_t in_window = 0;
    for (uint32_t i = 0; i < 256; ++i) hist[i] = 0;
    for (int64_t p = (-W > lo ? -W : lo); p < (W < hi ? W : hi); ++p) { ++hist[d[p]]; ++in_window; }
    for (uint32_t i = 0; i < len; ++i) {
      const int64_t out = (int64_t)i - W - 1, in = (int64_t)i + W - 1;
      if (i > 0) {
        if (out >= lo) { --hist[d[out]]; --in_window; }
        if (in < hi) { ++hist[d[in]]; ++in_window; }
      }
      pre[i + 1] = pre[i] + hq_lit_cost_q(lut, in_window, hist[d[i]], before + i, true);
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// Cost model (hq.rs:167-252 first pass; :1046-1154 second pass of quality 11).
// ---------------------------------------------------------------------------------------------------
struct HqCostModel {
  uint32_t cost_cmd[704];
  uint32_t cost_dist[64];
  uint32_t min_cost_cmd;
};
BRO_HD uint32_t hq_log2_q(const uint32_t* lut, uint32_t v) { return (log2_q16(lut, v) + (1u << (15 - HQ_QBITS))) >> (16 - HQ_QBITS); }
BRO_HD_NOINLINE void hq_model_initial(HqCostModel* M, const uint32_t* lut) {
  for (uint32_t i = 0; i < 704; ++i) M->cost_cmd[i] = hq_log2_q(lut, 11 + i);
  for (uint32_t i = 0; i < 64; ++i) M->cost_dist[i] = hq_log2_q(lut, 20 + i);
  M->min_cost_cmd = hq_log2_q(lut, 11);
}
// SetCost, hq.rs:1046-1074
BRO_HD void hq_set_cost(const uint32_t* histogram, uint32_t size, bool literal_histogram, const uint32_t* lut, uint32_t* cost) {
  uint32_t sum = 0;
  for (uint32_t i = 0; i < size; ++i) sum += histogram[i];
  const uint32_t log2sum = hq_log2_q(lut, sum);
  uint32_t missing = sum;
  if (!literal_histogram)
    for (uint32_t i = 0; i < size; ++i) if (histogram[i] == 0) ++missing;
  const uint32_t missing_cost = hq_log2_q(lut, missing) + 2 * HQ_ONE;
  for (uint32_t i = 0; i < size; ++i) {
    if (histogram[i] == 0) { cost[i] = missing_cost; continue; }
    const uint32_t l = hq_log2_q(lut, histogram[i]);
    uint32_t c = log2sum > l ? log2sum - l : 0;
    if (c < HQ_ONE) c = HQ_ONE;
    cost[i] = c;
  }
}

// second pass: costs from the histograms of the first pass; literal prefix sums are rebuilt from the per-symbol costs
BRO_HD_NOINLINE void hq_model_from_stats(HqCostModel* M, const uint32_t* stats, const uint32_t* lut, const uint8_t* d, uint32_t len,
                                         uint32_t* cost_literal /* scratch [256] */, uint32_t* pre) {
  hq_set_cost(stats, 256, true, lut, cost_literal);
  hq_set_cost(stats + 256, 704, false, lut, M->cost_cmd);
  hq_set_cost(stats + 256 + 704, 64, false, lut, M->cost_dist);
  uint32_t mn = M->cost_cmd[0];
  for (uint32_t i = 1; i < 704; ++i) mn = bmin(mn, M->cost_cmd[i]);
  M->min_cost_cmd = mn;
  pre[0] = 0;
  for (uint32_t i = 0; i < len; ++i) pre[i + 1] = pre[i] + cost_literal[d[i]];
}

// ---------------------------------------------------------------------------------------------------
// Shortest path over one unit.
// ---------------------------------------------------------------------------------------------------
struct ZNode {  // hash_to_binary_tree.rs:24-33
  uint32_t length;               // copy length | (copy length + 9 - length code) << 25
  uint32_t distance;
  uint32_t dcode_insert_length;  // insert length | (distance short code + 1) << 27
  uint32_t u;                    // cost (Q10) while ahead of the sweep, then the distance-cache shortcut, then `next`
};
BRO_HD uint32_t zn_copy_length(const ZNode& n) { return n.length & 0x1FFFFFFu; }
BRO_HD uint32_t zn_length_code(const ZNode& n) { return zn_copy_length(n) + 9u - (n.length >> 25); }
BRO_HD uint32_t zn_insert_length(const ZNode& n) { return n.dcode_insert_length & 0x7FFFFFFu; }
BRO_HD uint32_t zn_distance_code(const ZNode& n) {
  const uint32_t sc = n.dcode_insert_length >> 27;
  return sc == 0 ? n.distance + 15u : sc - 1u;
}

struct HqPosData {
  uint32_t pos;
  int32_t dc[4];
  int64_t costdiff;
  uint32_t cost;
};
struct HqQueue {  // StartPosQueue, hq.rs:185-188, :493-509
  HqPosData q[8];
  uint32_t idx;
};
BRO_HD uint32_t hq_queue_size(const HqQueue& Q) { return bmin(Q.idx, 8u); }
BRO_HD const HqPosData& hq_queue_at(const HqQueue& Q, uint32_t k) { return Q.q[(k - Q.idx) & 7u]; }
BRO_HD void hq_queue_push(HqQueue& Q, const HqPosData& pd) {
  uint32_t offset = ~Q.idx & 7u;
  ++Q.idx;
  const uint32_t len = hq_queue_size(Q);
  Q.q[offset] = pd;
  for (uint32_t i = 1; i < len; ++i) {
    if (Q.q[offset & 7u].costdiff > Q.q[(offset + 1) & 7u].costdiff) {
      const HqPosData t = Q.q[offset & 7u];
      Q.q[offset & 7u] = Q.q[(offset + 1) & 7u];
      Q.q[(offset + 1) & 7u] = t;
    }
    ++offset;
  }
}

struct HqUnit {  // everything UpdateNodes needs about the unit being parsed
  const uint8_t* data;     // range-relative base pointer
  uint32_t ustart, len;    // unit = data[ustart, ustart + len)
  uint64_t abs_base;       // absolute stream position of data[0]
  uint32_t max_backward;   // window limit
  int quality;
  const HqCostModel* model;
  const uint32_t* lit_pre; // [len + 1]
  const int32_t* start_dc; // [4]
  ZNode* nodes;            // [len + 1]
};
BRO_HD uint32_t hq_max_distance(const HqUnit& U, uint32_t pos) {
  const uint64_t a = U.abs_base + U.ustart + pos;
  return a < U.max_backward ? (uint32_t)a : U.max_backward;
}
BRO_HD uint32_t hq_shortcut(const HqUnit& U, uint32_t pos) {  // ComputeDistanceShortcut, hq.rs:421-447
  const ZNode& n = U.nodes[pos];
  const uint32_t clen = zn_copy_length(n), ilen = zn_insert_length(n), dist = n.distance;
  if (pos == 0) return 0;
  if ((uint64_t)dist + clen <= U.abs_base + U.ustart + pos && dist <= U.max_backward && zn_distance_code(n) > 0) return pos;
  return U.nodes[pos - clen - ilen].u;
}
BRO_HD void hq_distance_cache(const HqUnit& U, uint32_t pos, int32_t* dc) {  // ComputeDistanceCache, hq.rs:456-490
  int idx = 0;
  uint32_t p = U.nodes[pos].u;
  while (idx < 4 && p > 0) {
    const ZNode& n = U.nodes[p];
    dc[idx++] = (int32_t)n.distance;
    p = U.nodes[p - zn_copy_length(n) - zn_insert_length(n)].u;
  }
  for (int k = 0; idx < 4; ++idx, ++k) dc[idx] = U.start_dc[k];
}
BRO_HD void hq_evaluate_node(const HqUnit& U, uint32_t pos, HqQueue& Q) {  // EvaluateNode, hq.rs:511-548
  const uint32_t node_cost = U.nodes[pos].u;
  U.nodes[pos].u = hq_shortcut(U, pos);
  if (node_cost <= U.lit_pre[pos]) {
    HqPosData pd;
    pd.pos = pos;
    pd.cost = node_cost;
    pd.costdiff = (int64_t)node_cost - (int64_t)U.lit_pre[pos];
    hq_distance_cache(U, pos, pd.dc);
    hq_queue_push(Q, pd);
  }
}
BRO_HD void hq_update_node(ZNode* nodes, uint32_t pos, uint32_t start_pos, uint32_t len, uint32_t len_code, uint32_t dist,
                           uint32_t short_code, uint32_t cost) {  // UpdateZopfliNode, hq.rs:619-636
  ZNode& next = nodes[pos + len];
  next.length = len | ((len + 9u - len_code) << 25);
  next.distance = dist;
  next.dcode_insert_length = (pos - start_pos) | (short_code << 27);
  next.u = cost;
}
// UpdateNodes, hq.rs:644-821.  matches[0..num_matches) sorted by length ascending.  Returns the longest copy that improved a
// node.
BRO_HD_NOINLINE uint32_t hq_update_nodes(const HqUnit& U, uint32_t pos, const HqMatch* matches, uint32_t num_matches, HqQueue& Q) {
  const uint8_t* cur = U.data + U.ustart + pos;
  const uint32_t max_distance = hq_max_distance(U, pos);
  const uint32_t max_len = U.len - pos;
  const uint32_t max_zopfli_len = hq_max_zopfli_len(U.quality);
  const HqCostModel& M = *U.model;
  ZNode* nodes = U.nodes;
  uint32_t result = 0;
  hq_evaluate_node(U, pos, Q);
  uint32_t min_len;
  {
    const HqPosData& pd = hq_queue_at(Q, 0);
    uint64_t min_cost = (uint64_t)pd.cost + M.min_cost_cmd + (U.lit_pre[pos] - U.lit_pre[pd.pos]);
    // ComputeMinimumCopyLength, hq.rs:564-589
    uint32_t len = 2, next_len_bucket = 4, next_len_offset = 10;
    while (pos + len <= U.len && nodes[pos + len].u <= min_cost) {
      ++len;
      if (len == next_len_offset) {
        min_cost += HQ_ONE;
        next_len_offset += next_len_bucket;
        next_len_bucket *= 2;
      }
    }
    min_len = len;
  }
  const uint32_t ncand = bmin((uint32_t)hq_max_candidates(U.quality), hq_queue_size(Q));
#ifdef __CUDA_ARCH__
  // Half of the sweep's instructions were the 16 distance-cache probes per start position, almost always ending at the first-byte
  // test.  The (start k, cached distance j) pairs -- up to 5 x 16 at quality 11 -- are spread over the lanes, three independent
  // rounds whose loads overlap; only the pairs that can improve on min_len - 1 go through the sequential part below, in the same
  // order with the same test: identical nodes.  Every device caller must therefore run the unit with a full warp in lock step
  // (same data in every lane): the probes are shared through warp ballots and shuffles.
  uint32_t coop_len0 = 0, coop_len1 = 0, coop_len2 = 0, coop_ball0 = 0, coop_ball1 = 0, coop_ball2 = 0;
  {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t bl0 = min_len - 1;
#pragma unroll
    for (uint32_t r = 0; r < 3; ++r) {
      const uint32_t pidx = lane + 32u * r;
      uint32_t l = 0;
      if (pidx < 16u * ncand && bl0 < max_len) {
        const HqPosData& pq = hq_queue_at(Q, pidx >> 4);
        const int32_t bs = cache_candidate(pq.dc, (int)(pidx & 15u));
        if (bs > 0 && (uint32_t)bs <= max_distance) {
          const uint8_t* prev = cur - bs;
          if (cur[bl0] == prev[bl0]) l = hq_lcp(prev, cur, max_len);
        }
      }
      const uint32_t ball = __ballot_sync(0xffffffffu, l > bl0);
      if (r == 0) { coop_len0 = l; coop_ball0 = ball; } else if (r == 1) { coop_len1 = l; coop_ball1 = ball; } else { coop_len2 = l; coop_ball2 = ball; }
    }
  }
#endif
  for (uint32_t k = 0; k < ncand; ++k) {
    const HqPosData& pd = hq_queue_at(Q, k);
    const uint32_t start = pd.pos;
    const uint32_t inscode = insert_length_code(pos - start);
    const int64_t base_cost = pd.costdiff + ((int64_t)ins_extra(inscode) << HQ_QBITS) + (int64_t)U.lit_pre[pos];
    uint32_t best_len = min_len - 1;
#ifdef __CUDA_ARCH__
    const uint32_t coop_sh = (k & 1u) * 16u;
    const uint32_t coop_round_ball = (k >> 1) == 0 ? coop_ball0 : ((k >> 1) == 1 ? coop_ball1 : coop_ball2);
    const uint32_t coop_len = (k >> 1) == 0 ? coop_len0 : ((k >> 1) == 1 ? coop_len1 : coop_len2);
    uint32_t coop_hits = (coop_round_ball >> coop_sh) & 0xFFFFu;
#endif
    for (int j = 0; j < 16 && best_len < max_len; ++j) {
#ifdef __CUDA_ARCH__
      if (!coop_hits) break;
      j = __ffs((int)coop_hits) - 1;
      coop_hits &= coop_hits - 1u;
#endif
      const int32_t backward_s = cache_candidate(pd.dc, j);  // kDistanceCacheIndex / Offset, mod.rs:653-655
      if (backward_s <= 0 || (uint32_t)backward_s > max_distance) continue;
      const uint32_t backward = (uint32_t)backward_s;
      const uint8_t* prev = cur - backward;
      if (cur[best_len] != prev[best_len]) continue;
#ifdef __CUDA_ARCH__
      const uint32_t len = __shfl_sync(0xffffffffu, coop_len, (int)coop_sh + j);
#else
      const uint32_t len = hq_lcp(prev, cur, max_len);
#endif
      const int64_t dist_cost = base_cost + M.cost_dist[j];
      for (uint32_t l = best_len + 1; l <= len; ++l) {
        const uint32_t copycode = copy_length_code(l);
        const uint32_t cmdcode = combine_length_codes(inscode, copycode, j == 0);
        const int64_t cost = (cmdcode < 128 ? base_cost : dist_cost) + ((int64_t)copy_extra(copycode) << HQ_QBITS) + M.cost_cmd[cmdcode];
        if (cost < (int64_t)nodes[pos + l].u) {
          hq_update_node(nodes, pos, start, l, l, backward, (uint32_t)j + 1, (uint32_t)cost);
          result = bmax(result, l);
        }
        best_len = l;
      }
    }
    if (k >= 2) continue;
    uint32_t len = min_len;
    for (uint32_t j = 0; j < num_matches; ++j) {
      const HqMatch& m = matches[j];
      const bool is_dict = hqm_is_dict(m);
      const uint32_t dist = is_dict ? max_distance + 1u + m.dist : m.dist;
      if (!is_dict && dist > max_distance) continue;  // (cannot happen: the match stage applies the same window limit)
      uint32_t max_match_len = bmin(hqm_len(m), max_len);
      if (is_dict && hqm_len(m) > max_len) continue;
      uint32_t sym_nbits, extra;
      prefix_encode_copy_distance(dist + 15u, &sym_nbits, &extra);
      const int64_t dist_cost = base_cost + ((int64_t)(sym_nbits >> 10) << HQ_QBITS) + M.cost_dist[sym_nbits & 0x3ffu];
      if (len < max_match_len && (is_dict || max_match_len > max_zopfli_len)) len = max_match_len;
      for (; len <= max_match_len; ++len) {
        const uint32_t len_code = is_dict ? hqm_len_code(m) : len;
        const uint32_t copycode = copy_length_code(len_code);
        const uint32_t cmdcode = combine_length_codes(inscode, copycode, false);
        const int64_t cost = dist_cost + ((int64_t)copy_extra(copycode) << HQ_QBITS) + M.cost_cmd[cmdcode];
        if (cost < (int64_t)nodes[pos + len].u) {
          hq_update_node(nodes, pos, start, len, len_code, dist, 0, (uint32_t)cost);
          result = bmax(result, len);
        }
      }
    }
  }
  return result;
}

// Parses data[ustart, ustart + len) and writes its commands (copy_len packed as in bro_dict.cuh) to out[]; returns their
// number, *tail = literals after the last copy, *ncopy = bytes covered by copies.  matches / nmatch are indexed by
// range-relative position.
// stats (optional, [256 + 704 + 64], zeroed by the caller): literal / command / distance-symbol histograms of the commands, as the
// second pass of quality 11 wants them (set_from_commands, hq.rs:1076-1154).
BRO_HD_NOINLINE uint32_t hq_zopfli_unit(const HqUnit& U, const HqMatch* matches, const uint8_t* nmatch, RawCmd* out, uint32_t* tail,
                                       uint32_t* ncopy, uint32_t* stats) {
  ZNode* nodes = U.nodes;
  const uint32_t len = U.len;
  const uint32_t max_zopfli_len = hq_max_zopfli_len(U.quality);
  for (uint32_t i = 0; i <= len; ++i) { nodes[i].length = 1; nodes[i].distance = 0; nodes[i].dcode_insert_length = 0; nodes[i].u = HQ_INF; }
  nodes[0].length = 0;
  nodes[0].u = 0;
  HqQueue Q;
  Q.idx = 0;
  for (uint32_t i = 0; i + 3 < len; ++i) {  // ZopfliIterate, hq.rs:1157-1235
    const uint32_t p = U.ustart + i;
    const HqMatch* mp = matches + (size_t)p * HQ_MAXM;
    uint32_t nm = nmatch[p];
    HqMatch longm;
    if (nm > 0) {
      // a match that reached the cap of the match stage is extended to its true length here (the match stage leaves that
      // to the one position that really takes the copy)
      longm = mp[nm - 1];
      if (!hqm_is_dict(longm) && hqm_len(longm) >= HQ_LCAP && len - i > HQ_LCAP) {
        const uint8_t* cur = U.data + p;
        const uint32_t full = HQ_LCAP + hq_lcp(cur - longm.dist + HQ_LCAP, cur + HQ_LCAP, len - i - HQ_LCAP);
        longm.lc = bmin(full, 0xFFFFu);
      }
      if (bmin(hqm_len(longm), len - i) > max_zopfli_len) { mp = &longm; nm = 1; }  // hq.rs:917-921
    }
    uint32_t skip = hq_update_nodes(U, i, mp, nm, Q);
    if (skip < 16384) skip = 0;
    if (nm == 1 && bmin(hqm_len(mp[0]), len - i) > max_zopfli_len) skip = bmax(bmin(hqm_len(mp[0]), len - i), skip);
    if (skip > 1) {
      --skip;
      while (skip) {
        ++i;
        if (i + 3 >= len) break;
        hq_evaluate_node(U, i, Q);
        --skip;
      }
    }
  }
  // ComputeShortestPathFromNodes, hq.rs:837-854
  uint32_t index = len, ncmd = 0;
  while (zn_insert_length(nodes[index]) == 0 && nodes[index].length == 1 && index > 0) --index;
  nodes[index].u = 0xFFFFFFFFu;
  while (index != 0) {
    const uint32_t l = zn_copy_length(nodes[index]) + zn_insert_length(nodes[index]);
    index -= l;
    nodes[index].u = l;
    ++ncmd;
  }
  // BrotliZopfliCreateCommands, hq.rs:97-157 (codes are assigned later by the finalise stage)
  uint32_t pos = 0, offset = nodes[0].u, k = 0, copied = 0;
  while (offset != 0xFFFFFFFFu) {
    const ZNode& next = nodes[pos + offset];
    const uint32_t clen = zn_copy_length(next), ilen = zn_insert_length(next);
    pos += ilen;
    offset = next.u;
    const uint32_t max_distance = hq_max_distance(U, pos);
    const bool is_dict = next.distance > max_distance;
    out[k].insert_len = ilen;
    out[k].copy_len = is_dict ? pack_dict_len(clen, zn_length_code(next)) : clen;
    out[k].distance = next.distance;
    ++k;
    if (stats) {
      uint32_t sym_nbits, extra;
      const uint32_t dcode = zn_distance_code(next);
      prefix_encode_copy_distance(dcode, &sym_nbits, &extra);
      const uint32_t cmdcode = combine_length_codes(insert_length_code(ilen), copy_length_code(zn_length_code(next)), dcode == 0);
      ++stats[256 + cmdcode];
      if (cmdcode >= 128) ++stats[256 + 704 + (sym_nbits & 0x3ffu)];
      for (uint32_t j = 0; j < ilen; ++j) ++stats[U.data[U.ustart + pos - ilen + j]];
    }
    pos += clen;
    copied += clen;
  }
  *tail = len - pos;
  *ncopy = copied;
  return k;
}

// Parse unit of the shortest-path parse.  A unit is one serial node sweep, so its size is the latency of the whole stage (a 16 KiB
// unit at quality 11 takes longer than a CPU needs for a small file), while many units are needed to fill the machine.
// Large inputs: 8 KiB at quality 10, 16 KiB at quality 11 (the size / speed trade: DESIGN.md); inputs known to be small get
// smaller units: they cannot fill the GPU anyway, the pooled statistics (below) keep the cost model the same, and the size moves
// by +0.05 ... +0.1 %.  size_hint = 0 means unknown.
BRO_HD uint32_t hq_default_unit(int quality, uint32_t size_hint) {
  if (size_hint != 0 && size_hint <= (256u << 10)) return 2048u;
  if (size_hint != 0 && size_hint <= (1u << 20)) return 4096u;
  return quality >= 11 ? 16384u : 8192u;
}

// Default parameters of a (quality, lgwin, size hint, Q9_5) configuration, shared by the device encoder and its CPU model.  P->n
// and P->abs_base are left 0: they describe the range being compressed.  size_hint = 0 means unknown.
//
// Q9_5 ("quality 9.5", BROTLI_PARAM_Q9_5) keeps quality 10 / 11 from choosing H10, so the parse is the hash-chain greedy / lazy
// one (the reference picks the parse from the hasher, backward_references/mod.rs:2553-2780) while everything after the parse --
// context mode, block split, clustering, distance parameters -- follows the quality.  At every quality it also lowers the size
// hint above which H6 is chosen from 4 MiB to 1 MiB.
inline void default_enc_params(EncParams* P, int quality, int lgwin, uint32_t size_hint, int q9_5 = 0) {
  *P = EncParams{};
  quality = effective_quality(quality);
  lgwin = lgwin < 10 ? 10 : (lgwin > 24 ? 24 : lgwin);
  P->quality = quality;
  P->lgwin = lgwin;
  P->size_hint = size_hint;
  P->zopfli = quality >= 10 && !q9_5;
  P->hq_meta = quality >= 10;
  const int block_bits = quality - 1 < 9 ? quality - 1 : 9;
  const uint32_t h6_hint = q9_5 ? (1u << 20) : (1u << 22);
  // ChooseHasher, encode.rs:834-893 (H40-42 are not implemented there and fall back to H6 with default params)
  if (P->zopfli) { P->hash_type = 5; P->key_bits = 15; P->hash_len = 4; P->depth = 256; P->n_last = 16; }  // bucket lists for k_match_all (with the long-prefix levels on, 64..1024 give the same size +-0.02 %)
  else if (quality == 9 || quality == 10) { P->hash_type = 9; P->key_bits = 15; P->hash_len = 4; P->depth = 256; P->n_last = 16; }
  else if (lgwin <= 16) { P->hash_type = 6; P->key_bits = 15; P->hash_len = 5; P->depth = 256; P->n_last = 16; }
  else if (size_hint > h6_hint && lgwin >= 19) {
    P->hash_type = 6; P->key_bits = 15; P->hash_len = 5; P->depth = 1 << block_bits;
    P->n_last = quality < 7 ? 4 : quality < 9 ? 10 : 16;
  } else {
    P->hash_type = 5; P->key_bits = (quality < 7 && size_hint <= (1u << 20)) ? 14 : 15; P->hash_len = 4;
    P->depth = 1 << block_bits;
    P->n_last = quality < 7 ? 4 : quality < 9 ? 10 : 16;
  }
  P->lcap = 64;
  P->unit = 4096;
  P->mb_units = 1024;  // 4 MiB metablocks
  if (P->zopfli) {  // same metablock span, larger parse units
    P->lcap = HQ_LCAP;
    P->unit = hq_default_unit(quality, size_hint);
    P->mb_units = (4u << 20) / P->unit;
  }
  P->max_backward = (1u << lgwin) - 16;
  P->ctx_model = 1;
  P->use_dict = 1;
  P->hq_split = 1;
  P->hq_levels = P->zopfli ? HQ_MAX_LEVELS : 0;
}

// Quality 11 runs the shortest path twice, the second time with costs taken from the commands of the first pass
// (set_from_commands, hq.rs:1076-1154).  The reference has one 256 KiB block to take them from; a 8 KiB parse unit alone is too
// small a sample (+0.7 % on text against +0.37 % for 64 KiB units), so the statistics of the first pass are pooled over the units
// of one aligned HQ_STATS_SPAN window of the metablock before the second pass starts (two kernels: k_zopfli phase 1 / phase 2).
#define HQ_STATS_SPAN 65536u
#define HQ_STATS_WORDS (256u + 704u + 64u)

// Distance cache a parse unit starts with.  Units are parsed independently, so a unit does not know the last distances of its
// predecessor -- on record-structured input (JSON logs) that costs 0.35 %, because "same distance as before" is the cheapest code
// there is.  Like the q5..q9 parse (BRO_WARMUP_BYTES) the unit therefore first parses the HQ_WARMUP_BYTES in front of it, keeps the
// distance cache that parse ends with and throws its commands away (tmp: scratch for W / 2 + 1 commands; V: the warm-up range as a
// unit, V.lit_pre filled for it).  Not done for the first unit of a metablock: metablocks really start with an unknown cache.
#define HQ_WARMUP_BYTES 512u
BRO_HD_NOINLINE void hq_warm_start_cache(const HqUnit& V, const HqMatch* matches, const uint8_t* nmatch, RawCmd* tmp, int32_t* dc) {
  uint32_t t2, c2;
  const uint32_t nc = hq_zopfli_unit(V, matches, nmatch, tmp, &t2, &c2, nullptr);
  dc[0] = dc[1] = dc[2] = dc[3] = 0x3fffffff;
  for (uint32_t k = 0; k < nc; ++k)
    if (!len_is_dict(tmp[k].copy_len) && (int32_t)tmp[k].distance != dc[0]) {
      dc[3] = dc[2]; dc[2] = dc[1]; dc[1] = dc[0]; dc[0] = (int32_t)tmp[k].distance;
    }
}

}  // namespace bro

// bro_split.cuh -- greedy block splitter and literal-context decisions in Q16 integer arithmetic.
//
// Reference semantics: BlockSplitterFinishBlock / ContextBlockSplitterFinishBlock (metablock.rs:551-792),
// BrotliBuildMetaBlockGreedyInternal (:858-1021), DecideOverLiteralContextModeling / ChooseContextMap /
// ShouldUseComplexStaticContextMap (encode.rs:1717-1927), BitsEntropy (bit_cost.rs:13-42).
// Differences by design: entropies are fixed point (log2_q16) so that the GPU's parallel reductions and this
// sequential form agree exactly; the reference's u16 truncation of counts inside BitsEntropy is not reproduced.
#pragma once
#include "bro_common.cuh"

namespace bro {

// sum_c c*log2(c) in Q16 and total count of one histogram
BRO_HD void hist_sums(const uint32_t* h, uint32_t n, const uint32_t* lut, uint64_t* sum_xlogx, uint32_t* total) {
  uint64_t s = 0;
  uint32_t t = 0;
  for (uint32_t i = 0; i < n; ++i) {
    uint32_t c = h[i];
    if (c) { s += xlog2x_q16(lut, c); t += c; }
  }
  *sum_xlogx = s;
  *total = t;
}
// Shannon bits (Q16) of a histogram given its sums; bits_entropy applies the >= total floor.
BRO_HD uint64_t shannon_q16(uint64_t sum_xlogx, uint32_t total, const uint32_t* lut) {
  return total ? xlog2x_q16(lut, total) - sum_xlogx : 0;
}
BRO_HD uint64_t bits_entropy_q16(uint64_t sum_xlogx, uint32_t total, const uint32_t* lut) {
  uint64_t s = shannon_q16(sum_xlogx, total, lut);
  uint64_t floor_bits = (uint64_t)total << 16;
  return s < floor_bits ? floor_bits : s;
}

// Splitter scalar state shared by the sequential form below and by the CUDA kernel's deciding thread.
struct SplitState {
  uint32_t num_blocks, num_types, target_block_size, merge_last_count;
  uint32_t last_type[2];        // block types of the last / second-last histogram
  uint64_t last_entropy[2][13]; // per context
};
enum SplitAction { SPLIT_FIRST = 0, SPLIT_NEW_TYPE = 1, SPLIT_SECOND_LAST = 2, SPLIT_MERGE_LAST = 3 };

// Decision of one FinishBlock step.  e_cur[i], e_comb[j][i]: bits_entropy of the pending histogram and of
// pending+last[j], per context i.  Updates the scalar state; the caller applies the histogram moves.
BRO_HD SplitAction split_decide(SplitState& s, uint32_t nctx, uint32_t max_types, uint64_t thr_q16,
                                uint32_t min_block, const uint64_t* e_cur, const uint64_t* e_comb0,
                                const uint64_t* e_comb1) {
  if (s.num_blocks == 0) {
    for (uint32_t i = 0; i < nctx; ++i) { s.last_entropy[0][i] = e_cur[i]; s.last_entropy[1][i] = e_cur[i]; }
    s.num_blocks = 1;
    s.num_types = 1;
    s.last_type[0] = 0;
    s.last_type[1] = 0;
    return SPLIT_FIRST;
  }
  int64_t diff0 = 0, diff1 = 0;
  for (uint32_t i = 0; i < nctx; ++i) {
    diff0 += (int64_t)e_comb0[i] - (int64_t)e_cur[i] - (int64_t)s.last_entropy[0][i];
    diff1 += (int64_t)e_comb1[i] - (int64_t)e_cur[i] - (int64_t)s.last_entropy[1][i];
  }
  if (s.num_types < max_types && diff0 > (int64_t)thr_q16 && diff1 > (int64_t)thr_q16) {
    s.last_type[1] = s.last_type[0];
    s.last_type[0] = s.num_types;
    for (uint32_t i = 0; i < nctx; ++i) { s.last_entropy[1][i] = s.last_entropy[0][i]; s.last_entropy[0][i] = e_cur[i]; }
    ++s.num_blocks;
    ++s.num_types;
    s.merge_last_count = 0;
    s.target_block_size = min_block;
    return SPLIT_NEW_TYPE;
  }
  if (diff1 < diff0 - (int64_t)(20ull << 16)) {
    uint32_t t = s.last_type[0]; s.last_type[0] = s.last_type[1]; s.last_type[1] = t;
    for (uint32_t i = 0; i < nctx; ++i) { s.last_entropy[1][i] = s.last_entropy[0][i]; s.last_entropy[0][i] = e_comb1[i]; }
    ++s.num_blocks;
    s.merge_last_count = 0;
    s.target_block_size = min_block;
    return SPLIT_SECOND_LAST;
  }
  for (uint32_t i = 0; i < nctx; ++i) {
    s.last_entropy[0][i] = e_comb0[i];
    if (s.num_types == 1) s.last_entropy[1][i] = e_comb0[i];
  }
  if (++s.merge_last_count > 1) s.target_block_size += min_block;
  return SPLIT_MERGE_LAST;
}

// ---- literal context decision (one metablock) ----
// Strided sampling histograms as in encode.rs:1802-1927: 64-byte strides every 4096 bytes.
struct CtxSampleHist {
  uint32_t combined[32];
  uint32_t ctx[13][32];
  uint32_t bigram[9];
  uint32_t total;
};
BRO_HD void ctx_sample_stride(const uint8_t* d, uint32_t sp, CtxSampleHist* h, bool complex_map) {
  if (complex_map) {
    uint8_t prev2 = d[sp], prev1 = d[sp + 1];
    for (uint32_t pos = sp + 2; pos < sp + 64; ++pos) {
      uint8_t lit = d[pos];
      uint32_t cx = ctxmap_lookup(CTXMAP_COMPLEX13, context_utf8(prev1, prev2));
      ++h->total;
      ++h->combined[lit >> 3];
      ++h->ctx[cx][lit >> 3];
      prev2 = prev1;
      prev1 = lit;
    }
  }
  static constexpr uint8_t lut4[4] = {0, 0, 1, 2};
  uint32_t prev = lut4[d[sp] >> 6] * 3u;
  for (uint32_t pos = sp + 1; pos < sp + 64; ++pos) {
    uint8_t lit = d[pos];
    ++h->bigram[prev + lut4[lit >> 6]];
    prev = lut4[lit >> 6] * 3u;
  }
}
BRO_HD int ctx_decide_from_hist(int quality, uint32_t size_hint, const CtxSampleHist* h, const uint32_t* lut) {
  if (size_hint >= (1u << 20) && h->total) {
    uint64_t sx; uint32_t t;
    hist_sums(h->combined, 32, lut, &sx, &t);
    int64_t s1 = (int64_t)shannon_q16(sx, t, lut), s2 = 0;
    for (int i = 0; i < 13; ++i) {
      hist_sums(h->ctx[i], 32, lut, &sx, &t);
      s2 += (int64_t)shannon_q16(sx, t, lut);
    }
    int64_t tot = (int64_t)h->total << 16;
    if (!(s2 > 3 * tot || (s1 - s2) * 5 < tot)) return CTXMAP_COMPLEX13;
  }
  uint32_t mono[3] = {0, 0, 0}, two[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 9; ++i) { mono[i % 3] += h->bigram[i]; two[i % 6] += h->bigram[i]; }
  uint64_t sx; uint32_t t, total;
  hist_sums(mono, 3, lut, &sx, &total);
  if (total == 0) return CTXMAP_NONE;
  int64_t e1 = (int64_t)shannon_q16(sx, total, lut);
  hist_sums(two, 3, lut, &sx, &t);
  int64_t e2 = (int64_t)shannon_q16(sx, t, lut);
  hist_sums(two + 3, 3, lut, &sx, &t);
  e2 += (int64_t)shannon_q16(sx, t, lut);
  int64_t e3 = 0;
  for (int i = 0; i < 3; ++i) {
    hist_sums(h->bigram + 3 * i, 3, lut, &sx, &t);
    e3 += (int64_t)shannon_q16(sx, t, lut);
  }
  if (quality < 7) e3 = e1 * 10;
  int64_t tot = (int64_t)total << 16;
  if ((e1 - e2) * 5 < tot && (e1 - e3) * 5 < tot) return CTXMAP_NONE;
  if ((e2 - e3) * 50 < tot) return CTXMAP_SIMPLE2;
  return CTXMAP_CONT3;
}

#ifndef __CUDACC__
}  // namespace bro
#include <vector>
namespace bro {
// ---- sequential forms used by the CPU model (tools/gpu_model.cpp) ----
inline int decide_literal_context_map(int quality, uint32_t size_hint, const uint8_t* d, uint32_t start, uint32_t len,
                                      const uint32_t* lut) {
  if (quality < 5 || len < 64) return CTXMAP_NONE;
  CtxSampleHist h;
  memset(&h, 0, sizeof(h));
  const bool complex_map = size_hint >= (1u << 20);
  for (uint32_t sp = start; sp + 64 <= start + len; sp += 4096) ctx_sample_stride(d, sp, &h, complex_map);
  return ctx_decide_from_hist(quality, size_hint, &h, lut);
}

struct SplitResult {
  uint32_t num_types;
  std::vector<uint8_t> types;
  std::vector<uint32_t> lengths, starts;
  std::vector<uint32_t> histograms;  // [num_types * nctx][alphabet]
};

// symbols: for nctx == 1 the symbol itself; otherwise literal | ctx << 8
inline void greedy_split(const uint16_t* syms, uint32_t count, uint32_t A, uint32_t nctx, uint32_t min_block,
                         uint32_t thr_bits, const uint32_t* lut, SplitResult* out) {
  const uint32_t HA = nctx * A;
  const uint32_t max_types = nctx == 1 ? 256u : 256u / nctx;
  std::vector<uint32_t> hist((size_t)(max_types + 1) * HA, 0);  // slot t = block type t, slot num_types = pending
  SplitState s;
  memset(&s, 0, sizeof(s));
  s.target_block_size = min_block;
  out->types.clear(); out->lengths.clear();
  uint32_t pending = 0;
  auto finish = [&](bool is_final) {
    uint32_t bs = pending < min_block ? min_block : pending;  // metablock.rs:561
    if (s.num_blocks != 0 && pending == 0 && !is_final) return;
    uint32_t* cur = &hist[(size_t)s.num_types * HA];
    uint64_t e_cur[13], e0[13], e1[13];
    if (s.num_blocks == 0) {
      for (uint32_t i = 0; i < nctx; ++i) {
        uint64_t sx; uint32_t t;
        hist_sums(cur + i * A, A, lut, &sx, &t);
        e_cur[i] = bits_entropy_q16(sx, t, lut);
      }
      split_decide(s, nctx, max_types, (uint64_t)thr_bits << 16, min_block, e_cur, e0, e1);
      out->types.push_back(0);
      out->lengths.push_back(bs);
      pending = 0;
      return;
    }
    std::vector<uint32_t> comb((size_t)2 * HA);
    uint32_t* l0 = &hist[(size_t)s.last_type[0] * HA];
    uint32_t* l1 = &hist[(size_t)s.last_type[1] * HA];
    for (uint32_t i = 0; i < nctx; ++i) {
      uint64_t sx; uint32_t t;
      hist_sums(cur + i * A, A, lut, &sx, &t);
      e_cur[i] = bits_entropy_q16(sx, t, lut);
      for (uint32_t k = 0; k < A; ++k) {
        comb[i * A + k] = cur[i * A + k] + l0[i * A + k];
        comb[HA + i * A + k] = cur[i * A + k] + l1[i * A + k];
      }
      hist_sums(&comb[i * A], A, lut, &sx, &t);
      e0[i] = bits_entropy_q16(sx, t, lut);
      hist_sums(&comb[HA + i * A], A, lut, &sx, &t);
      e1[i] = bits_entropy_q16(sx, t, lut);
    }
    uint32_t old_types = s.num_types;
    SplitAction a = split_decide(s, nctx, max_types, (uint64_t)thr_bits << 16, min_block, e_cur, e0, e1);
    if (a == SPLIT_NEW_TYPE) {
      out->types.push_back((uint8_t)old_types);
      out->lengths.push_back(bs);
      // pending histogram stays in slot old_types and becomes that type's histogram
      memset(&hist[(size_t)s.num_types * HA], 0, (size_t)HA * 4);
    } else if (a == SPLIT_SECOND_LAST) {
      out->types.push_back((uint8_t)s.last_type[0]);
      out->lengths.push_back(bs);
      memcpy(&hist[(size_t)s.last_type[0] * HA], &comb[HA], (size_t)HA * 4);
      memset(cur, 0, (size_t)HA * 4);
    } else {
      out->lengths.back() += bs;
      memcpy(&hist[(size_t)s.last_type[0] * HA], &comb[0], (size_t)HA * 4);
      memset(cur, 0, (size_t)HA * 4);
    }
    pending = 0;
  };
  for (uint32_t i = 0; i < count; ++i) {
    uint32_t sym = nctx == 1 ? syms[i] : (syms[i] & 0xFF) + (syms[i] >> 8) * A;
    ++hist[(size_t)s.num_types * HA + sym];
    if (++pending == s.target_block_size) finish(false);
  }
  finish(true);
  out->num_types = s.num_types;
  out->histograms.assign(hist.begin(), hist.begin() + (size_t)s.num_types * HA);
  out->starts.resize(out->lengths.size());
  uint32_t acc = 0;
  for (size_t b = 0; b < out->lengths.size(); ++b) { out->starts[b] = acc; acc += out->lengths[b]; }
}
#endif

}  // namespace bro

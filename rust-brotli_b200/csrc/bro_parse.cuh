// bro_parse.cuh -- match scoring and the greedy+lazy parse of one parse unit (one GPU thread per unit).
//
// Reference semantics: FindLongestMatch scoring (backward_references/mod.rs:1871-1889, 1151-1154; H9 :657-708)
// and CreateBackwardReferences (mod.rs:2376-2552).  GPU re-design: the hash-bucket walk is NOT done here --
// the match kernel has already produced, for every position, the best bucket candidate (best[p] =
// distance << 8 | min(len, LCAP)) in parallel; the serial part left is the last-distance probes, lazy
// deferral, and command emission, over a unit of a few KiB with a unit-local distance cache.
#pragma once
#include "bro_common.cuh"

// bytes per pipeline pass: one chunk = 6 metablocks of 4 MiB; with its 4 MiB window halo it is one 2^25 sort batch
#define BRO_CHUNK_BYTES (24u << 20)

namespace bro {

// length of the chunk that starts `done` bytes into a range of `total` bytes (shared by the encoder and its CPU model)
BRO_HD uint32_t chunk_len_at(uint64_t done, uint64_t total) {
  // (a short first chunk, to start computing before the whole first 24 MiB are staged, does not pay: e2e gains nothing and
  // the HBM-resident throughput drops because the last chunk then no longer hides behind the others)
  const uint64_t left = total - done;
  return (uint32_t)(left < BRO_CHUNK_BYTES ? left : BRO_CHUNK_BYTES);
}

// The quality the encoder runs for a requested one: 5..9 hash-chain family (encode.rs:834-893), 10 / 11 shortest-path parse;
// q0..q4 (BasicHasher H2..H54, fragment compressors) are not built and run as 5.
BRO_HD int effective_quality(int requested_quality) {
  return requested_quality < 5 ? 5 : (requested_quality > 11 ? 11 : requested_quality);
}

// The defaults of every configuration are set by default_enc_params() (bro_hq.cuh), which the encoder and its CPU model share.
struct EncParams {
  int quality;        // 5..11
  int lgwin;          // 10..24
  int hash_type;      // 5, 6 or 9 (encode.rs:834-893)
  int key_bits;       // bucket_bits
  int hash_len;       // 4 or 5 bytes hashed
  int depth;          // bucket depth = 1 << block_bits
  int n_last;         // num_last_distances_to_check
  uint32_t lcap;      // per-position match length cap of the match kernel (<= 255)
  uint32_t unit;      // parse unit size in bytes
  uint32_t mb_units;  // parse units per metablock
  uint32_t max_backward;  // (1 << lgwin) - 16
  uint32_t n;         // size of the range being compressed (positions are relative to its start)
  uint32_t abs_base;  // absolute stream position of relative position 0 (window limit at the stream start)
  uint32_t size_hint;
  int ctx_model;      // literal context modelling on/off
  int use_dict;       // static-dictionary matches on/off
  int hq_split;       // with hq_meta: 1 = BrotliSplitBlock + clustered context maps (default), 0 = the greedy splitter of q5..q9
  int hq_levels;      // with zopfli: number of long-prefix candidate levels (8, 16, 32 bytes) on top of the 4-byte buckets: 0..3
  // The two families a configuration runs, derived from (quality, Q9_5) by default_enc_params and read everywhere else:
  int zopfli;         // parse: 1 = all matches + shortest path (H10, q10 / q11), 0 = bucket match + greedy / lazy (q5..q9, 9.5)
  int hq_meta;        // metablock builder: 1 = ChooseContextMode, BrotliSplitBlock, clustered context maps and the NPOSTFIX /
                      //   NDIRECT search (quality 10 / 11, with or without Q9_5), 0 = the greedy splitter of q5..q9
};

// ---- scores ----
BRO_HD uint32_t score_regular(int hash_type, uint32_t len, uint32_t backward) {
  if (hash_type == 9) return (7680u + 540u * len - 120u * log2_floor_nz(backward)) >> 2;
  return 1920u + 135u * len - 30u * log2_floor_nz(backward);
}
BRO_HD uint32_t score_last_distance(int hash_type, uint32_t len, uint32_t i) {
  if (hash_type == 9) {
    // kDistanceShortCodeCost (mod.rs:664-683) = 7553 + {187,32,10,0,34,34,31,31 | 28,28,22,22,12,12,2,2}, one byte each
    const uint64_t lo = 0x1F1F2222000A20BBull, hi = 0x02020C0C16161C1Cull;
    const uint32_t delta = (uint32_t)(((i < 8 ? lo : hi) >> ((i & 7u) * 8u)) & 0xFFu);
    return (540u * len + 7553u + delta) >> 2;
  }
  uint32_t s = 135u * len + 1935u;
  if (i != 0) s -= 39u + ((0x1ca10u >> (i & 0xe)) & 0xe);
  return s;
}
#define BRO_MIN_SCORE 2020u

// Cache probes of n_last = 10 / 16 resolved in parallel (one candidate per lane or per probe).  The sequential fold of
// find_match(), with its "must be longer" pre-filter, reduces to: the longest valid candidate wins, lowest index first; only
// among candidates that reach max_len does the score (i.e. the per-index bonus) decide -- 135 points per byte always outweigh
// the bonus spread (<= 47).  That is a max over this key of every valid candidate i of length len (0 = none).
BRO_HD uint32_t last_distance_key(int hash_type, uint32_t len, uint32_t max_len, uint32_t i) {
  const uint32_t bonus = len == max_len ? score_last_distance(hash_type, 0, i) - 1880u : 0u;
  return ((len << 12) | (bonus << 4) | (15u - i)) + 1u;
}
// the winning candidate of a non-zero maximum of last_distance_key: its cache index, and its length in *len
BRO_HD uint32_t last_distance_key_decode(uint32_t key, uint32_t* len) {
  *len = (key - 1u) >> 12;
  return 15u - ((key - 1u) & 15u);
}

// hash key of the bytes at p (buffer must be readable 8 bytes past p)
BRO_HD uint32_t load32(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
BRO_HD uint32_t hash_key_from_words(int hash_type, int key_bits, uint32_t lo, uint32_t hi) {
  if (hash_type == 6) {  // 5 bytes: mod.rs:1138-1140, encode.rs:1066-1067
    uint64_t v = ((uint64_t)(hi & 0xFFu) << 32) | lo;
    return (uint32_t)((v * 0x1fe35a7bd3579bd3ull) >> (64 - key_bits));
  }
  return (uint32_t)(lo * 0x1e35a7bdu) >> (32 - key_bits);  // mod.rs:990-991, :734-738
}
BRO_HD uint32_t hash_key(int hash_type, int key_bits, const uint8_t* p) {
  return hash_key_from_words(hash_type, key_bits, load32(p), (uint32_t)p[4]);
}

BRO_HD uint32_t lcp_bytes(const uint8_t* a, const uint8_t* b, uint32_t max_len) {
  uint32_t i = 0;
  while (i < max_len && a[i] == b[i]) ++i;
  return i;
}
// exact common-prefix length of cur[..] and (cur - back)[..], known to be >= start, capped at max_len
BRO_HD uint32_t lcp_ext(const uint8_t* cur, uint32_t back, uint32_t start, uint32_t max_len) {
  return start + lcp_bytes(cur - back + start, cur + start, max_len - start);
}

struct Match {
  uint32_t len, dist, score;
};

}  // namespace bro
#include "bro_dict.cuh"
namespace bro {

// candidate i of the (expanded) distance cache: mod.rs:632-655
BRO_HD int32_t cache_candidate(const int32_t* dc, int i) {
  // i: 0..3 -> dc[i]; 4..9 -> dc[0] -1,+1,-2,+2,-3,+3; 10..15 -> dc[1] -1,+1,...   (pure arithmetic: no lookup
  // table, so dc[] stays in registers on the device)
  if (i < 4) return i == 0 ? dc[0] : (i == 1 ? dc[1] : (i == 2 ? dc[2] : dc[3]));
  uint32_t k = (uint32_t)i - 4u;
  uint32_t base = (uint32_t)dc[0];
  if (k >= 6u) { k -= 6u; base = (uint32_t)dc[1]; }
  const uint32_t mag = (k >> 1) + 1u;
  return (int32_t)((k & 1u) ? base + mag : base - mag);  // unsigned on purpose: no signed-overflow assumptions
}

// The match stage's candidate b = best[p] at cur = data + p, folded into *m, the result of the cache probes (found: it is a
// match).  A dictionary candidate is taken only when nothing else was found (use_dict; it comes back with Match::len packed by
// pack_dict_len()).  A bucket candidate is clamped to max_len, extended by ext past the match stage's cap lcap (ext = lcp_ext,
// lane_lcp_ext or warp_lcp_ext), and taken when it scores strictly better.  Returns whether *m is a match.
template <typename Ext>
BRO_HD bool take_best_candidate(uint32_t b, int hash_type, uint32_t lcap, const uint8_t* cur, uint32_t max_len, uint32_t max_backward,
                                bool use_dict, Ext ext, bool found, Match* m) {
  if (b & BRO_BEST_DICT) {
    Match dm;
    if (!found && use_dict && dict_decode(b, hash_type, max_len, max_backward, &dm)) { *m = dm; return true; }
    return found;
  }
  const uint32_t blen = b & 0xFFu;
  if (blen != 0) {
    const uint32_t bdist = b >> 8;
    uint32_t len = bmin(blen, max_len);
    if (blen >= lcap && max_len > len) len = ext(cur, bdist, len, max_len);
    if (len >= 4) {
      const uint32_t score = score_regular(hash_type, len, bdist);
      if (m->score < score) { m->len = len; m->dist = bdist; m->score = score; return true; }
    }
  }
  return found;
}

// Best match at pos: last-distance probes (serial state) combined with the precomputed bucket candidate.
BRO_HD_NOINLINE bool find_match(const EncParams& P, const uint8_t* data, const uint32_t* best, const int32_t* dc,
                                uint32_t pos, uint32_t max_len, Match* out, bool use_dict) {
  const uint32_t max_backward = (P.abs_base >= P.max_backward) ? P.max_backward : bmin(pos + P.abs_base, P.max_backward);
  uint32_t best_score = BRO_MIN_SCORE, best_len = 0, best_dist = 0;
  bool found = false;
  const uint8_t* cur = data + pos;
  for (int i = 0; i < P.n_last; ++i) {
    int32_t back = cache_candidate(dc, i);
    if (back <= 0 || (uint32_t)back > max_backward) continue;
    const uint8_t* prev = cur - back;
    if (best_len < max_len && cur[best_len] != prev[best_len]) continue;
    uint32_t len = lcp_bytes(prev, cur, max_len);
    if (len >= 3 || (len == 2 && i < 2)) {
      uint32_t score = score_last_distance(P.hash_type, len, (uint32_t)i);
      if (best_score < score) {
        best_score = score; best_len = len; best_dist = (uint32_t)back;
        found = true;
      }
    }
  }
  out->len = best_len; out->dist = best_dist; out->score = best_score;
  return take_best_candidate(best[pos], P.hash_type, P.lcap, cur, max_len, max_backward, use_dict, lcp_ext, found, out);
}

// Greedy + lazy parse of [rstart, rend) starting from the distance cache dc[4] (updated in place).  find(pos, max_len, Match*)
// is the best match at pos (find_match() or its device forms, reading dc); store(k, insert_len, copy_len, distance) writes
// command k (copy_len >= 2).  Returns the number of commands; *tail = literals after the last copy, *ncopy = total bytes
// covered by copies.  The device walkers that instantiate it keep their state in registers only because it is inlined.
template <typename Find, typename Store>
BRO_HD uint32_t parse_range(const EncParams& P, uint32_t rstart, uint32_t rend, int32_t* dc, Find find, Store store,
                            uint32_t* tail, uint32_t* ncopy) {
  const uint32_t hash_type_len = P.hash_type == 6 ? 8u : 4u;
  const uint32_t window = P.quality < 9 ? 64u : 512u;
  const uint32_t uend = rend;
  uint32_t pos = rstart, insert_len = 0, ncmd = 0, copied = 0;
  uint32_t apply_random_heuristics = pos + window;
  while (pos + hash_type_len < uend) {
    uint32_t max_len = uend - pos;
    Match m;
    if (find(pos, max_len, &m)) {
      int delayed = 0;
      max_len--;
      for (;; max_len--) {
        Match m2;
        bool f2 = find(pos + 1, max_len, &m2);
        if (f2 && m2.score >= m.score + 175u) {
          pos++;
          insert_len++;
          m = m2;
          if (++delayed < 4 && pos + hash_type_len < uend) continue;
        }
        break;
      }
      const uint32_t mlen = len_bytes(m.len);
      apply_random_heuristics = pos + 2 * mlen + window;
      if (!len_is_dict(m.len) && (int32_t)m.dist != dc[0]) {  // dictionary references never enter the distance cache
        dc[3] = dc[2]; dc[2] = dc[1]; dc[1] = dc[0]; dc[0] = (int32_t)m.dist;
      }
      store(ncmd, insert_len, m.len, m.dist);
      ++ncmd;
      insert_len = 0;
      copied += mlen;
      pos += mlen;
    } else {
      insert_len++;
      pos++;
      if (pos > apply_random_heuristics) {
        const uint32_t margin = bmax(hash_type_len - 1u, 4u);
        if (pos + 16 + margin >= uend) {
          insert_len += uend - pos;
          pos = uend;
        } else if (pos > apply_random_heuristics + 4 * window) {
          insert_len += 16;
          pos += 16;
        } else {
          insert_len += 8;
          pos += 8;
        }
      }
    }
  }
  insert_len += uend - pos;
  *tail = insert_len;
  *ncopy = copied;
  return ncmd;
}

// Bytes in front of a unit that are parsed first, only to learn a plausible incoming distance cache (the commands of that
// warm-up are discarded).  Without it every unit starts with an unknown cache and repetitive, record-structured input
// loses ~1.4 % (4 MB of JSON logs, q5); with it +0.06 %.  The cache is only a heuristic input of the match choice: the
// real short codes are assigned by the finalise stage from the true distance sequence.
#define BRO_WARMUP_BYTES 256u

// One parse unit [ustart, uend): warm-up (not for the first unit of a metablock, whose cache really is unknown), parse.
BRO_HD_NOINLINE uint32_t parse_unit(const EncParams& P, const uint8_t* data, const uint32_t* best, uint32_t ustart,
                                    uint32_t uend, RawCmd* out, uint32_t* tail, uint32_t* ncopy) {
  int32_t dc[4] = {0x3fffffff, 0x3fffffff, 0x3fffffff, 0x3fffffff};
  auto find = [&](uint32_t pos, uint32_t max_len, Match* m) { return find_match(P, data, best, dc, pos, max_len, m, P.use_dict != 0); };
  if ((ustart / P.unit) % P.mb_units != 0 && ustart >= BRO_WARMUP_BYTES) {
    uint32_t t2, c2;
    parse_range(P, ustart - BRO_WARMUP_BYTES, ustart, dc, find, [](uint32_t, uint32_t, uint32_t, uint32_t) {}, &t2, &c2);
  }
  return parse_range(P, ustart, uend, dc, find, [&](uint32_t k, uint32_t ins, uint32_t len, uint32_t dist) { out[k] = RawCmd{ins, len, dist}; },
                     tail, ncopy);
}

}  // namespace bro

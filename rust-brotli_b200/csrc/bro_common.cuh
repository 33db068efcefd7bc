// bro_common.cuh -- host/device building blocks of the GPU brotli compression path.
//
// Everything here is a small sequential routine that runs inside ONE GPU thread (or on the host, for the
// CPU model under tools/ that is used to check the kernels bit-for-bit).  Format constants are RFC 7932's;
// the encoder-side semantics follow the reference (dropbox/rust-brotli) files cited at each function.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stddef.h>

#ifdef __CUDACC__
#define BRO_HD __host__ __device__ __forceinline__
#define BRO_HD_NOINLINE __host__ __device__
#else
#define BRO_HD inline
#define BRO_HD_NOINLINE inline
#endif

namespace bro {

// ---------------------------------------------------------------------------------------------------
// small integer helpers
// ---------------------------------------------------------------------------------------------------
BRO_HD uint32_t log2_floor_nz(uint32_t v) {
#ifdef __CUDA_ARCH__
  return 31u - (uint32_t)__clz((int)v);
#else
  return 31u - (uint32_t)__builtin_clz(v);
#endif
}
BRO_HD uint32_t log2_floor_nz64(uint64_t v) {
#ifdef __CUDA_ARCH__
  return 63u - (uint32_t)__clzll((long long)v);
#else
  return 63u - (uint32_t)__builtin_clzll(v);
#endif
}
template <typename T> BRO_HD T bmin(T a, T b) { return a < b ? a : b; }
template <typename T> BRO_HD T bmax(T a, T b) { return a > b ? a : b; }

// ---------------------------------------------------------------------------------------------------
// Fixed-point log2 (Q16).  All cost arithmetic of this implementation is integer so that reductions are
// order-independent and the CPU model matches the GPU bit-for-bit.  lut[x] = round(log2(x) * 65536) for
// x in [1, 65535], lut[0] = 0; larger x are reduced to their top 16 bits.
// (Replaces the reference's f32 FastLog2 tables, util.rs:13-25 / bit_cost.rs:13-42.)
// ---------------------------------------------------------------------------------------------------
BRO_HD uint32_t log2_q16(const uint32_t* lut, uint32_t x) {
  if (x < 65536u) return lut[x];
  uint32_t s = log2_floor_nz(x) - 15u;
  return (s << 16) + lut[x >> s];
}
BRO_HD uint64_t xlog2x_q16(const uint32_t* lut, uint32_t x) { return (uint64_t)x * log2_q16(lut, x); }
// the table itself (host; 65536 entries)
inline void fill_log2_q16_lut(uint32_t* lut) {
  lut[0] = 0;
  for (uint32_t i = 1; i < 65536; ++i) lut[i] = (uint32_t)llround(log2((double)i) * 65536.0);
}

// ---------------------------------------------------------------------------------------------------
// RFC 7932 constants
// ---------------------------------------------------------------------------------------------------
BRO_HD uint32_t ins_base(uint32_t code) {
  static constexpr uint32_t t[24] = {0, 1, 2, 3, 4, 5, 6, 8, 10, 14, 18, 26, 34, 50, 66, 98, 130, 194, 322, 578, 1090, 2114, 6210, 22594};
  return t[code];
}
BRO_HD uint32_t ins_extra(uint32_t code) {
  static constexpr uint8_t t[24] = {0, 0, 0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 7, 8, 9, 10, 12, 14, 24};
  return t[code];
}
BRO_HD uint32_t copy_base(uint32_t code) {
  static constexpr uint32_t t[24] = {2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 14, 18, 22, 30, 38, 54, 70, 102, 134, 198, 326, 582, 1094, 2118};
  return t[code];
}
BRO_HD uint32_t copy_extra(uint32_t code) {
  static constexpr uint8_t t[24] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 7, 8, 9, 10, 24};
  return t[code];
}
BRO_HD uint32_t blocklen_offset(uint32_t code) {
  static constexpr uint32_t t[26] = {1, 5, 9, 13, 17, 25, 33, 41, 49, 65, 81, 97, 113, 145, 177, 209,
                          241, 305, 369, 497, 753, 1265, 2289, 4337, 8433, 16625};
  return t[code];
}
BRO_HD uint32_t blocklen_nbits(uint32_t code) {
  static constexpr uint8_t t[26] = {2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 6, 6, 7, 8, 9, 10, 11, 12, 13, 24};
  return t[code];
}
BRO_HD uint32_t blocklen_prefix_code(uint32_t len) {  // brotli_bit_stream.rs:1370-1388
  uint32_t code = (len >= 177) ? (len >= 753 ? 20u : 14u) : (len >= 41 ? 7u : 0u);
  while (code < 25 && len >= blocklen_offset(code + 1)) ++code;
  return code;
}

// UTF8 literal context (RFC 7932 7.1).  lut0 is indexed by the previous byte, lut1 by the one before.
BRO_HD uint8_t utf8_lut0(uint32_t c) {
  static constexpr uint8_t ascii0[128] = {
      0,  0,  0,  0,  0,  0,  0,  0,  0,  4,  4,  0,  0,  4,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,
      0,  0,  0,  0,  0,  0,  8,  12, 16, 12, 12, 20, 12, 16, 24, 28, 12, 12, 32, 12, 36, 12, 44, 44, 44, 44,
      44, 44, 44, 44, 44, 44, 32, 32, 24, 40, 28, 12, 12, 48, 52, 52, 52, 48, 52, 52, 52, 48, 52, 52, 52, 52,
      52, 48, 52, 52, 52, 52, 52, 48, 52, 52, 52, 52, 52, 24, 12, 28, 12, 12, 12, 56, 60, 60, 60, 56, 60, 60,
      60, 56, 60, 60, 60, 60, 60, 56, 60, 60, 60, 60, 60, 56, 60, 60, 60, 60, 60, 24, 12, 28, 12, 0};
  if (c < 128) return ascii0[c];
  if (c < 192) return (uint8_t)(c & 1);
  return (uint8_t)(2 + (c & 1));
}
BRO_HD uint8_t utf8_lut1(uint32_t c) {
  if (c < 32) return 0;
  if (c < 128) {
    if (c == 32 || c == 127) return 0;
    if (c >= '0' && c <= '9') return 2;
    if (c >= 'A' && c <= 'Z') return 2;
    if (c >= 'a' && c <= 'z') return 3;
    return 1;
  }
  if (c < 224) return 0;
  return 2;
}
BRO_HD uint32_t context_utf8(uint8_t p1, uint8_t p2) { return utf8_lut0(p1) | utf8_lut1(p2); }

// SIGNED literal context (RFC 7932 7.1): 3-bit class of each of the two previous bytes
BRO_HD uint32_t signed_lut(uint32_t c) {
  if (c == 0) return 0;
  if (c < 16) return 1;
  if (c < 64) return 2;
  if (c < 128) return 3;
  if (c < 192) return 4;
  if (c < 240) return 5;
  if (c < 255) return 6;
  return 7;
}
BRO_HD uint32_t context_signed(uint8_t p1, uint8_t p2) { return (signed_lut(p1) << 3) | signed_lut(p2); }

// static literal context maps (encode.rs:1723-1732, 1782-1798); id 0 = no context modelling.  Ids 4 / 5 (quality >= 10): all 64
// contexts of the UTF8 / SIGNED mode, mapped to prefix codes by a clustered context map (metablock.rs:133-301).
enum { CTXMAP_NONE = 0, CTXMAP_SIMPLE2 = 1, CTXMAP_CONT3 = 2, CTXMAP_COMPLEX13 = 3, CTXMAP_FULL_UTF8 = 4, CTXMAP_FULL_SIGNED = 5 };
BRO_HD uint32_t ctxmap_num_contexts(int id) { return id == 0 ? 1u : id == 1 ? 2u : id == 2 ? 3u : id == 3 ? 13u : 64u; }
BRO_HD uint32_t literal_context(int id, uint8_t p1, uint8_t p2) { return id == CTXMAP_FULL_SIGNED ? context_signed(p1, p2) : context_utf8(p1, p2); }
// context of a command's distance symbol (CommandDistanceContext, command.rs:203-215)
BRO_HD uint32_t distance_context(uint32_t cmd_prefix) {
  const uint32_t r = cmd_prefix >> 6, c = cmd_prefix & 7u;
  if ((r == 0 || r == 2 || r == 4 || r == 7) && c <= 2) return c;
  return 3;
}
BRO_HD uint32_t ctxmap_lookup(int id, uint32_t ctx6) {
  static constexpr uint8_t complex13[64] = {11, 11, 12, 12, 0, 0, 0, 0, 1, 1, 9, 9, 2, 2, 2, 2, 1, 1, 1, 1, 8, 3,
                                 3,  3,  1,  1,  1, 1, 2, 2, 2, 2, 8, 4, 4, 4, 8, 7, 4, 4, 8, 0, 0, 0,
                                 3,  3,  3,  3,  5, 5, 10, 5, 5, 5, 10, 5, 6, 6, 6, 6, 6, 6, 6, 6};
  if (id == CTXMAP_NONE) return 0;
  if (id >= CTXMAP_FULL_UTF8) return ctx6;
  if (id == CTXMAP_SIMPLE2) return (ctx6 == 2 || ctx6 == 3) ? 1u : 0u;
  if (id == CTXMAP_CONT3) return ctx6 < 2 ? 1u : (ctx6 < 4 ? 2u : 0u);
  return complex13[ctx6];
}

// ---------------------------------------------------------------------------------------------------
// Command codes: command.rs:48-68, 71-121, 134-173 (NPOSTFIX = NDIRECT = 0)
// ---------------------------------------------------------------------------------------------------
BRO_HD uint32_t insert_length_code(uint32_t insertlen) {
  if (insertlen < 6) return insertlen;
  if (insertlen < 130) {
    uint32_t nbits = log2_floor_nz(insertlen - 2) - 1u;
    return (nbits << 1) + ((insertlen - 2) >> nbits) + 2;
  }
  if (insertlen < 2114) return log2_floor_nz(insertlen - 66) + 10;
  if (insertlen < 6210) return 21;
  if (insertlen < 22594) return 22;
  return 23;
}
BRO_HD uint32_t copy_length_code(uint32_t copylen) {
  if (copylen < 10) return copylen - 2;
  if (copylen < 134) {
    uint32_t nbits = log2_floor_nz(copylen - 6) - 1u;
    return (nbits << 1) + ((copylen - 6) >> nbits) + 4;
  }
  if (copylen < 2118) return log2_floor_nz(copylen - 70) + 12;
  return 23;
}
BRO_HD uint32_t combine_length_codes(uint32_t inscode, uint32_t copycode, bool use_last_distance) {
  uint32_t bits64 = (copycode & 0x7u) | ((inscode & 0x7u) << 3);
  if (use_last_distance && inscode < 8 && copycode < 16) return (copycode < 8) ? bits64 : (bits64 | 64u);
  uint32_t sub_offset = 2 * ((copycode >> 3) + 3 * (inscode >> 3));
  uint32_t offset = (sub_offset << 5) + 0x40u + ((0x520D40u >> sub_offset) & 0xC0u);
  return offset | bits64;
}
// distance -> short code given the 4-entry cache (most recent first); returns distance + 15 when no short code fits
BRO_HD uint32_t compute_distance_code(uint32_t distance, const int32_t* dc) {
  uint32_t d3 = distance + 3;
  uint32_t offset0 = d3 - (uint32_t)dc[0];
  uint32_t offset1 = d3 - (uint32_t)dc[1];
  if (distance == (uint32_t)dc[0]) return 0;
  if (distance == (uint32_t)dc[1]) return 1;
  if (offset0 < 7) return (0x09750468u >> (4 * offset0)) & 0xF;
  if (offset1 < 7) return (0x0FDB1ACEu >> (4 * offset1)) & 0xF;
  if (distance == (uint32_t)dc[2]) return 2;
  if (distance == (uint32_t)dc[3]) return 3;
  return distance + 15;
}
// distance code -> (symbol | nbits << 10, extra)
BRO_HD void prefix_encode_copy_distance(uint32_t distance_code, uint32_t* sym_nbits, uint32_t* extra) {
  if (distance_code < 16) {
    *sym_nbits = distance_code;
    *extra = 0;
  } else {
    uint32_t dist = 4u + (distance_code - 16u);
    uint32_t bucket = log2_floor_nz(dist) - 1u;
    uint32_t prefix = (dist >> bucket) & 1u;
    uint32_t offset = (2u + prefix) << bucket;
    *sym_nbits = (bucket << 10) | (16u + 2u * (bucket - 1u) + prefix);
    *extra = dist - offset;
  }
}

// General form with NPOSTFIX / NDIRECT (PrefixEncodeCopyDistance, command.rs:134-173); quality >= 10 searches these per metablock.
BRO_HD void prefix_encode_copy_distance_params(uint32_t distance_code, uint32_t npostfix, uint32_t ndirect, uint32_t* sym_nbits, uint32_t* extra) {
  if (distance_code < 16u + ndirect) {
    *sym_nbits = distance_code;
    *extra = 0;
    return;
  }
  const uint32_t dist = (1u << (npostfix + 2u)) + (distance_code - 16u - ndirect);
  const uint32_t bucket = log2_floor_nz(dist) - 1u;
  const uint32_t postfix = dist & ((1u << npostfix) - 1u);
  const uint32_t prefix = (dist >> bucket) & 1u;
  const uint32_t offset = (2u + prefix) << bucket;
  const uint32_t nbits = bucket - npostfix;
  *sym_nbits = (nbits << 10) | (16u + ndirect + ((2u * (nbits - 1u) + prefix) << npostfix) + postfix);
  *extra = (dist - offset) >> npostfix;
}
// distance code of a command that was encoded with NPOSTFIX = NDIRECT = 0 (Command::restore_distance_code, command.rs:176-200)
BRO_HD uint32_t restore_distance_code00(uint32_t sym_nbits, uint32_t extra) {
  const uint32_t sym = sym_nbits & 0x3ffu;
  if (sym < 16) return sym;
  const uint32_t nbits = sym_nbits >> 10, hcode = sym - 16u;
  return ((2u + (hcode & 1u)) << nbits) - 4u + extra + 16u;
}
BRO_HD uint32_t distance_alphabet_size(uint32_t npostfix, uint32_t ndirect) { return 16u + ndirect + (48u << npostfix); }
#define BRO_DIST_A_MAX 544u  // histogram width of the distance alphabet when NPOSTFIX / NDIRECT are searched (<= 520 symbols)
// The reference's search order over (NPOSTFIX, NDIRECT) given the cost of every combination (metablock.rs:152-207):
// cost[npostfix * 16 + ndirect_msb], ndirect = ndirect_msb << npostfix.  Returns npostfix | ndirect << 8.
BRO_HD uint32_t choose_distance_params(const uint64_t* cost) {
  uint64_t best = ~0ull;
  uint32_t best_np = 0, best_nd = 0, msb = 0;
  bool check_orig = true;
  for (uint32_t np = 0; np <= 3; ++np) {
    while (msb < 16) {
      const uint32_t nd = msb << np;
      if (np == 0 && nd == 0) check_orig = false;
      const uint64_t c = cost[np * 16 + msb];
      if (c > best) break;
      best = c;
      best_np = np;
      best_nd = nd;
      ++msb;
    }
    if (msb > 0) --msb;
    msb /= 2;
  }
  if (check_orig && cost[0] < best) { best_np = 0; best_nd = 0; }
  return best_np | (best_nd << 8);
}

// Final command record produced by the command-finalise stage (the analogue of command.rs:11-21).
struct Cmd {
  uint32_t insert_len;
  uint32_t copy_len;    // 0 for the trailing insert-only command of a metablock
  uint32_t dist_extra;
  uint16_t cmd_prefix;
  uint16_t dist_prefix;  // symbol | nbits << 10 ; valid iff has_distance()
  BRO_HD bool has_distance() const { return copy_len != 0 && cmd_prefix >= 128; }
};
// Raw match record written by the parse stage.
struct RawCmd {
  uint32_t insert_len;
  uint32_t copy_len;
  uint32_t distance;
};

// ---------------------------------------------------------------------------------------------------
// Sequential LSB-first bit writer over a byte buffer that this thread owns exclusively
// (brotli_bit_stream.rs:742-757).
// ---------------------------------------------------------------------------------------------------
struct BitWriter {
  uint8_t* buf;
  uint64_t acc;
  uint32_t nacc;   // bits in acc (< 8 after flush)
  uint64_t nbytes; // bytes already flushed
  BRO_HD void init(uint8_t* b) { buf = b; acc = 0; nacc = 0; nbytes = 0; }
  BRO_HD void put(uint32_t nbits, uint64_t bits) {  // nbits <= 32
    acc |= bits << nacc;
    nacc += nbits;
    while (nacc >= 8) {
      buf[nbytes++] = (uint8_t)acc;
      acc >>= 8;
      nacc -= 8;
    }
  }
  BRO_HD void skip(uint32_t nbits) { while (nbits) { uint32_t k = nbits > 32 ? 32 : nbits; put(k, 0); nbits -= k; } }
  BRO_HD uint64_t bit_pos() const { return nbytes * 8 + nacc; }
  BRO_HD void flush_partial() {
    if (nacc) buf[nbytes] = (uint8_t)acc;  // keeps nacc so that bit_pos stays correct
  }
};

}  // namespace bro

// bro_meta.cuh -- metablock header serialisation and per-command body emission.
//
// Reference semantics: store_meta_block (brotli_bit_stream.rs:2035-2261) with its helpers
// StoreCompressedMetaBlockHeader :1292, BuildAndStoreBlockSplitCode :1536, StoreBlockSwitch :1506,
// StoreTrivialContextMap :1613, EncodeContextMap :1783, StoreCommandExtra :1947.
// GPU re-design: the header of a metablock is produced by one thread into a private scratch buffer; the
// body is emitted by one thread per command at a bit offset obtained from a prefix sum of exact bit
// lengths (the same routine is instantiated with a counting writer and with an atomic-OR writer).
#pragma once
#include "bro_common.cuh"
#include "bro_huffman.cuh"

namespace bro {

// One block-split category (literals / commands / distances) of one metablock.
struct SplitView {
  uint32_t num_types;
  uint32_t num_blocks;
  const uint8_t* types;     // [num_blocks]
  const uint32_t* lengths;  // [num_blocks]
  const uint32_t* starts;   // [num_blocks] exclusive prefix sum of lengths
};
struct SplitCode {
  uint8_t type_depth[258];
  uint16_t type_code[258];
  uint8_t len_depth[26];
  uint16_t len_code[26];
};

BRO_HD void store_var_len_uint8(BitWriter& bw, uint32_t n) {
  if (n == 0) bw.put(1, 0);
  else {
    uint32_t nbits = log2_floor_nz(n);
    bw.put(1, 1);
    bw.put(3, nbits);
    bw.put(nbits, n - (1u << nbits));
  }
}
// type code of block b given the two previous block types (brotli_bit_stream.rs:1357-1368)
BRO_HD uint32_t block_type_code(const uint8_t* types, uint32_t b) {
  uint32_t t = types[b];
  uint32_t last = b >= 1 ? types[b - 1] : 1u;
  uint32_t second = b >= 2 ? types[b - 2] : (b == 1 ? 1u : 0u);
  if (b == 0) { last = 1; second = 0; }
  if (t == last + 1) return 1;
  if (t == second) return 0;
  return t + 2;
}
template <typename W>
BRO_HD void put_block_switch(W& w, const SplitView& sv, const SplitCode& sc, uint32_t b, bool is_first) {
  if (!is_first) {
    uint32_t tc = block_type_code(sv.types, b);
    w.put(sc.type_depth[tc], sc.type_code[tc]);
  }
  uint32_t len = sv.lengths[b];
  uint32_t lc = blocklen_prefix_code(len);
  w.put(sc.len_depth[lc], sc.len_code[lc]);
  w.put(blocklen_nbits(lc), len - blocklen_offset(lc));
}
BRO_HD_NOINLINE void store_block_split_code(BitWriter& bw, const SplitView& sv, SplitCode* sc, HuffStoreWs* ws) {
  uint32_t type_histo[258], length_histo[26];
  for (int i = 0; i < 258; ++i) type_histo[i] = 0;
  for (int i = 0; i < 26; ++i) length_histo[i] = 0;
  for (uint32_t b = 0; b < sv.num_blocks; ++b) {
    if (b != 0) ++type_histo[block_type_code(sv.types, b)];
    ++length_histo[blocklen_prefix_code(sv.lengths[b])];
  }
  store_var_len_uint8(bw, sv.num_types - 1);
  if (sv.num_types > 1) {
    huff_build_and_store(bw, type_histo, sv.num_types + 2, sv.num_types + 2, ws, sc->type_depth, sc->type_code);
    huff_build_and_store(bw, length_histo, 26, 26, ws, sc->len_depth, sc->len_code);
    put_block_switch(bw, sv, *sc, 0, true);
  }
}
BRO_HD_NOINLINE void store_trivial_context_map(BitWriter& bw, uint32_t num_types, uint32_t context_bits, HuffStoreWs* ws) {
  store_var_len_uint8(bw, num_types - 1);
  if (num_types > 1) {
    uint32_t repeat_code = context_bits - 1;
    uint32_t repeat_bits = (1u << repeat_code) - 1;
    uint32_t alphabet_size = num_types + repeat_code;
    uint32_t histogram[272];
    uint8_t depths[272];
    uint16_t bits[272];
    for (uint32_t i = 0; i < 272; ++i) histogram[i] = 0;
    bw.put(1, 1);
    bw.put(4, repeat_code - 1);
    histogram[repeat_code] = num_types;
    histogram[0] = 1;
    for (uint32_t i = context_bits; i < alphabet_size; ++i) histogram[i] = 1;
    huff_build_and_store(bw, histogram, alphabet_size, alphabet_size, ws, depths, bits);
    for (uint32_t i = 0; i < num_types; ++i) {
      uint32_t code = i == 0 ? 0 : i + context_bits - 1;
      bw.put(depths[code], bits[code]);
      bw.put(depths[repeat_code], bits[repeat_code]);
      bw.put(repeat_code, repeat_bits);
    }
    bw.put(1, 1);
  }
}
// Literal context map of a metablock with static contexts: entry (type, ctx6) -> type * nctx + static_map[ctx6]
// (metablock.rs:832-857), serialised per brotli_bit_stream.rs:1690-1858.  rle: workspace of num_types * 64 u32.
BRO_HD_NOINLINE void store_static_literal_context_map(BitWriter& bw, uint32_t num_types, int map_id, uint32_t* rle,
                                                      HuffStoreWs* ws) {
  const uint32_t nctx = ctxmap_num_contexts(map_id);
  const uint32_t num_clusters = num_types * nctx;
  const uint32_t size = num_types << 6;
  store_var_len_uint8(bw, num_clusters - 1);
  if (num_clusters == 1) return;
  {  // move-to-front transform
    uint8_t mtf[256];
    for (uint32_t i = 0; i < num_clusters; ++i) mtf[i] = (uint8_t)i;
    for (uint32_t i = 0; i < size; ++i) {
      uint32_t v = (i >> 6) * nctx + ctxmap_lookup(map_id, i & 63);
      uint32_t index = 0;
      while (mtf[index] != (uint8_t)v) ++index;
      rle[i] = index;
      uint8_t value = mtf[index];
      for (uint32_t k = index; k != 0; --k) mtf[k] = mtf[k - 1];
      mtf[0] = value;
    }
  }
  uint32_t max_run_length_prefix = 6, out_size = 0;
  {  // RunLengthCodeZeros
    uint32_t max_reps = 0;
    for (uint32_t i = 0; i < size;) {
      uint32_t reps = 0;
      for (; i < size && rle[i] != 0; ++i) {}
      for (; i < size && rle[i] == 0; ++i) ++reps;
      max_reps = bmax(reps, max_reps);
    }
    uint32_t max_prefix = max_reps > 0 ? log2_floor_nz(max_reps) : 0;
    max_prefix = bmin(max_prefix, max_run_length_prefix);
    max_run_length_prefix = max_prefix;
    for (uint32_t i = 0; i < size;) {
      if (rle[i] != 0) {
        rle[out_size++] = rle[i] + max_run_length_prefix;
        ++i;
      } else {
        uint32_t reps = 1;
        for (uint32_t k = i + 1; k < size && rle[k] == 0; ++k) ++reps;
        i += reps;
        while (reps != 0) {
          if (reps < (2u << max_prefix)) {
            uint32_t p = log2_floor_nz(reps);
            rle[out_size++] = p + ((reps - (1u << p)) << 9);
            break;
          } else {
            rle[out_size++] = max_prefix + (((1u << max_prefix) - 1u) << 9);
            reps -= (2u << max_prefix) - 1u;
          }
        }
      }
    }
  }
  uint32_t histogram[272];
  uint8_t depths[272];
  uint16_t bits[272];
  for (uint32_t i = 0; i < 272; ++i) histogram[i] = 0;
  for (uint32_t i = 0; i < out_size; ++i) ++histogram[rle[i] & 0x1ff];
  bool use_rle = max_run_length_prefix > 0;
  bw.put(1, use_rle ? 1u : 0u);
  if (use_rle) bw.put(4, max_run_length_prefix - 1);
  huff_build_and_store(bw, histogram, num_clusters + max_run_length_prefix, num_clusters + max_run_length_prefix, ws,
                       depths, bits);
  for (uint32_t i = 0; i < out_size; ++i) {
    uint32_t sym = rle[i] & 0x1ff, extra = rle[i] >> 9;
    bw.put(depths[sym], bits[sym]);
    if (sym > 0 && sym <= max_run_length_prefix) bw.put(sym, extra);
  }
  bw.put(1, 1);
}

// General context map (EncodeContextMap, brotli_bit_stream.rs:1783-1858): cmap[size] -> cluster < num_clusters.
// rle: workspace of `size` u32.
BRO_HD_NOINLINE void store_context_map(BitWriter& bw, const uint8_t* cmap, uint32_t size, uint32_t num_clusters, uint32_t* rle,
                                       HuffStoreWs* ws) {
  store_var_len_uint8(bw, num_clusters - 1);
  if (num_clusters == 1) return;
  {  // move-to-front transform
    uint8_t mtf[256];
    for (uint32_t i = 0; i < 256; ++i) mtf[i] = (uint8_t)i;
    for (uint32_t i = 0; i < size; ++i) {
      const uint8_t v = cmap[i];
      uint32_t index = 0;
      while (mtf[index] != v) ++index;
      rle[i] = index;
      for (uint32_t k = index; k != 0; --k) mtf[k] = mtf[k - 1];
      mtf[0] = v;
    }
  }
  uint32_t max_run_length_prefix = 6, out_size = 0;
  {  // RunLengthCodeZeros
    uint32_t max_reps = 0;
    for (uint32_t i = 0; i < size;) {
      uint32_t reps = 0;
      for (; i < size && rle[i] != 0; ++i) {}
      for (; i < size && rle[i] == 0; ++i) ++reps;
      max_reps = bmax(reps, max_reps);
    }
    uint32_t max_prefix = max_reps > 0 ? log2_floor_nz(max_reps) : 0;
    max_prefix = bmin(max_prefix, max_run_length_prefix);
    max_run_length_prefix = max_prefix;
    for (uint32_t i = 0; i < size;) {
      if (rle[i] != 0) {
        rle[out_size++] = rle[i] + max_run_length_prefix;
        ++i;
      } else {
        uint32_t reps = 1;
        for (uint32_t k = i + 1; k < size && rle[k] == 0; ++k) ++reps;
        i += reps;
        while (reps != 0) {
          if (reps < (2u << max_prefix)) {
            uint32_t p = log2_floor_nz(reps);
            rle[out_size++] = p + ((reps - (1u << p)) << 9);
            break;
          } else {
            rle[out_size++] = max_prefix + (((1u << max_prefix) - 1u) << 9);
            reps -= (2u << max_prefix) - 1u;
          }
        }
      }
    }
  }
  uint32_t histogram[272];
  uint8_t depths[272];
  uint16_t bits[272];
  for (uint32_t i = 0; i < 272; ++i) histogram[i] = 0;
  for (uint32_t i = 0; i < out_size; ++i) ++histogram[rle[i] & 0x1ff];
  const bool use_rle = max_run_length_prefix > 0;
  bw.put(1, use_rle ? 1u : 0u);
  if (use_rle) bw.put(4, max_run_length_prefix - 1);
  huff_build_and_store(bw, histogram, num_clusters + max_run_length_prefix, num_clusters + max_run_length_prefix, ws, depths, bits);
  for (uint32_t i = 0; i < out_size; ++i) {
    const uint32_t sym = rle[i] & 0x1ff, extra = rle[i] >> 9;
    bw.put(depths[sym], bits[sym]);
    if (sym > 0 && sym <= max_run_length_prefix) bw.put(sym, extra);
  }
  bw.put(1, 1);  // inverse move-to-front at the decoder
}

BRO_HD void store_compressed_metablock_header(BitWriter& bw, bool is_last, uint32_t length) {
  bw.put(1, is_last ? 1u : 0u);
  if (is_last) bw.put(1, 0);
  uint32_t lg = length == 1 ? 1u : log2_floor_nz(length - 1) + 1u;
  uint32_t mnibbles = (lg < 16 ? 16u : lg + 3u) / 4u;
  bw.put(2, mnibbles - 4);
  bw.put(mnibbles * 4, length - 1);
  if (!is_last) bw.put(1, 0);
}
// number of bits of an uncompressed-metablock header before byte alignment (ISLAST=0, MNIBBLES, MLEN-1, ISUNCOMPRESSED=1)
BRO_HD uint32_t raw_metablock_header_bits(uint32_t length) {
  uint32_t lg = length == 1 ? 1u : log2_floor_nz(length - 1) + 1u;
  uint32_t mnibbles = (lg < 16 ? 16u : lg + 3u) / 4u;
  return 1 + 2 + mnibbles * 4 + 1;
}

// ---------------------------------------------------------------------------------------------------
// Per-metablock coding tables as the emission stage sees them.
// ---------------------------------------------------------------------------------------------------
struct MetaCodes {
  SplitView lit, cmd, dist;
  const SplitCode *lit_sc, *cmd_sc, *dist_sc;
  const uint8_t* lit_depth;   // [lit trees][256]
  const uint16_t* lit_code;
  const uint8_t* cmd_depth;   // [cmd types][704]
  const uint16_t* cmd_code;
  const uint8_t* dist_depth;  // [dist types][64]
  const uint16_t* dist_code;
  int ctx_map_id;
  uint32_t nctx;
  // quality >= 10 (ctx_map_id >= CTXMAP_FULL_UTF8): clustered context maps, entries are prefix-code indices
  const uint8_t* lit_cmap;    // [lit types][64]
  const uint8_t* dist_cmap;   // [dist types][4], null = one code per distance block type
  uint32_t dist_A;            // width of a distance code table: 64, or BRO_DIST_A_MAX when NPOSTFIX / NDIRECT are searched
};
BRO_HD uint32_t literal_tree(const MetaCodes& mc, uint32_t type, uint8_t p1, uint8_t p2) {
  if (mc.ctx_map_id >= CTXMAP_FULL_UTF8) return mc.lit_cmap[type * 64u + literal_context(mc.ctx_map_id, p1, p2)];
  uint32_t tree = type * mc.nctx;
  if (mc.ctx_map_id) tree += ctxmap_lookup(mc.ctx_map_id, context_utf8(p1, p2));
  return tree;
}

// largest b with starts[b] <= idx
BRO_HD uint32_t find_block(const uint32_t* starts, uint32_t num_blocks, uint32_t idx) {
  uint32_t lo = 0, hi = num_blocks;
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (starts[mid] <= idx) lo = mid; else hi = mid;
  }
  return lo;
}

// Bits of the literal of rank `rank` (block switch that falls on it + its code); used by the long-insert kernels.
static constexpr uint32_t NOT_LONG = 0xFFFFFFFFu;
template <typename W>
BRO_HD void emit_one_literal(W& w, const MetaCodes& mc, uint32_t rank, const uint8_t* data, uint32_t pos, uint32_t abs_base) {
  uint32_t b = 0;
  if (mc.lit.num_blocks > 1) {
    b = find_block(mc.lit.starts, mc.lit.num_blocks, rank);
    if (b > 0 && mc.lit.starts[b] == rank) put_block_switch(w, mc.lit, *mc.lit_sc, b, false);
  }
  uint32_t tree = mc.lit.types[b] * mc.nctx;
  if (mc.ctx_map_id) {
    uint8_t p1 = ((uint64_t)abs_base + pos >= 1) ? data[(int64_t)pos - 1] : 0, p2 = ((uint64_t)abs_base + pos >= 2) ? data[(int64_t)pos - 2] : 0;
    tree = literal_tree(mc, mc.lit.types[b], p1, p2);
  }
  const uint8_t lit = data[pos];
  w.put(mc.lit_depth[tree * 256 + lit], mc.lit_code[tree * 256 + lit]);
}
// Bits a command writes before its literals (command block switch, command symbol, insert/copy extra bits).
template <typename W>
BRO_HD void emit_command_head(W& w, const MetaCodes& mc, const Cmd& c, uint32_t cmd_idx) {
  uint32_t b = 0;
  if (mc.cmd.num_blocks > 1) {
    b = find_block(mc.cmd.starts, mc.cmd.num_blocks, cmd_idx);
    if (b > 0 && mc.cmd.starts[b] == cmd_idx) put_block_switch(w, mc.cmd, *mc.cmd_sc, b, false);
  }
  uint32_t t = mc.cmd.types[b];
  w.put(mc.cmd_depth[t * 704 + c.cmd_prefix], mc.cmd_code[t * 704 + c.cmd_prefix]);
  // StoreCommandExtra: brotli_bit_stream.rs:1947-1961
  uint32_t copylen_code = c.copy_len ? c.copy_len : 4u;
  uint32_t inscode = insert_length_code(c.insert_len), copycode = copy_length_code(copylen_code);
  uint32_t insnumextra = ins_extra(inscode);
  uint64_t v = ((uint64_t)(copylen_code - copy_base(copycode)) << insnumextra) | (c.insert_len - ins_base(inscode));
  uint32_t nb = insnumextra + copy_extra(copycode);
  if (nb > 32) { w.put(32, (uint32_t)v); w.put(nb - 32, v >> 32); }
  else w.put(nb, v);
}

// Emits (or counts) all bits of command `c`: block switches that fall on its symbols, the command symbol and
// extra bits, its literals, its distance.  cmd_idx / lit_idx / dist_idx are symbol ranks inside the metablock,
// pos = input position of the first literal of the command.
template <typename W>
BRO_HD_NOINLINE void emit_command(W& w, const MetaCodes& mc, const Cmd& c, uint32_t cmd_idx, uint32_t lit_idx,
                                  uint32_t dist_idx, const uint8_t* data, uint32_t pos, uint32_t abs_base,
                                  uint32_t long_lit_bits = NOT_LONG) {
  emit_command_head(w, mc, c, cmd_idx);
  if (long_lit_bits != NOT_LONG) {
    w.skip(long_lit_bits);  // the literals of a long insert are counted / written by the k_*_long kernels
  } else if (c.insert_len) {
    uint32_t b = 0, bend = 0xFFFFFFFFu;
    if (mc.lit.num_blocks > 1) {
      b = find_block(mc.lit.starts, mc.lit.num_blocks, lit_idx);
      bend = (b + 1 < mc.lit.num_blocks) ? mc.lit.starts[b + 1] : 0xFFFFFFFFu;
      if (b > 0 && mc.lit.starts[b] == lit_idx) put_block_switch(w, mc.lit, *mc.lit_sc, b, false);
    }
    uint32_t type = mc.lit.types[b];
    uint8_t p1 = ((uint64_t)abs_base + pos >= 1) ? data[(int64_t)pos - 1] : 0, p2 = ((uint64_t)abs_base + pos >= 2) ? data[(int64_t)pos - 2] : 0;
    for (uint32_t j = 0; j < c.insert_len; ++j) {
      if (lit_idx + j == bend) {
        ++b;
        bend = (b + 1 < mc.lit.num_blocks) ? mc.lit.starts[b + 1] : 0xFFFFFFFFu;
        put_block_switch(w, mc.lit, *mc.lit_sc, b, false);
        type = mc.lit.types[b];
      }
      uint8_t lit = data[pos + j];
      const uint32_t tree = literal_tree(mc, type, p1, p2);
      w.put(mc.lit_depth[tree * 256 + lit], mc.lit_code[tree * 256 + lit]);
      p2 = p1;
      p1 = lit;
    }
  }
  if (c.has_distance()) {
    uint32_t b = 0;
    if (mc.dist.num_blocks > 1) {
      b = find_block(mc.dist.starts, mc.dist.num_blocks, dist_idx);
      if (b > 0 && mc.dist.starts[b] == dist_idx) put_block_switch(w, mc.dist, *mc.dist_sc, b, false);
    }
    uint32_t t = mc.dist.types[b];
    if (mc.dist_cmap) t = mc.dist_cmap[t * 4u + distance_context(c.cmd_prefix)];
    uint32_t sym = c.dist_prefix & 0x3ffu;
    w.put(mc.dist_depth[t * mc.dist_A + sym], mc.dist_code[t * mc.dist_A + sym]);
    w.put(c.dist_prefix >> 10, c.dist_extra);
  }
}

struct CountWriter {
  uint64_t bits;
  BRO_HD void put(uint32_t n, uint64_t) { bits += n; }
  BRO_HD void skip(uint32_t n) { bits += n; }
};

}  // namespace bro

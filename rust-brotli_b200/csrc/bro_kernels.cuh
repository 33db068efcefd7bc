// bro_kernels.cuh -- CUDA kernels (sm_90a) of the brotli compression hot path.
//
// Stage map (DESIGN.md has the data layout and the per-kernel roofline):
//   sort    k_sort_count / k_sort_onesweep (x2)   stable one-sweep LSD radix sort of positions by bucket key
//                                                 (replaces hasher Store*)
//   match   k_match_shallow / k_match_deep   every position vs the `depth` most recent earlier positions of its bucket
//                            (replaces the bucket walk of FindLongestMatch, backward_references/mod.rs:1754-1792)
//   parse   k_parse          greedy+lazy parse per unit (CreateBackwardReferences mod.rs:2376)
//   final   k_fin_count / k_fin_write / k_fin_dist    command records, literal/distance ranks
//   ctx     k_ctx_decide     literal context map choice (encode.rs:1873)
//   syms    k_symbols        symbol streams for the splitter
//   split   k_split_greedy   histograms + greedy block split (metablock.rs:551-1021)
//   header  k_header         Huffman codes + metablock header bits (brotli_bit_stream.rs:2035-2190)
//   emit    k_bitlen / k_bitscan / k_layout / k_emit_header / k_emit_body / k_emit_raw
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "bro_common.cuh"
#include "bro_encoder.h"
#include "bro_finalize.cuh"
#include "bro_huffman.cuh"
#include "bro_meta.cuh"
#include "bro_parse.cuh"
#include "bro_split.cuh"
#include "bro_hq.cuh"

namespace bro {

// ---------------------------------------------------------------------------------------------------
// device-side descriptors
// ---------------------------------------------------------------------------------------------------
struct MBDesc {
  uint32_t start, len;        // input span
  uint32_t u0, u1;            // parse units
  uint32_t ncmd, nlit, ndist; // symbol counts
  int ctx_map_id;
  uint32_t hdr_bits;
  uint32_t raw;               // stored uncompressed
  uint32_t has_long;          // some command has more than LONG_INS literals
  uint32_t dist_params;       // NPOSTFIX | NDIRECT << 8 (0 below quality 10)
  uint64_t body_bits;
  uint64_t out_bitpos;        // position of the metablock in the output stream
};

struct SplitArrays {  // per metablock, per category
  uint8_t* types;
  uint32_t* lengths;
  uint32_t* starts;
  uint32_t* num_blocks;   // [1]
  uint32_t* num_types;    // [1]
  uint32_t* histograms;   // [(max_types + 1)][nctx * A]
  SplitCode* sc;
};

struct Workspace {
  // input
  const uint8_t* data;  // padded with >= 320 zero bytes
  const uint32_t* lut;
  DictView dict;        // static dictionary words + hash table (device copies)
  EncParams P;
  uint32_t num_units, num_mb;
  // match
  uint32_t* best;
  HqMatch* hqm;         // quality >= 10: [n][HQ_MAXM] all matches per position (range-relative index)
  uint8_t* hqn;         //                [n] number of matches
  // parse
  RawCmd* raw;
  uint32_t *unit_ncmd, *unit_tail, *unit_ncopy;
  uint32_t *unit_cmd_off, *unit_lit_off, *unit_ndist, *unit_dist_off;  // metablock-relative
  // commands
  GCmd* cmds;           // [num_mb][cmd_cap]
  uint32_t cmd_cap;     // per metablock
  uint32_t* cmd_bits;   // [num_mb][cmd_cap] exclusive bit prefix inside the command's 256-tile
  uint32_t* cmd_tile;   // [num_mb][tile_cap] tile totals, then exclusive tile offsets
  uint32_t tile_cap;
  uint2* long_tab;      // [num_mb][long_cap] long-insert commands by (pos - mb.start) / LONG_INS: x = command + 1, y = literal bits
  uint32_t* seg_bits;   // [num_mb][long_cap] literal bits of each LONG_INS-literal segment of a long insert
  uint32_t long_cap;
  // symbol streams
  uint16_t* lit_syms;   // [n]  literal | ctx << 8, metablock m at m.start
  uint16_t* cmd_syms;   // [num_mb][cmd_cap]
  uint16_t* dist_syms;  // [num_mb][cmd_cap]
  // metablocks
  MBDesc* mb;
  // splits: capacities per metablock
  uint32_t lit_blk_cap, cmd_blk_cap, dist_blk_cap;
  uint32_t max_lit_trees, max_cmd_types, max_dist_types;
  uint32_t dist_A;         // width of a distance histogram / code table: 64, or BRO_DIST_A_MAX when NPOSTFIX / NDIRECT are searched
  uint8_t *lit_types, *cmd_types, *dist_types;
  uint32_t *lit_lengths, *cmd_lengths, *dist_lengths;
  uint32_t *lit_starts, *cmd_starts, *dist_starts;
  uint32_t* split_counts;  // [num_mb][6]: lit nb, lit nt, cmd nb, cmd nt, dist nb, dist nt
  uint32_t *lit_hist, *cmd_hist, *dist_hist;
  SplitCode* split_codes;  // [num_mb][3]
  // codes
  uint8_t *lit_depth, *cmd_depth, *dist_depth;
  uint16_t *lit_code, *cmd_code, *dist_code;
  // header
  uint8_t* hdr;           // [num_mb][hdr_cap]
  uint32_t hdr_cap;
  uint8_t* tree_bits;     // [num_mb][tree_cap][TREE_SLOT_BYTES]
  uint32_t* tree_nbits;   // [num_mb][tree_cap]
  uint8_t* sect_bits;     // [num_mb][HDR_SECTIONS][SECT_BYTES] header sections built beside the trees
  uint32_t* sect_nbits;   // [num_mb][HDR_SECTIONS]
  uint32_t* ctxmap_ws;    // [num_mb][max_lit_types * 64 + 1024]
  // quality >= 10: clustered context maps of the metablocks (bro_kernels_hq.cuh fills them)
  uint8_t* lit_cmap;      // [num_mb][256 * 64] literal (block type, context) -> prefix code
  uint8_t* dist_cmap;     // [num_mb][256 * 4]
  uint32_t* cm_counts;    // [num_mb][2] number of literal / distance prefix codes
  // output
  uint32_t* out;          // zero-initialised words
  uint64_t out_cap_bytes;
  uint64_t* total_bits;   // [1]
};

__device__ __forceinline__ SplitView make_view(const Workspace& W, uint32_t m, int cat) {
  SplitView v;
  const uint32_t* cnt = W.split_counts + (size_t)m * 6;
  if (cat == 0) {
    v.types = W.lit_types + (size_t)m * W.lit_blk_cap; v.lengths = W.lit_lengths + (size_t)m * W.lit_blk_cap;
    v.starts = W.lit_starts + (size_t)m * W.lit_blk_cap; v.num_blocks = cnt[0]; v.num_types = cnt[1];
  } else if (cat == 1) {
    v.types = W.cmd_types + (size_t)m * W.cmd_blk_cap; v.lengths = W.cmd_lengths + (size_t)m * W.cmd_blk_cap;
    v.starts = W.cmd_starts + (size_t)m * W.cmd_blk_cap; v.num_blocks = cnt[2]; v.num_types = cnt[3];
  } else {
    v.types = W.dist_types + (size_t)m * W.dist_blk_cap; v.lengths = W.dist_lengths + (size_t)m * W.dist_blk_cap;
    v.starts = W.dist_starts + (size_t)m * W.dist_blk_cap; v.num_blocks = cnt[4]; v.num_types = cnt[5];
  }
  return v;
}
__device__ __forceinline__ MetaCodes make_codes(const Workspace& W, uint32_t m) {
  MetaCodes mc;
  mc.lit = make_view(W, m, 0); mc.cmd = make_view(W, m, 1); mc.dist = make_view(W, m, 2);
  mc.lit_sc = W.split_codes + (size_t)m * 3; mc.cmd_sc = mc.lit_sc + 1; mc.dist_sc = mc.lit_sc + 2;
  mc.lit_depth = W.lit_depth + (size_t)m * W.max_lit_trees * 256; mc.lit_code = W.lit_code + (size_t)m * W.max_lit_trees * 256;
  mc.cmd_depth = W.cmd_depth + (size_t)m * W.max_cmd_types * 704; mc.cmd_code = W.cmd_code + (size_t)m * W.max_cmd_types * 704;
  mc.dist_depth = W.dist_depth + (size_t)m * W.max_dist_types * W.dist_A; mc.dist_code = W.dist_code + (size_t)m * W.max_dist_types * W.dist_A;
  mc.dist_A = W.dist_A;
  mc.ctx_map_id = W.mb[m].ctx_map_id;
  mc.nctx = ctxmap_num_contexts(mc.ctx_map_id);
  const bool full = mc.ctx_map_id >= CTXMAP_FULL_UTF8;  // quality >= 10: clustered context maps
  mc.lit_cmap = full ? W.lit_cmap + (size_t)m * 256 * 64 : nullptr;
  mc.dist_cmap = full ? W.dist_cmap + (size_t)m * 256 * 4 : nullptr;
  return mc;
}

// ---------------------------------------------------------------------------------------------------
// TMA bulk copies (sm_90+ `cp.async.bulk`, SASS UBLKCP): a contiguous tile travels global -> shared memory through the copy
// engine and signals an mbarrier with its byte count; no thread spends issue slots on LDG / STS pairs or address arithmetic.
// Addresses and sizes must be multiples of 16 bytes.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_addr_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr_u32(bar)), "r"(arrivals) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_addr_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "MBAR_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra MBAR_DONE;\n"
      "bra MBAR_WAIT;\n"
      "MBAR_DONE:\n"
      "}" ::"r"(smem_addr_u32(bar)),
      "r"(parity)
      : "memory");
}
// The whole CTA calls this: thread 0 arms the barrier and issues one bulk copy of `bytes` (multiple of 16, both addresses 16-byte
// aligned), everybody waits for the bytes to land.
__device__ __forceinline__ void tma_stage_tile(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  if (threadIdx.x == 0) mbar_init(bar, 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, bytes);
    tma_load_1d(smem_dst, gmem_src, bytes, bar);
  }
  mbar_wait(bar, 0);
}

// ---------------------------------------------------------------------------------------------------
// Radix sort of the positions of one batch by bucket key (stable => ascending position inside a bucket): a one-sweep LSD sort
// with two digits, key & 0xFF and then key >> 8 (7 bits for 15-bit keys, 6 for 14-bit ones).
//   k_sort_count     reads the input bytes once (TMA-staged tiles) and counts both digits over the whole batch; its last CTA turns
//                    the counts into each digit's base offset
//   k_sort_onesweep  one pass: ranks a tile's elements in shared memory, finds the tile's offset of every digit by a decoupled
//                    look-back over the tiles before it, and writes the tile out in digit order (runs of consecutive addresses)
// Pass 0 takes its keys from the staged input and writes the element word (key >> 8) << 25 | (position - batch_origin);
// pass 1 reads those words and writes plain batch-relative positions.
// ---------------------------------------------------------------------------------------------------
#define SORT_THREADS 256
#define SORT_ITEMS 16
#define SORT_TILE (SORT_THREADS * SORT_ITEMS)
// sort state of a lane (32-bit words), zeroed before every sort
#define SORT_ST_COUNT 0     // [2][256] digit counts of pass 0 / pass 1 over the batch
#define SORT_ST_BASE 512    // [2][256] first output index of each digit
#define SORT_ST_DONE 1024   // k_sort_count CTAs that have added their counts
#define SORT_ST_TILE 1025   // [2] next tile index of each pass
#define SORT_ST_SLAB 1032   // [BEST_MAX_SLABS] records claimed in each best[] slab by k_match_shallow in the batch (match_store)
#define SORT_ST_BTILE 1056  // [BEST_MAX_TILES] records claimed in each best[] tile by k_best_bin in the batch
#define SORT_ST_FLAGS 5152  // [2][num_tiles][256] look-back words: flag bits | count
#define SORT_LB_AGG (1u << 30)  // count of the digit in this tile alone
#define SORT_LB_INC (2u << 30)  // count of the digit in this tile and every tile before it
#define SORT_LB_VAL 0x3FFFFFFFu
__host__ __device__ constexpr size_t sort_state_words(uint32_t num_tiles) { return SORT_ST_FLAGS + (size_t)2 * num_tiles * 256; }

struct SortArgs {
  const uint8_t* data;   // data + batch_origin
  uint32_t count;        // positions in batch (halo + payload)
  const uint32_t* in;    // pass 1 input
  uint32_t* outw;        // pass output
  uint32_t* state;       // [sort_state_words(num_tiles)], zeroed
  uint32_t num_tiles;
  int hash_type, key_bits;
  int pass;
};

#define BRO_HASH_LEVEL0 100  // hash_type 100 + l: the long-prefix level l of quality 10 / 11 (bro_hq.cuh: 8, 16, 32 bytes)
template <bool LEVEL>
__device__ __forceinline__ uint32_t smem_key(const uint32_t* sw, uint32_t e, int hash_type, int key_bits) {
  // bytes e..e+7 of the tile staged as little-endian words
  const uint32_t sh = (e & 3u) * 8u;
  if (LEVEL) {
    const uint32_t* q = sw + (e >> 2);
    const uint64_t h = hq_level_hash_with([q, sh](uint32_t k) {
      const uint32_t w0 = q[k >> 2], w1 = q[(k >> 2) + 1], w2 = q[(k >> 2) + 2];
      return ((uint64_t)__funnelshift_r(w1, w2, sh) << 32) | __funnelshift_r(w0, w1, sh);
    }, hq_level_bytes(hash_type - BRO_HASH_LEVEL0));
    return hq_level_key(h, key_bits);
  }
  uint32_t w0 = sw[e >> 2], w1 = sw[(e >> 2) + 1], w2 = sw[(e >> 2) + 2];
  uint32_t lo = __funnelshift_r(w0, w1, sh);
  uint32_t hi = __funnelshift_r(w1, w2, sh);
  return hash_key_from_words(hash_type, key_bits, lo, hi);
}

// TMA bulk copy of tile `tile` (SORT_TILE + 48 bytes: the input is padded, so reading past `count` is safe; the batch origin is
// 4096-byte aligned) into sw; the whole CTA calls this and waits on phase `parity` of the (already initialised) barrier
__device__ __forceinline__ void sort_stage_tile(const SortArgs& a, uint32_t tile, uint32_t* sw, uint64_t* bar, uint32_t parity) {
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, SORT_TILE + 48);
    tma_load_1d(sw, a.data + (size_t)tile * SORT_TILE, SORT_TILE + 48, bar);
  }
  mbar_wait(bar, parity);
}

// exclusive prefix sum over the CTA's 256 threads (s_warp: 8 words of shared memory); all threads call it
__device__ __forceinline__ uint32_t block_excl_scan256(uint32_t v, uint32_t* s_warp) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= (uint32_t)o) x += y;
  }
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  uint32_t woff = 0;
  for (uint32_t w = 0; w < wid; ++w) woff += s_warp[w];
  return woff + x - v;
}

// Look-back words carry their own count, so nothing is read after them that their publication has to order; relaxed loads let
// SORT_LB_WINDOW of them be in flight at once (both passes of a 29 M-position batch on an H100 80GB HBM3 at 700 W: 587 µs, against
// 622 µs with one acquire load per step).
#define SORT_LB_WINDOW 8
__device__ __forceinline__ uint32_t ld_relaxed_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// grid-stride over the tiles; a.state zeroed
template <bool LEVEL>
__global__ void __launch_bounds__(SORT_THREADS) k_sort_count(SortArgs a) {
  __shared__ __align__(16) uint32_t sw[SORT_TILE / 4 + 12];
  __shared__ __align__(8) uint64_t s_bar;
  __shared__ uint32_t sh[2][256];
  __shared__ uint32_t s_warp[SORT_THREADS / 32];
  __shared__ bool s_last;
  const uint32_t tid = threadIdx.x;
  sh[0][tid] = 0;
  sh[1][tid] = 0;
  if (tid == 0) mbar_init(&s_bar, 1);
  __syncthreads();
  uint32_t parity = 0;
  for (uint32_t tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x, parity ^= 1u) {
    sort_stage_tile(a, tile, sw, &s_bar, parity);
    const uint32_t base = tile * SORT_TILE;
#pragma unroll 4
    for (int r = 0; r < SORT_ITEMS; ++r) {
      const uint32_t e = r * SORT_THREADS + tid;
      if (base + e < a.count) {
        const uint32_t key = smem_key<LEVEL>(sw, e, a.hash_type, a.key_bits);
        atomicAdd(&sh[0][key & 0xFFu], 1u);
        atomicAdd(&sh[1][key >> 8], 1u);
      }
    }
    __syncthreads();  // sw is read before the next tile's copy lands in it
  }
  if (sh[0][tid]) atomicAdd(&a.state[SORT_ST_COUNT + tid], sh[0][tid]);
  if (sh[1][tid]) atomicAdd(&a.state[SORT_ST_COUNT + 256 + tid], sh[1][tid]);
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(&a.state[SORT_ST_DONE], 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();  // every other CTA's counts are in
  for (int p = 0; p < 2; ++p) {
    const uint32_t c = __ldcg(&a.state[SORT_ST_COUNT + p * 256 + tid]);
    a.state[SORT_ST_BASE + p * 256 + tid] = block_excl_scan256(c, s_warp);
    __syncthreads();  // s_warp is reused
  }
}

// one pass; one tile per CTA, taken in order from the state's tile counter
template <bool LEVEL>
__global__ void __launch_bounds__(SORT_THREADS, 4) k_sort_onesweep(SortArgs a) {
  __shared__ __align__(16) uint32_t s_buf[SORT_TILE];  // pass 0: the staged input bytes; then the tile's words in digit order
  __shared__ uint8_t s_dig[SORT_TILE];                  // digit of each word of s_buf
  __shared__ uint32_t wc[SORT_THREADS / 32][256];       // per warp and digit: count, then the first slot of s_buf
  __shared__ uint32_t s_gofs[256];                      // per digit: output index minus slot
  __shared__ uint32_t s_warp[SORT_THREADS / 32];
  __shared__ uint32_t s_tile;
  __shared__ __align__(8) uint64_t s_bar;
  const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int nbits = a.pass == 0 ? 8 : a.key_bits - 8;
  for (uint32_t i = tid; i < (SORT_THREADS / 32) * 256; i += SORT_THREADS) (&wc[0][0])[i] = 0;
  if (tid == 0) {
    s_tile = atomicAdd(&a.state[SORT_ST_TILE + a.pass], 1u);
    if (a.pass == 0) mbar_init(&s_bar, 1);
  }
  __syncthreads();
  const uint32_t tile = s_tile;
  if (a.pass == 0) sort_stage_tile(a, tile, s_buf, &s_bar, 0);
  const uint32_t base = tile * SORT_TILE;
  uint32_t word[SORT_ITEMS];
  uint32_t rk[SORT_ITEMS];  // digit << 16 | rank among the warp's elements of that digit; ~0u past the end of the batch
  if (a.pass == 1) {  // all loads in flight before the ranking (its __syncwarp()s would keep them one round apart)
#pragma unroll
    for (int r = 0; r < SORT_ITEMS; ++r) {
      const uint32_t e = wid * (32 * SORT_ITEMS) + r * 32 + lane;
      word[r] = base + e < a.count ? a.in[base + e] : 0u;
    }
  }
  // element order inside the tile: warp-major, then round, then lane  (=> ascending position)
#pragma unroll
  for (int r = 0; r < SORT_ITEMS; ++r) {
    const uint32_t e = wid * (32 * SORT_ITEMS) + r * 32 + lane;
    const bool valid = base + e < a.count;
    uint32_t digit = 0x100u, w = 0;
    if (valid) {
      if (a.pass == 0) {
        const uint32_t key = smem_key<LEVEL>(s_buf, e, a.hash_type, a.key_bits);
        digit = key & 0xFFu;
        w = ((key >> 8) << 25) | (base + e);
      } else {
        const uint32_t v = word[r];
        digit = v >> 25;
        w = v & 0x1FFFFFFu;
      }
    }
    // lanes with the same digit, from 1 + nbits ballots (MATCH.ANY measured slower: it goes through the MIO queue)
    uint32_t peers = __ballot_sync(0xffffffffu, valid);
    if (!valid) peers = ~peers;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      if (b < nbits) {
        const bool bit = (digit >> b) & 1u;
        const uint32_t bal = __ballot_sync(0xffffffffu, bit);
        peers &= bit ? bal : ~bal;
      }
    }
    const uint32_t rank_in_round = __popc(peers & ((1u << lane) - 1u));
    uint32_t old = 0;
    if (valid) old = wc[wid][digit];
    __syncwarp();
    if (valid && rank_in_round == 0) wc[wid][digit] = old + __popc(peers);
    __syncwarp();
    word[r] = w;
    rk[r] = valid ? (digit << 16) | (old + rank_in_round) : ~0u;
  }
  __syncthreads();
  // per digit d: the tile's count, its first slot in the tile, and the first slot of each warp's elements
  const uint32_t d = tid;
  uint32_t agg = 0;
#pragma unroll
  for (int w = 0; w < SORT_THREADS / 32; ++w) agg += wc[w][d];
  const uint32_t first = block_excl_scan256(agg, s_warp);
  {
    uint32_t acc = first;
#pragma unroll
    for (int w = 0; w < SORT_THREADS / 32; ++w) {
      const uint32_t t = wc[w][d];
      wc[w][d] = acc;
      acc += t;
    }
  }
  if (d < (1u << nbits)) {  // decoupled look-back: this digit's count in the tiles before this one
    uint32_t* flags = a.state + SORT_ST_FLAGS + (size_t)a.pass * a.num_tiles * 256;
    uint32_t before = 0;
    if (tile == 0) {
      st_release_gpu(flags + d, SORT_LB_INC | agg);
    } else {
      st_release_gpu(flags + (size_t)tile * 256 + d, SORT_LB_AGG | agg);
      // Tiles are handed out in order by an atomic counter, so every tile before this one was claimed by a CTA that is already
      // running, and that CTA publishes its aggregate before it waits on anything.  Tile 0 publishes its inclusive count
      // without waiting.  So each word this loop waits on gets written, and the walk ends at tile 0 at the latest.
      uint32_t t = tile;  // tiles t - 1, t - 2, ... are still to be added
      bool done = false;
      while (!done) {
        uint32_t v[SORT_LB_WINDOW];
#pragma unroll
        for (uint32_t j = 0; j < SORT_LB_WINDOW; ++j) v[j] = j < t ? ld_relaxed_gpu(flags + (size_t)(t - 1 - j) * 256 + d) : 0u;
        uint32_t j = 0;
#pragma unroll
        for (; j < SORT_LB_WINDOW; ++j) {
          if (v[j] == 0) break;  // not published yet: read again from here
          before += v[j] & SORT_LB_VAL;
          if (v[j] & SORT_LB_INC) { done = true; break; }
        }
        t -= j;
      }
      st_release_gpu(flags + (size_t)tile * 256 + d, SORT_LB_INC | (before + agg));
    }
    s_gofs[d] = a.state[SORT_ST_BASE + a.pass * 256 + d] + before - first;
  }
  __syncthreads();  // (pass 0: every key is computed before s_buf is overwritten)
#pragma unroll
  for (int r = 0; r < SORT_ITEMS; ++r) {
    if (rk[r] != ~0u) {
      const uint32_t dg = rk[r] >> 16;
      const uint32_t slot = wc[wid][dg] + (rk[r] & 0xFFFFu);
      s_buf[slot] = word[r];
      s_dig[slot] = (uint8_t)dg;
    }
  }
  __syncthreads();
  const uint32_t n_tile = min((uint32_t)SORT_TILE, a.count - base);
  for (uint32_t i = tid; i < n_tile; i += SORT_THREADS) a.outw[s_gofs[s_dig[i]] + i] = s_buf[i];
}

// unaligned little-endian loads built from aligned words (the input has >= 512 readable bytes of padding)
__device__ __forceinline__ uint32_t ldu32(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
  const uint32_t sh = (uint32_t)(a & 3u) * 8u;
  uint32_t w0 = q[0];
  if (sh == 0) return w0;
  return __funnelshift_r(w0, q[1], sh);
}
__device__ __forceinline__ uint64_t ldu64(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
  const uint32_t sh = (uint32_t)(a & 3u) * 8u;
  uint32_t w0 = q[0], w1 = q[1], w2 = q[2];
  uint32_t lo = __funnelshift_r(w0, w1, sh), hi = __funnelshift_r(w1, w2, sh);
  return ((uint64_t)hi << 32) | lo;
}
// ---------------------------------------------------------------------------------------------------
// Match search over the sorted position list of one batch.
// ---------------------------------------------------------------------------------------------------
#ifndef MATCH_THREADS
#define MATCH_THREADS 256
#endif

struct MatchArgs {
  const uint8_t* data;      // whole input (padded)
  const uint32_t* sorted;   // [count] batch-relative positions sorted by (key, position)
  uint32_t count;
  uint32_t origin;          // absolute position of batch-relative 0
  uint32_t payload_begin;   // batch-relative first position whose match is wanted
  uint32_t n;               // input size
  uint32_t* best;
  int hash_type, key_bits, depth;
  uint32_t lcap, max_backward;
  DictView dict;            // static dictionary (device copies)
  int use_dict;
};

// best[] of a batch at depth 16 / 32 is written in three steps.  k_match_shallow's positions are in bucket order, so a direct best[p]
// store puts 4 bytes at a random address of the whole payload: every store is a write request of its own.  Instead the payload
// [b0, b1) is cut into slabs of 2^BEST_SLAB_BITS positions and those into tiles of 2^BEST_TILE_BITS positions, both counted from
// b0.  Every payload position yields exactly one record, so slab s receives exactly min(2^BEST_SLAB_BITS, b1 - b0 - (s <<
// BEST_SLAB_BITS)) records and owns that many 8-byte slots of `stage` from s << BEST_SLAB_BITS on, and tile t likewise owns its
// size's slots of the tile-major buffer from t << BEST_TILE_BITS on; no count has to be scanned first.
//   match_store   bins a CTA's records by slab, claims one run per slab with one atomic and writes the run (slab-major `stage`)
//   k_best_bin    reads BEST_BIN_SPAN records of one slab, reorders them by tile in shared memory, claims one run per tile and
//                 writes the runs (tile-major buffer; a run is about 32 records at 2^13-position tiles)
//   k_best_tile   reads one tile's records, places each value in a shared-memory image of the tile's best[] and writes the image
//                 with 16-byte stores
// Every global access of the last two is a coalesced stream.  The values placed are the ones a direct store writes; only the
// order of the records within a slab or a tile varies from run to run.
#define BEST_SLAB_BITS 21
#define BEST_MAX_SLABS 16                                  // kBatchMax >> BEST_SLAB_BITS
#define BEST_TILE_BITS 13                                  // a 32 KiB tile of best[]
#define BEST_MAX_TILES (1u << (25 - BEST_TILE_BITS))       // kBatchMax >> BEST_TILE_BITS
#define BEST_TILES_PER_SLAB (1u << (BEST_SLAB_BITS - BEST_TILE_BITS))
#define BEST_BIN_SPAN 8192                                 // records per k_best_bin CTA; divides a slab, so a span lies in one slab
#define BEST_BIN_THREADS 256
#define BEST_TILE_THREADS 256
static_assert(SORT_ST_SLAB + BEST_MAX_SLABS <= SORT_ST_BTILE, "slab cursors overlap the tile cursors");
static_assert(SORT_ST_BTILE + BEST_MAX_TILES <= SORT_ST_FLAGS, "tile cursors overlap the look-back words");
static_assert(((1u << BEST_SLAB_BITS) % BEST_BIN_SPAN) == 0 && BEST_BIN_SPAN % BEST_BIN_THREADS == 0, "a span crosses a slab");
static_assert(BEST_TILE_BITS <= BEST_SLAB_BITS && ((1u << BEST_TILE_BITS) % (4 * BEST_TILE_THREADS)) == 0, "tile shape");
struct BestStage {
  uint2* stage;           // [payload] (position, value) records, slab-major
  uint32_t* slab_cursor;  // [BEST_MAX_SLABS] records claimed per slab, zeroed with the sort state
};

// Called by every thread of the CTA (it synchronises the CTA); `active` threads store best[p] = v of payload position p.
__device__ __forceinline__ void match_store(const MatchArgs& a, const BestStage& st, bool active, uint32_t p, uint32_t v) {
  static_assert(MATCH_THREADS >= BEST_MAX_SLABS, "one thread per slab claims the runs");
  __shared__ uint32_t s_cnt[BEST_MAX_SLABS], s_run[BEST_MAX_SLABS];
  const uint32_t tid = threadIdx.x, lane = tid & 31u;
  if (tid < BEST_MAX_SLABS) s_cnt[tid] = 0;
  __syncthreads();
  const uint32_t slab = active ? (p - (a.origin + a.payload_begin)) >> BEST_SLAB_BITS : BEST_MAX_SLABS;
  // lanes of one slab take consecutive ranks of the CTA's run with one shared atomic per warp and slab
  const uint32_t peers = __match_any_sync(0xffffffffu, slab);
  const uint32_t leader = (uint32_t)__ffs((int)peers) - 1u;
  uint32_t first = 0;
  if (active && lane == leader) first = atomicAdd(&s_cnt[slab], (uint32_t)__popc(peers));
  const uint32_t rank = __shfl_sync(0xffffffffu, first, leader) + (uint32_t)__popc(peers & ((1u << lane) - 1u));
  __syncthreads();
  if (tid < BEST_MAX_SLABS && s_cnt[tid]) s_run[tid] = atomicAdd(&st.slab_cursor[tid], s_cnt[tid]);
  __syncthreads();
  if (active) st.stage[((size_t)slab << BEST_SLAB_BITS) + s_run[slab] + rank] = make_uint2(p, v);
}

// slab-major `stage` -> tile-major `tiles` for the `payload` records of the batch whose payload starts at absolute position b0;
// one CTA per span of BEST_BIN_SPAN records, dynamic shared memory BEST_BIN_SPAN records, tile_cursor zeroed with the sort state
__global__ void __launch_bounds__(BEST_BIN_THREADS, 2) k_best_bin(const uint2* __restrict__ stage, uint32_t payload, uint32_t b0,
                                                                 uint2* __restrict__ tiles, uint32_t* __restrict__ tile_cursor) {
  constexpr uint32_t ITEMS = BEST_BIN_SPAN / BEST_BIN_THREADS;
  constexpr uint32_t TPS = BEST_TILES_PER_SLAB;
  constexpr uint32_t TPT = (TPS + BEST_BIN_THREADS - 1) / BEST_BIN_THREADS;  // tiles per thread in the scan
  extern __shared__ uint2 s_rec[];                                             // [BEST_BIN_SPAN] the span in tile order
  __shared__ uint32_t s_cnt[TPS], s_off[TPS], s_run[TPS];
  __shared__ uint32_t s_warp[BEST_BIN_THREADS / 32];
  const uint32_t tid = threadIdx.x;
  const uint32_t k0 = blockIdx.x * BEST_BIN_SPAN;
  const uint32_t nk = min((uint32_t)BEST_BIN_SPAN, payload - k0);
  for (uint32_t t = tid; t < TPS; t += BEST_BIN_THREADS) s_cnt[t] = 0;
  uint2 r[ITEMS];
#pragma unroll
  for (uint32_t j = 0; j < ITEMS; ++j) {
    const uint32_t k = j * BEST_BIN_THREADS + tid;
    r[j] = k < nk ? __ldcs(&stage[k0 + k]) : make_uint2(0u, 0u);  // read once
  }
  __syncthreads();
  // rank of each record among the span's records of its tile
  uint32_t rank[ITEMS];
#pragma unroll
  for (uint32_t j = 0; j < ITEMS; ++j)
    if (j * BEST_BIN_THREADS + tid < nk) rank[j] = atomicAdd(&s_cnt[((r[j].x - b0) >> BEST_TILE_BITS) & (TPS - 1)], 1u);
  __syncthreads();
  // each tile's first slot in s_rec, and its run in the tile-major buffer
  uint32_t c[TPT], sum = 0;
#pragma unroll
  for (uint32_t q = 0; q < TPT; ++q) {
    const uint32_t t = tid * TPT + q;
    c[q] = t < TPS ? s_cnt[t] : 0u;
    sum += c[q];
  }
  uint32_t off = block_excl_scan256(sum, s_warp);
  const uint32_t tile0 = (k0 >> BEST_SLAB_BITS) * TPS;  // the slab's first tile
#pragma unroll
  for (uint32_t q = 0; q < TPT; ++q) {
    const uint32_t t = tid * TPT + q;
    if (t < TPS) {
      s_off[t] = off;
      if (c[q]) s_run[t] = atomicAdd(&tile_cursor[tile0 + t], c[q]);
      off += c[q];
    }
  }
  __syncthreads();
#pragma unroll
  for (uint32_t j = 0; j < ITEMS; ++j)
    if (j * BEST_BIN_THREADS + tid < nk) s_rec[s_off[((r[j].x - b0) >> BEST_TILE_BITS) & (TPS - 1)] + rank[j]] = r[j];
  __syncthreads();
  // one run per tile, consecutive threads on consecutive slots
  for (uint32_t i = tid; i < nk; i += BEST_BIN_THREADS) {
    const uint2 rec = s_rec[i];
    const uint32_t g = (rec.x - b0) >> BEST_TILE_BITS, t = g & (TPS - 1);
    tiles[((size_t)g << BEST_TILE_BITS) + s_run[t] + (i - s_off[t])] = rec;
  }
}

// tile-major `tiles` -> best[pos] = value (best indexed by absolute position; best + b0 is 16-byte aligned); one CTA per tile
__global__ void __launch_bounds__(BEST_TILE_THREADS) k_best_tile(const uint2* __restrict__ tiles, uint32_t payload, uint32_t b0,
                                                                 uint32_t* __restrict__ best) {
  constexpr uint32_t TILE = 1u << BEST_TILE_BITS, ITEMS = TILE / BEST_TILE_THREADS;
  __shared__ __align__(16) uint32_t s_img[TILE];
  const uint32_t tid = threadIdx.x;
  const uint32_t base = blockIdx.x << BEST_TILE_BITS;  // payload-relative first position of the tile
  const uint32_t m = min(TILE, payload - base);
  const uint2* rec = tiles + base;
  uint2 r[ITEMS];
#pragma unroll
  for (uint32_t j = 0; j < ITEMS; ++j) {
    const uint32_t i = j * BEST_TILE_THREADS + tid;
    if (i < m) r[j] = __ldcs(&rec[i]);  // read once
  }
  const uint32_t pos0 = b0 + base;
#pragma unroll
  for (uint32_t j = 0; j < ITEMS; ++j)
    if (j * BEST_TILE_THREADS + tid < m) s_img[r[j].x - pos0] = r[j].y;
  __syncthreads();
  uint4* d4 = reinterpret_cast<uint4*>(best + pos0);
  const uint4* s4 = reinterpret_cast<const uint4*>(s_img);
  for (uint32_t i = tid; i < m / 4; i += BEST_TILE_THREADS) d4[i] = s4[i];
  for (uint32_t i = (m & ~3u) + tid; i < m; i += BEST_TILE_THREADS) best[pos0 + i] = s_img[i];
}

// dict_candidate() of bro_dict.cuh with the position's first 16 bytes already in registers and 8-byte word compares
__device__ __forceinline__ uint32_t dict_candidate_dev(const DictView& D, int hash_type, uint32_t m0, uint32_t m1, uint32_t m2,
                                                       uint32_t m3, const uint8_t* cur, uint32_t max_len, uint32_t mb) {
  uint32_t best = 0, best_score = BRO_MIN_SCORE;
  const uint32_t key = dict_hash14(m0) << 1;
#pragma unroll
  for (uint32_t s = 0; s < 2; ++s) {
    const uint32_t item = D.hash[key + s];
    const uint32_t wl = item & 31u, idx = item >> 5;
    if (item == 0 || wl > max_len) continue;
    const uint8_t* w = D.words + dict_offset(wl) + wl * idx;
    uint64_t x = ldu64(w) ^ (((uint64_t)m1 << 32) | m0);
    if ((uint32_t)x != 0) continue;  // hash collision
    uint32_t ml = x ? ((uint32_t)(__ffsll((long long)x) - 1) >> 3) : 8u;
    if (ml == 8u && wl > 8u) {
      x = ldu64(w + 8) ^ (((uint64_t)m3 << 32) | m2);
      ml += x ? ((uint32_t)(__ffsll((long long)x) - 1) >> 3) : 8u;
      if (ml == 16u && wl > 16u) {
        x = ldu64(w + 16) ^ ldu64(cur + 16);
        ml += x ? ((uint32_t)(__ffsll((long long)x) - 1) >> 3) : 8u;
      }
    }
    ml = bmin(ml, wl);
    if (ml + 10u <= wl) continue;
    const uint32_t word_id = idx + (dict_omit_last_transform(wl - ml) << dict_size_bits(wl));
    const uint32_t score = score_regular(hash_type, ml, mb + 1u + word_id);
    if (score < best_score) continue;
    best = best_pack_dict(ml, wl, idx);
    best_score = score;
  }
  return best;
}

__device__ __forceinline__ void load16_unaligned(const uint8_t* p, uint32_t* w) {
  const uint32_t* q = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(p) & ~(uintptr_t)3);
  uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u) * 8u;
  uint32_t a0 = __ldg(q), a1 = __ldg(q + 1), a2 = __ldg(q + 2), a3 = __ldg(q + 3), a4 = __ldg(q + 4);
  w[0] = __funnelshift_r(a0, a1, sh);
  w[1] = __funnelshift_r(a1, a2, sh);
  w[2] = __funnelshift_r(a2, a3, sh);
  w[3] = __funnelshift_r(a3, a4, sh);
}

// Sorted positions of a CTA's entries [j0, j0 + E) -> s_pos: interior CTAs take them with one TMA bulk copy (j0 * 4 and E * 4 are
// multiples of 16), the first / last CTA of a batch with guarded loads (0xFFFFFFFF = no entry).  Ends with a CTA barrier.
__device__ __forceinline__ void match_stage_positions(const MatchArgs& a, int64_t j0, uint32_t E, uint32_t* s_pos, uint64_t* bar) {
  if (j0 >= 0 && j0 + (int64_t)E <= (int64_t)a.count) {
    tma_stage_tile(s_pos, a.sorted + j0, E * 4u, bar);
  } else {
    for (uint32_t i = threadIdx.x; i < E; i += MATCH_THREADS) {
      const int64_t j = j0 + i;
      s_pos[i] = (j >= 0 && j < (int64_t)a.count) ? a.sorted[j] : 0xFFFFFFFFu;
    }
  }
  __syncthreads();
}

// dynamic shared memory: (MATCH_THREADS + depth) entries x 6 words.
// Shallow buckets (depth 16 / 32: q5, q6) -- the bench path.  In a loop version most of the warp instructions were the
// divergent per-survivor loop.  Here every candidate
// whose match is shorter than 8 bytes -- the bulk on text -- is resolved branch-free inside the unrolled scan (its length
// comes from one XOR of the second data word), and only candidates that agree on all 8 bytes go through the exact
// (divergent) evaluation.  Result identical to the sequential newest-first walk: highest score, nearest on ties.
template <int DEPTH>
__global__ void __launch_bounds__(MATCH_THREADS) k_match_shallow(MatchArgs a, BestStage st) {
  extern __shared__ __align__(16) uint32_t smem[];
  constexpr uint32_t E = MATCH_THREADS + (uint32_t)DEPTH;
  uint32_t* s_pos = smem;
  uint32_t* s_key = smem + E;
  uint32_t* s_d0 = smem + 2 * E;
  uint32_t* s_d1 = smem + 3 * E;
  uint32_t* s_d2 = smem + 4 * E;
  uint32_t* s_d3 = smem + 5 * E;
  const int64_t j0 = (int64_t)blockIdx.x * MATCH_THREADS - DEPTH;
  __shared__ __align__(8) uint64_t s_bar;
  match_stage_positions(a, j0, E, s_pos, &s_bar);
  for (uint32_t i = threadIdx.x; i < E; i += MATCH_THREADS) {
    const uint32_t pos = s_pos[i];
    uint32_t key = 0xFFFFFFFFu, w[4] = {0, 0, 0, 0};
    if (pos != 0xFFFFFFFFu) {
      load16_unaligned(a.data + a.origin + pos, w);
      key = hash_key_from_words(a.hash_type, a.key_bits, w[0], w[1]);
    }
    s_key[i] = key; s_d0[i] = w[0]; s_d1[i] = w[1]; s_d2[i] = w[2]; s_d3[i] = w[3];
  }
  __syncthreads();
  const uint32_t i = threadIdx.x + (uint32_t)DEPTH;
  const uint32_t prel = s_pos[i];
  const bool active = !(prel == 0xFFFFFFFFu || prel < a.payload_begin);  // inactive threads only take part in match_store
  const uint32_t p = a.origin + (active ? prel : 0u);
  const uint32_t maxl = bmin(a.lcap, a.n - p);
  uint32_t best_score = BRO_MIN_SCORE, best_len = 0, best_dist = 0;
  if (active && a.n - p >= 8) {  // keys of the last 7 positions would depend on bytes past the range: they get no bucket match
    const uint32_t key = s_key[i];
    const uint32_t max_backward = bmin(p, a.max_backward);
    const uint32_t m0 = s_d0[i], m1 = s_d1[i], m2 = s_d2[i], m3 = s_d3[i];
    for (uint32_t cbase = 0; cbase < (uint32_t)DEPTH; cbase += 16) {
      uint32_t mask8 = 0;
#pragma unroll
      for (uint32_t c = 0; c < 16; ++c) {
        const uint32_t ci = i - 1u - cbase - c;
        const uint32_t backward = prel - s_pos[ci];
        const uint32_t x1 = s_d1[ci] ^ m1;
        const bool ok = (s_key[ci] == key) & (s_d0[ci] == m0) & (backward <= max_backward);
        mask8 |= (uint32_t)(ok & (x1 == 0u)) << c;
        const uint32_t len = 4u + ((uint32_t)(__ffs((int)x1) - 1) >> 3);  // 4..7 when x1 != 0
        const uint32_t score = score_regular(5, len, backward | 1u);      // H5 / H6 share the score; |1 keeps log2 defined
        const bool better = ok & (x1 != 0u) & (score > best_score);
        best_score = better ? score : best_score;
        best_len = better ? len : best_len;
        best_dist = better ? backward : best_dist;
      }
      // candidates that agree on 8 bytes: exact length, nearest first
      while (mask8) {
        const uint32_t c = (uint32_t)__ffs((int)mask8) - 1u;
        mask8 &= mask8 - 1u;
        const uint32_t ci = i - 1u - cbase - c;
        const uint32_t backward = prel - s_pos[ci];
        uint32_t len;
        uint32_t x = s_d2[ci] ^ m2;
        if (x) len = 8 + ((uint32_t)(__ffs((int)x) - 1) >> 3);
        else {
          x = s_d3[ci] ^ m3;
          if (x) len = 12 + ((uint32_t)(__ffs((int)x) - 1) >> 3);
          else {
            len = 16;
            const uint8_t* pa = a.data + p;
            const uint8_t* pb = pa - backward;
            while (len + 8 <= maxl) {
              const uint64_t y = ldu64(pa + len) ^ ldu64(pb + len);
              if (y) { len += (uint32_t)(__ffsll((long long)y) - 1) >> 3; break; }
              len += 8;
            }
            if (len + 8 > maxl) while (len < maxl && pa[len] == pb[len]) ++len;
          }
        }
        if (len > maxl) len = maxl;
        const uint32_t score = score_regular(5, len, backward);
        if (score > best_score || (score == best_score && backward < best_dist)) { best_score = score; best_len = len; best_dist = backward; }
        if (len == maxl) break;  // nothing farther in this group can be better
      }
      if (best_len == maxl) break;  // nor in an older group
      if (s_key[i - 16u - cbase] != key) break;  // the bucket ended inside this group
    }
  }
  uint32_t outv = best_len ? ((best_dist << 8) | best_len) : 0u;
  if (active && best_len == 0 && a.use_dict && a.n - p >= 8)  // nothing in the bucket: static dictionary (mod.rs:1797, :1942)
    outv = dict_candidate_dev(a.dict, a.hash_type, s_d0[i], s_d1[i], s_d2[i], s_d3[i], a.data + p, a.n - p, bmin(p, a.max_backward));
  match_store(a, st, active, p, outv);
}

// Candidate key of the deep searches: score << 16 | (IMAX - candidate index) << LB | len, so that a maximum is "highest score,
// nearest on ties".  Scores stay below 2^16.  Up to 256 candidates the index takes 8 bits and the length 8; a 512-deep bucket
// (quality 11 with Q9_5) takes a 9-bit index and leaves 7 bits to the length, which the match cap (lcap = 64) fits.
template <int DEPTH>
struct DeepKey {
  static_assert(DEPTH <= 512, "candidate index wider than 9 bits");
  static constexpr uint32_t LB = DEPTH > 256 ? 7u : 8u;
  static constexpr uint32_t IMAX = (1u << (16u - LB)) - 1u;
  static constexpr uint32_t LMASK = (1u << LB) - 1u;
  static __device__ __forceinline__ uint32_t make(uint32_t score, uint32_t idx, uint32_t len) { return (score << 16) | ((IMAX - idx) << LB) | len; }
  static __device__ __forceinline__ uint32_t index(uint32_t k) { return IMAX - ((k >> LB) & IMAX); }
};

// Deep buckets (depth 64..512: q7..q9, lgwin <= 16 and quality 11 with Q9_5).  With one position per lane the survivors of the
// 4-byte filter are evaluated by a few active lanes on average, so here the (position,
// candidate) pairs of a whole warp are compacted and evaluated 32 at a time; results meet in a per-position atomicMax on
// DeepKey.  "Highest score, nearest on ties" is exactly what the sequential
// newest-first walk with strict improvement computes.  The "must be strictly longer" pre-filter uses the best of the
// *previous* groups only (all nearer), which keeps it exact.
template <int DEPTH>
__global__ void __launch_bounds__(MATCH_THREADS) k_match_deep(MatchArgs a) {
  using K = DeepKey<DEPTH>;
  extern __shared__ __align__(16) uint32_t smem[];
  constexpr uint32_t E = MATCH_THREADS + (uint32_t)DEPTH;
  uint32_t* s_pos = smem;
  uint32_t* s_key = smem + E;
  uint32_t* s_d0 = smem + 2 * E;
  uint32_t* s_d1 = smem + 3 * E;
  uint32_t* s_d2 = smem + 4 * E;
  uint32_t* s_d3 = smem + 5 * E;
  __shared__ uint16_t s_pairs[MATCH_THREADS / 32][512];
  __shared__ uint32_t s_bestk[MATCH_THREADS / 32][32];
  __shared__ uint32_t s_snap[MATCH_THREADS / 32][32];  // best length of the previous groups
  __shared__ uint32_t s_far[MATCH_THREADS / 32];
  const int64_t j0 = (int64_t)blockIdx.x * MATCH_THREADS - DEPTH;
  __shared__ __align__(8) uint64_t s_bar;
  match_stage_positions(a, j0, E, s_pos, &s_bar);
  for (uint32_t i = threadIdx.x; i < E; i += MATCH_THREADS) {
    const uint32_t pos = s_pos[i];
    uint32_t key = 0xFFFFFFFFu, w[4] = {0, 0, 0, 0};
    if (pos != 0xFFFFFFFFu) {
      load16_unaligned(a.data + a.origin + pos, w);
      key = hash_key_from_words(a.hash_type, a.key_bits, w[0], w[1]);
    }
    s_key[i] = key; s_d0[i] = w[0]; s_d1[i] = w[1]; s_d2[i] = w[2]; s_d3[i] = w[3];
  }
  __syncthreads();
  const uint32_t FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t i = threadIdx.x + (uint32_t)DEPTH;
  const uint32_t prel = s_pos[i];
  const bool active = !(prel == 0xFFFFFFFFu || prel < a.payload_begin);
  const uint32_t p = a.origin + (active ? prel : 0u);
  const uint32_t maxl = active ? bmin(a.lcap, a.n - p) : 0u;
  const uint32_t kNone = (BRO_MIN_SCORE << 16) | 0xFFFFu;
  s_bestk[wid][lane] = kNone;
  s_snap[wid][lane] = 0;
  if (lane == 0) s_far[wid] = 0;
  __syncwarp();
  const uint32_t key = s_key[i], m0 = s_d0[i];
  bool done = !active || a.n - p < 8;
  const uint32_t wbase = wid * 32u + (uint32_t)DEPTH;  // smem index of lane 0's entry
  for (uint32_t cbase = 0; cbase < (uint32_t)DEPTH; cbase += 16) {
    if (!__any_sync(FULL, !done)) break;
    uint32_t mask = 0;
    if (!done) {
      const uint32_t bl = s_snap[wid][lane];
      if (bl >= 4 && bl < 16) {
        const uint32_t wsel = (2u + (bl >> 2)) * E, sh = (bl & 3u) * 8u;
        const uint32_t mw = smem[wsel + i];
#pragma unroll
        for (uint32_t c = 0; c < 16; ++c) {
          const uint32_t ci = i - 1u - cbase - c;
          mask |= (uint32_t)((s_key[ci] == key) & (s_d0[ci] == m0) & ((((smem[wsel + ci] ^ mw) >> sh) & 0xFFu) == 0u)) << c;
        }
      } else {
#pragma unroll
        for (uint32_t c = 0; c < 16; ++c) {
          const uint32_t ci = i - 1u - cbase - c;
          mask |= (uint32_t)((s_key[ci] == key) & (s_d0[ci] == m0)) << c;
        }
      }
      if (s_key[i - 16u - cbase] != key) done = true;  // the bucket ends inside this group
    }
    // compact the (lane, candidate) pairs of the warp
    const uint32_t cnt = __popc(mask);
    uint32_t incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(FULL, incl, o);
      if (lane >= (uint32_t)o) incl += y;
    }
    const uint32_t total = __shfl_sync(FULL, incl, 31);
    {
      uint32_t off = incl - cnt, mm = mask;
      while (mm) {
        const uint32_t c = (uint32_t)__ffs((int)mm) - 1u;
        mm &= mm - 1u;
        s_pairs[wid][off++] = (uint16_t)((lane << 4) | c);
      }
    }
    __syncwarp();
    for (uint32_t k = lane; k < total; k += 32) {
      const uint32_t pr = s_pairs[wid][k];
      const uint32_t ln = pr >> 4, c = pr & 15u;
      const uint32_t ie = wbase + ln;
      const uint32_t ci = ie - 1u - cbase - c;
      const uint32_t eprel = s_pos[ie];
      const uint32_t ep = a.origin + eprel;
      const uint32_t emaxl = bmin(a.lcap, a.n - ep);
      const uint32_t backward = eprel - s_pos[ci];
      if (backward > bmin(ep, a.max_backward)) { atomicOr(&s_far[wid], 1u << ln); continue; }
      const uint32_t bl = s_snap[wid][ln];
      if (bl >= 16 && bl < emaxl && a.data[ep + bl] != a.data[ep - backward + bl]) continue;  // cannot be strictly longer
      uint32_t len;
      uint32_t x = s_d1[ci] ^ s_d1[ie];
      if (x) len = 4 + ((uint32_t)(__ffs((int)x) - 1) >> 3);
      else {
        x = s_d2[ci] ^ s_d2[ie];
        if (x) len = 8 + ((uint32_t)(__ffs((int)x) - 1) >> 3);
        else {
          x = s_d3[ci] ^ s_d3[ie];
          if (x) len = 12 + ((uint32_t)(__ffs((int)x) - 1) >> 3);
          else {
            len = 16;
            const uint8_t* pa = a.data + ep;
            const uint8_t* pb = pa - backward;
            while (len + 8 <= emaxl) {
              const uint64_t y = ldu64(pa + len) ^ ldu64(pb + len);
              if (y) { len += (uint32_t)(__ffsll((long long)y) - 1) >> 3; break; }
              len += 8;
            }
            if (len + 8 > emaxl) while (len < emaxl && pa[len] == pb[len]) ++len;
          }
        }
      }
      if (len > emaxl) len = emaxl;
      const uint32_t score = score_regular(a.hash_type, len, backward);
      atomicMax(&s_bestk[wid][ln], K::make(score, cbase + c, len));
    }
    __syncwarp();
    if (!done) {
      const uint32_t bk = s_bestk[wid][lane];
      if (bk != kNone) {
        s_snap[wid][lane] = bk & K::LMASK;
        if ((bk & K::LMASK) == maxl) done = true;  // a full-length match: nothing farther can beat it
      }
      if ((s_far[wid] >> lane) & 1u) done = true;  // candidates beyond the window: all older ones too
    }
    __syncwarp();
  }
  if (active) {
    const uint32_t bk = s_bestk[wid][lane];
    uint32_t r = 0;
    if (bk != kNone) {
      const uint32_t cc = K::index(bk);
      r = ((prel - s_pos[i - 1u - cc]) << 8) | (bk & K::LMASK);
    } else if (a.use_dict && a.n - p >= 8) {
      r = dict_candidate_dev(a.dict, a.hash_type, s_d0[i], s_d1[i], s_d2[i], s_d3[i], a.data + p, a.n - p, bmin(p, a.max_backward));
    }
    a.best[p] = r;  // (a long kernel: the scattered store drains under its work, where staging it costs more than it saves)
  }
}

// ---------------------------------------------------------------------------------------------------
// Parse: one thread per unit.
// ---------------------------------------------------------------------------------------------------
#define PARSE_WARPS 4

// exact common-prefix length of cur[..] and (cur - back)[..], known to be >= start, capped at max_len (whole warp)
__device__ __forceinline__ uint32_t warp_lcp_ext(const uint8_t* cur, uint32_t back, uint32_t start, uint32_t max_len) {
  const uint32_t lane = threadIdx.x & 31;
  for (uint32_t off = start; off < max_len; off += 128) {
    const uint32_t o = off + 4 * lane;
    const bool in = o < max_len;
    uint32_t nbytes = 0;
    if (in) {
      uint32_t x = ldu32(cur + o) ^ ldu32(cur - back + o);
      nbytes = x ? ((uint32_t)(__ffs((int)x) - 1) >> 3) : 4u;
      nbytes = bmin(nbytes, max_len - o);
    }
    const bool full = in && nbytes == 4 && (o + 4 <= max_len);
    const uint32_t stop = __ballot_sync(0xffffffffu, !full);
    if (stop) {
      const int first = __ffs((int)stop) - 1;
      const uint32_t nb = __shfl_sync(0xffffffffu, nbytes, first);
      return bmin(off + 4u * (uint32_t)first + nb, max_len);
    }
  }
  return max_len;
}

// lane-local exact common-prefix length (>= start), used for the rare candidates that match the whole probe width
__device__ __forceinline__ uint32_t lane_lcp_ext(const uint8_t* cur, uint32_t back, uint32_t start, uint32_t max_len) {
  while (start + 8 <= max_len) {
    const uint64_t x = ldu64(cur + start) ^ ldu64(cur - back + start);
    if (x) return start + ((uint32_t)(__ffsll((long long)x) - 1) >> 3);
    start += 8;
  }
  while (start < max_len && cur[start] == (cur - back)[start]) ++start;
  return start;
}

// One parse unit per warp for NL = n_last = 10 / 16 (q7..q9, incl. the H9 scores): all 8 positions of a window are resolved
// completely in parallel -- each of the 4 lanes of a position probes the cached distances i = lane, lane + 4, ..., and the
// position's winner is the maximum of last_distance_key (2 shuffle-max steps) -- and the serial greedy / lazy walk only reads
// finished (found, len, dist, score) tuples: ballots locate the next match, shuffles fetch it.
template <int NL>
__device__ __forceinline__ uint32_t parse_unit_warp4(const EncParams& P, const uint8_t* data, const uint32_t* best,
                                                     uint32_t ustart, uint32_t uend, RawCmd* out, uint32_t* tail,
                                                     uint32_t* ncopy, bool D, int32_t* dc) {
  constexpr int G = 8;
  constexpr int K = (NL + 3) / 4;  // candidates per lane
  const int ht = P.hash_type;
  constexpr uint32_t CAPA = 8;
  const uint32_t FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t j_lane = lane >> 2, i_lane = lane & 3;
  int32_t dc0 = dc[0], dc1 = dc[1], dc2 = dc[2], dc3 = dc[3];
  const uint32_t htl = P.hash_type == 6 ? 8u : 4u;
  const uint32_t window = P.quality < 9 ? 64u : 512u;
  uint32_t pos = ustart, insert_len = 0, ncmd = 0, copied = 0;
  uint32_t arh = pos + window;
  bool have_m = false;
  uint32_t m_len = 0, m_dist = 0, m_score = 0;
  int delayed = 0;
  const bool near_start = P.abs_base < P.max_backward;

  while (have_m || pos + htl < uend) {
    // ---------------- phase A: every position of the window fully resolved, in parallel ----------------
    const uint32_t wbase = pos;
    const uint32_t p = wbase + j_lane;
    const bool p_ok = p < uend;
    const uint32_t maxl = p_ok ? uend - p : 0u;
    uint32_t key = 0;
    const int32_t dca[4] = {dc0, dc1, dc2, dc3};
    if (p_ok) {
      const uint32_t mb = near_start ? bmin(p + P.abs_base, P.max_backward) : P.max_backward;
      const uint64_t cw = ldu64(data + p);
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int i = (int)i_lane + 4 * k;
        if (i < NL) {
          const int32_t back = cache_candidate(dca, i);
          if (back > 0 && (uint32_t)back <= mb) {
            const uint64_t x = cw ^ ldu64(data + p - back);
            uint32_t len = x ? ((uint32_t)(__ffsll((long long)x) - 1) >> 3) : CAPA;
            len = bmin(len, maxl);
            if (len == CAPA && maxl > CAPA) len = lane_lcp_ext(data + p, (uint32_t)back, CAPA, maxl);
            if (len >= 3 || (len == 2 && i < 2)) key = max(key, last_distance_key(ht, len, maxl, (uint32_t)i));
          }
        }
      }
    }
    key = max(key, __shfl_xor_sync(FULL, key, 1));
    key = max(key, __shfl_xor_sync(FULL, key, 2));
    Match f;  // every lane of the position decodes the winner
    f.len = 0; f.dist = 0; f.score = BRO_MIN_SCORE;
    if (key) {
      const uint32_t wi = last_distance_key_decode(key, &f.len);
      f.dist = (uint32_t)cache_candidate(dca, (int)wi);
      f.score = score_last_distance(ht, f.len, wi);
    }
    bool f_found = key != 0;
    if (p_ok && i_lane == 0)  // then the bucket candidate of the match kernel
      f_found = take_best_candidate(best[p], ht, P.lcap, data + p, maxl, near_start ? bmin(p + P.abs_base, P.max_backward) : P.max_backward, D,
                                    lane_lcp_ext, f_found, &f);
    const uint32_t f_len = f.len, f_dist = f.dist, f_score = f.score;
    // lane 4*j now holds the finished result of position wbase + j
    uint32_t found8 = __ballot_sync(FULL, f_found && i_lane == 0);  // bits 0,4,8,.. -> compress to bits 0..7
    found8 = (found8 | (found8 >> 3)) & 0x03030303u;
    found8 = (found8 | (found8 >> 6)) & 0x000F000Fu;
    found8 = (found8 | (found8 >> 12)) & 0xFFu;  // bit j <=> a match exists at wbase + j

    // ---------------- phase B: serial greedy / lazy walk over finished results (warp-uniform scalars) ----------------
    int j = 0;
    for (;;) {
      if (!have_m) {
        if (!(pos + htl < uend) || j >= G) break;
        // searchable positions of this window from j on: wbase + j' + htl < uend
        const uint32_t lim = bmin((uint32_t)G, uend - htl - wbase);  // positions j' < lim are searchable (pos + htl < uend holds)
        const uint32_t cand = found8 & ~((1u << j) - 1u) & ((lim >= 32 ? 0xFFFFFFFFu : ((1u << lim) - 1u)));
        const uint32_t f = cand ? (uint32_t)(__ffs((int)cand) - 1) : lim;  // first match, or end of searchable range
        // literal steps j .. f-1, but the sparse-search heuristic may cut the run short
        const uint32_t run = f - (uint32_t)j;
        uint32_t steps = run;
        bool jump = false;
        if (run > 0 && pos + run > arh) {  // some step k (1..run) has pos + k > arh: the first such k triggers the skip
          steps = pos > arh ? 1u : (arh - pos + 1u);
          jump = true;
        }
        insert_len += steps;
        pos += steps;
        j += (int)steps;
        if (jump) {
          const uint32_t margin = bmax(htl - 1u, 4u);
          if (pos + 16 + margin >= uend) { insert_len += uend - pos; pos = uend; }
          else if (pos > arh + 4 * window) { insert_len += 16; pos += 16; }
          else { insert_len += 8; pos += 8; }
          break;
        }
        if (!cand || j >= G) break;  // window exhausted without a match
        const int src = 4 * j;
        m_len = __shfl_sync(FULL, f_len, src);
        m_dist = __shfl_sync(FULL, f_dist, src);
        m_score = __shfl_sync(FULL, f_score, src);
        have_m = true;
        delayed = 0;
      }
      // a match is pending at pos: lazy evaluation against pos + 1
      if (j + 1 >= G) break;  // re-probe with the window starting at pos
      {
        const int src = 4 * (j + 1);
        const bool f2 = (found8 >> (j + 1)) & 1u;
        const uint32_t s2 = __shfl_sync(FULL, f_score, src);
        if (f2 && s2 >= m_score + 175u) {
          pos++;
          insert_len++;
          j++;
          m_len = __shfl_sync(FULL, f_len, src);
          m_dist = __shfl_sync(FULL, f_dist, src);
          m_score = s2;
          if (++delayed < 4 && pos + htl < uend) continue;
        }
      }
      const uint32_t m_bytes = len_bytes(m_len);
      arh = pos + 2 * m_bytes + window;
      if (!len_is_dict(m_len) && (int32_t)m_dist != dc0) { dc3 = dc2; dc2 = dc1; dc1 = dc0; dc0 = (int32_t)m_dist; }
      if (out && lane < 3) reinterpret_cast<uint32_t*>(out + ncmd)[lane] = lane == 0 ? insert_len : (lane == 1 ? m_len : m_dist);  // one store
      ++ncmd;
      insert_len = 0;
      copied += m_bytes;
      pos += m_bytes;
      have_m = false;
      break;
    }
  }
  insert_len += uend - pos;
  *tail = insert_len;
  *ncopy = copied;
  dc[0] = dc0; dc[1] = dc1; dc[2] = dc2; dc[3] = dc3;
  return ncmd;
}

// Four parse units per warp (q5 / q6: n_last = 4, the H5/H6 scores): each quarter-warp resolves a window of G = 2 positions x 4
// cached distances, and the greedy / lazy walk is written as straight-line predicated code so that the quarters never diverge.
// With penalties 0,39,43,43 (non-decreasing) the sequential candidate fold of find_match() is exactly "highest score, ties to the
// lower cache index", so a position is resolved in parallel by 4 lanes and 2 shuffle-max steps.  Every "scalar" of
// parse_unit_warp4 is a per-unit value here, held redundantly by the 8 lanes of the unit.  tools/window_emul.cpp checks on the
// CPU that this windowed formulation with G = 2 reproduces parse_range() command for command; it needs about 1.3x the windows of
// G = 8 on text (1.1x - 1.7x over the test inputs), each of them cheaper (one lazy step instead of seven), and a warp retires
// four units at once.
__global__ void __launch_bounds__(PARSE_WARPS * 32, 10) k_parse_pair(Workspace W) {
  constexpr int G = 2;           // positions per window
  constexpr uint32_t SUB = 8;    // lanes per unit
  constexpr uint32_t CAPA = 8;
  const uint32_t FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t hbase = lane & ~7u, hl = lane & 7u;
  const uint32_t j_lane = hl >> 2, i_lane = lane & 3u;
  const bool il1 = (lane & 1u) != 0, il2 = (lane & 2u) != 0;
  const uint32_t gw = blockIdx.x * PARSE_WARPS + (threadIdx.x >> 5);
  const uint32_t u = 4u * gw + lane / SUB;
  const EncParams& P = W.P;
  const uint8_t* data = W.data;
  const uint32_t* best = W.best;
  const bool unit_ok = u < W.num_units;
  const uint32_t s = unit_ok ? u * P.unit : 0u, e = unit_ok ? bmin(P.n, s + P.unit) : 0u;
  uint32_t* const out_w = reinterpret_cast<uint32_t*>(W.raw + (size_t)(unit_ok ? u : 0u) * (P.unit / 2 + 1));
  const uint32_t htl = P.hash_type == 6 ? 8u : 4u;
  const uint32_t window = 64u;
  const bool D = P.use_dict != 0;
  const bool near_start = P.abs_base < P.max_backward;
  const bool warm = unit_ok && (u % P.mb_units) != 0 && s >= BRO_WARMUP_BYTES;
  int stage = unit_ok ? (warm ? 0 : 1) : 2;  // 0 warm-up in front of the unit, 1 the unit, 2 done
  uint32_t pos = stage == 0 ? s - BRO_WARMUP_BYTES : s, uend = stage == 0 ? s : e;
  uint32_t insert_len = 0, ncmd = 0, copied = 0, arh = pos + window;
  bool have_m = false;
  uint32_t m_len = 0, m_dist = 0, m_score = 0;
  int delayed = 0;
  int32_t dc0 = 0x3fffffff, dc1 = 0x3fffffff, dc2 = 0x3fffffff, dc3 = 0x3fffffff;
  uint32_t tail_out = 0, ncopy_out = 0, ncmd_out = 0;
  auto advance = [&]() {  // leaves a finished stage (predicated per half)
    if (stage < 2 && !(have_m || pos + htl < uend)) {
      if (stage == 1) { tail_out = insert_len + (uend - pos); ncopy_out = copied; ncmd_out = ncmd; stage = 2; }
      else { stage = 1; pos = s; uend = e; insert_len = 0; ncmd = 0; copied = 0; arh = s + window; }
    }
  };
  advance();
  advance();
  while (__any_sync(FULL, stage < 2)) {
    const bool act = stage < 2;
    // ---------------- phase A: the 4 positions of this half's window, 4 cache candidates each ----------------
    const uint32_t wbase = pos;
    const uint32_t p = wbase + j_lane;
    const bool p_ok = act && p < uend;
    const uint32_t maxl = p_ok ? uend - p : 0u;
    uint32_t clen = 0, cdist = 0, key = 0;
    if (p_ok) {
      const int32_t back = il2 ? (il1 ? dc3 : dc2) : (il1 ? dc1 : dc0);
      const uint32_t mb = near_start ? bmin(p + P.abs_base, P.max_backward) : P.max_backward;
      if (back > 0 && (uint32_t)back <= mb) {
        const uint64_t x = ldu64(data + p) ^ ldu64(data + p - back);
        uint32_t len = x ? ((uint32_t)(__ffsll((long long)x) - 1) >> 3) : CAPA;
        len = bmin(len, maxl);
        if (len == CAPA && maxl > CAPA) len = lane_lcp_ext(data + p, (uint32_t)back, CAPA, maxl);
        if (len >= 3 || (len == 2 && i_lane < 2)) {
          const uint32_t score = score_last_distance(5, len, i_lane);
          key = (score << 2) | (3u - i_lane);
          clen = len;
          cdist = (uint32_t)back;
        }
      }
    }
    {
      uint32_t k = key;
      k = max(k, __shfl_xor_sync(FULL, k, 1));
      k = max(k, __shfl_xor_sync(FULL, k, 2));
      const int src = (int)((lane & ~3u) + (3u - (k & 3u)));
      const uint32_t wl = __shfl_sync(FULL, clen, src), wd = __shfl_sync(FULL, cdist, src);
      key = k; clen = wl; cdist = wd;
    }
    Match f;
    f.len = key ? clen : 0u; f.dist = key ? cdist : 0u; f.score = key ? (key >> 2) : BRO_MIN_SCORE;
    bool f_found = key != 0;
    if (p_ok && i_lane == 0)  // then the bucket candidate of the match kernel (scores of hash types 5 and 6 are the same)
      f_found = take_best_candidate(best[p], 5, P.lcap, data + p, maxl, near_start ? bmin(p + P.abs_base, P.max_backward) : P.max_backward, D,
                                    lane_lcp_ext, f_found, &f);
    const uint32_t f_len = f.len, f_dist = f.dist, f_score = f.score;
    const uint32_t bal = __ballot_sync(FULL, f_found && i_lane == 0) >> hbase;  // bits 0, 4, .. of this unit's lanes
    uint32_t found = 0;                                                         // bit j <=> a match exists at wbase + j
#pragma unroll
    for (int jj = 0; jj < G; ++jj) found |= ((bal >> (4 * jj)) & 1u) << jj;

    // ---------------- phase B: the walk of parse_unit_warp4 as straight-line predicated code ----------------
    bool wdone = !act, accept = false;
    uint32_t j = 0;
    {
      const bool doA = act && !have_m;
      const uint32_t lim = doA ? bmin((uint32_t)G, uend - htl - wbase) : 0u;
      const uint32_t cand = found & ((1u << lim) - 1u);
      const uint32_t f = cand ? (uint32_t)(__ffs((int)cand) - 1) : lim;
      uint32_t steps = f;
      bool jump = false;
      if (f > 0 && pos + f > arh) { steps = pos > arh ? 1u : (arh - pos + 1u); jump = true; }
      if (doA) { insert_len += steps; pos += steps; j = steps; }
      const int src = (int)(hbase + 4u * bmin(j, (uint32_t)G - 1u));
      const uint32_t a_len = __shfl_sync(FULL, f_len, src), a_dist = __shfl_sync(FULL, f_dist, src), a_score = __shfl_sync(FULL, f_score, src);
      if (doA && jump) {
        const uint32_t margin = bmax(htl - 1u, 4u);
        if (pos + 16 + margin >= uend) { insert_len += uend - pos; pos = uend; }
        else if (pos > arh + 4 * window) { insert_len += 16; pos += 16; }
        else { insert_len += 8; pos += 8; }
        wdone = true;
      } else if (doA && (!cand || j >= (uint32_t)G)) {
        wdone = true;
      } else if (doA) {
        m_len = a_len; m_dist = a_dist; m_score = a_score;
        have_m = true;
        delayed = 0;
      }
    }
#pragma unroll
    for (int st = 0; st < G - 1; ++st) {
      const bool doB = !wdone && !accept && have_m;
      const int src = (int)(hbase + 4u * bmin(j + 1u, (uint32_t)G - 1u));
      const uint32_t b_len = __shfl_sync(FULL, f_len, src), b_dist = __shfl_sync(FULL, f_dist, src), b_score = __shfl_sync(FULL, f_score, src);
      if (doB && j + 1u >= (uint32_t)G) {
        wdone = true;  // re-probe with the window starting at pos
      } else if (doB) {
        const bool f2 = (found >> (j + 1u)) & 1u;
        if (f2 && b_score >= m_score + 175u) {
          pos++;
          insert_len++;
          j++;
          m_len = b_len; m_dist = b_dist; m_score = b_score;
          if (!(++delayed < 4 && pos + htl < uend)) accept = true;
        } else {
          accept = true;
        }
      }
    }
    if (accept) {
      const uint32_t m_bytes = len_bytes(m_len);
      arh = pos + 2 * m_bytes + window;
      if (!len_is_dict(m_len) && (int32_t)m_dist != dc0) { dc3 = dc2; dc2 = dc1; dc1 = dc0; dc0 = (int32_t)m_dist; }
      if (stage == 1 && hl < 3) out_w[3u * ncmd + hl] = hl == 0 ? insert_len : (hl == 1 ? m_len : m_dist);
      ++ncmd;
      insert_len = 0;
      copied += m_bytes;
      pos += m_bytes;
      have_m = false;
    }
    advance();
    advance();
  }
  if (unit_ok && hl == 0) {
    W.unit_ncmd[u] = ncmd_out;
    W.unit_tail[u] = tail_out;
    W.unit_ncopy[u] = ncopy_out;
  }
}

// ---------------------------------------------------------------------------------------------------
// Deep buckets, searched on demand (q7..q9).  k_match_deep looks at up to 256 candidates for EVERY position, but the greedy / lazy
// walk only ever asks for the positions it visits -- about half of them on text, a tenth on record-structured data with long
// copies.  The reference has the same shape (FindLongestMatch runs where the parse stands, mod.rs:2376-2552); what it cannot do is
// run 6144 walks at once.  Here one warp walks one unit with parse_range() of bro_parse.cuh, and at every position it stands on the 32 lanes
// search the bucket list of the sort stage: rank[p] (written by k_rank_sig into the best[] buffer) is the position's index in the
// sorted list, the `depth` entries in front of it are its candidates, nearest first, 32 per round.  sig[] carries, in sorted order,
// key << 17 | 17 hash bits of the entry's first four bytes, so bucket end and the four-byte filter are decided from two coalesced
// 128-byte reads; only the surviving candidates touch their data.  The value computed for a position is exactly k_match_deep's
// best[p], so find_match_ondemand() is find_match() of bro_parse.cuh and the streams are identical.
// ---------------------------------------------------------------------------------------------------
struct DeepArgs {
  MatchArgs m;          // sorted list of the chunk's (single) batch; m.best holds the ranks
  const uint32_t* sig;  // [m.count]
};
__device__ __forceinline__ uint32_t entry_sig(int hash_type, int key_bits, uint32_t w0, uint32_t w1) {
  return (hash_key_from_words(hash_type, key_bits, w0, w1) << 17) | ((w0 * 0x9E3779B1u) >> 15);
}
__global__ void __launch_bounds__(256) k_rank_sig(MatchArgs a, uint32_t* sig) {
  const uint32_t j = blockIdx.x * 256u + threadIdx.x;
  if (j >= a.count) return;
  const uint32_t pos = a.sorted[j];
  const uint64_t w = ldu64(a.data + a.origin + pos);
  sig[j] = entry_sig(a.hash_type, a.key_bits, (uint32_t)w, (uint32_t)(w >> 32));
  if (pos >= a.payload_begin) a.best[a.origin + pos] = j;
}

// Words of a warp's survivor list (s_back): every candidate of a bucket may survive the signature filter.
template <int DEPTH>
struct DeepSurvivors { static constexpr int N = DEPTH > 256 ? DEPTH : 256; };

// best[p] of k_match_deep for the absolute position p, computed by the whole warp (result uniform).  r = rank of p in the sorted
// list, s_back = DeepSurvivors<DEPTH>::N words of shared memory owned by this warp.  A walk is a chain of dependent positions, so what counts is the
// number of memory round trips per position:
//   1. positions and signatures of all DEPTH candidates in one go (lane l: candidates l, l + 32, ..; coalesced), bucket / window
//      end by ballots; the distances of the candidates whose signature agrees are compacted into s_back, nearest first,
//   2. those survivors 32 at a time: first 8 bytes, then 8 more per trip; a candidate that cannot be strictly longer than the
//      best so far is dropped after one byte, and a full-length match ends the search (both exact: a farther candidate that is
//      not longer cannot score higher, score_regular is monotone in both).
template <int DEPTH>
__device__ __forceinline__ void deep_fetch(const DeepArgs& A, uint32_t r, uint32_t* cpos, uint32_t* csig) {  // phase 1 loads
  const uint32_t lane = threadIdx.x & 31;
#pragma unroll
  for (int t = 0; t < DEPTH / 32; ++t) {
    const uint32_t k = (uint32_t)t * 32u + lane;
    cpos[t] = 0; csig[t] = 0;
    if (r >= k + 1u) {
      const uint32_t j = r - 1u - k;
      cpos[t] = __ldg(A.m.sorted + j);
      csig[t] = __ldg(A.sig + j);
    }
  }
}
// L2 prefetch of the candidate lines of a position that will probably be asked for next
template <int DEPTH>
__device__ __forceinline__ void deep_prefetch(const DeepArgs& A, uint32_t r) {
  constexpr uint32_t T = DEPTH / 32;
  const uint32_t lane = threadIdx.x & 31;
  if (lane < 2u * (T + 1u)) {
    const uint32_t* base = lane <= T ? A.m.sorted : A.sig;
    const uint32_t line = lane <= T ? lane : lane - (T + 1u);
    if (r >= 32u * line + 1u) asm volatile("prefetch.global.L2 [%0];" ::"l"(base + (r - 1u - 32u * line)));
  }
}
template <int DEPTH>
__device__ __forceinline__ uint32_t deep_best_warp(const DeepArgs& A, uint32_t p, uint32_t r, const uint32_t* cpos, const uint32_t* csig,
                                                   uint32_t* s_back) {
  constexpr int T = DEPTH / 32;
  const MatchArgs& a = A.m;
  const uint32_t FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x & 31;
  if (a.n - p < 8) return 0u;
  const uint32_t prel = p - a.origin;
  const uint8_t* cur = a.data + p;
  const uint64_t c8 = ldu64(cur);
  const uint32_t mysig = entry_sig(a.hash_type, a.key_bits, (uint32_t)c8, (uint32_t)(c8 >> 32));
  const uint32_t maxl = bmin(a.lcap, a.n - p);
  const uint32_t mbk = bmin(p, a.max_backward);
  const uint32_t kNone = (BRO_MIN_SCORE << 16) | 0xFFFFu;
  uint32_t S = 0;  // survivors so far
  __syncwarp();
#pragma unroll
  for (int t = 0; t < T; ++t) {
    const uint32_t k = (uint32_t)t * 32u + lane;
    const uint32_t backward = prel - cpos[t];
    const bool inwin = r >= k + 1u && (csig[t] >> 17) == (mysig >> 17) && backward <= mbk;  // failing lanes form a suffix
    const uint32_t ended = __ballot_sync(FULL, !inwin);
    const uint32_t surv = __ballot_sync(FULL, inwin && csig[t] == mysig);
    if (inwin && csig[t] == mysig) s_back[S + __popc(surv & ((1u << lane) - 1u))] = backward;
    S += __popc(surv);
    if (ended) break;
  }
  __syncwarp();
  uint32_t bestk = kNone, bl = 0;
  for (uint32_t base = 0; base < S; base += 32) {
    const uint32_t sidx = base + lane;
    uint32_t cand = 0;
    if (sidx < S) {
      const uint32_t backward = s_back[sidx];
      const uint8_t* cp = cur - backward;
      const uint64_t x = ldu64(cp) ^ c8;
      if ((uint32_t)x == 0u) {  // else: signature collision
        uint32_t len = 0;
        if (x) len = 4u + ((uint32_t)(__ffs((int)(uint32_t)(x >> 32)) - 1) >> 3);
        else if (!(bl >= 8u && bl < maxl && cur[bl] != cp[bl])) {
          len = 8;
          while (len + 8 <= maxl) {
            const uint64_t y = ldu64(cur + len) ^ ldu64(cp + len);
            if (y) { len += (uint32_t)(__ffsll((long long)y) - 1) >> 3; break; }
            len += 8;
          }
          if (len + 8 > maxl) while (len < maxl && cur[len] == cp[len]) ++len;
        }
        if (len) {
          len = bmin(len, maxl);
          cand = DeepKey<DEPTH>::make(score_regular(a.hash_type, len, backward), sidx, len);
        }
      }
    }
    const uint32_t wmax = __reduce_max_sync(FULL, cand);
    if (wmax > bestk) { bestk = wmax; bl = wmax & DeepKey<DEPTH>::LMASK; }
    if (bestk != kNone && bl == maxl) break;
  }
  uint32_t res = 0;
  if (bestk != kNone) res = (s_back[DeepKey<DEPTH>::index(bestk)] << 8) | (bestk & DeepKey<DEPTH>::LMASK);
  else if (a.use_dict) {
    const uint64_t c16 = ldu64(cur + 8);
    res = dict_candidate_dev(a.dict, a.hash_type, (uint32_t)c8, (uint32_t)(c8 >> 32), (uint32_t)c16, (uint32_t)(c16 >> 32), cur, a.n - p, mbk);
  }
  __syncwarp();
  return res;
}

// Test probe of the on-demand search: deep_best_warp() at every position of [start, start + len), one warp per position, into
// out[len].  Launched right after k_rank_sig (while the ranks, signatures and sorted list are intact) only when a stage hook asks.
template <int DEPTH>
__global__ void __launch_bounds__(256) k_od_probe(DeepArgs A, uint32_t start, uint32_t len, uint32_t* out) {
  __shared__ uint32_t s_back_all[8][DeepSurvivors<DEPTH>::N];
  const uint32_t w = blockIdx.x * 8u + (threadIdx.x >> 5);
  if (w >= len) return;
  const uint32_t p = start + w;
  const uint32_t r = A.m.best[p];
  uint32_t cpos[DEPTH / 32], csig[DEPTH / 32];
  deep_fetch<DEPTH>(A, r, cpos, csig);
  const uint32_t b = deep_best_warp<DEPTH>(A, p, r, cpos, csig, s_back_all[threadIdx.x >> 5]);
  if ((threadIdx.x & 31) == 0) out[w] = b;
}

// find_match() of bro_parse.cuh at the range-relative position pos, whole warp: lane i probes cached distance i, then the bucket
template <int NL, int DEPTH>
__device__ __forceinline__ bool find_match_ondemand(const EncParams& P, const DeepArgs& A, const uint8_t* data, const int32_t* dca,
                                                    uint32_t pos, uint32_t maxl, bool D, uint32_t rank, uint32_t rank_next,
                                                    uint32_t* s_back, Match* out) {
  constexpr uint32_t CAPA = 8;
  const uint32_t FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x & 31;
  const int ht = P.hash_type;
  uint32_t cpos[DEPTH / 32], csig[DEPTH / 32];
  deep_fetch<DEPTH>(A, rank, cpos, csig);   // in flight while the cached distances are probed
  deep_prefetch<DEPTH>(A, rank_next);
  const uint32_t mb = (P.abs_base >= P.max_backward) ? P.max_backward : bmin(pos + P.abs_base, P.max_backward);
  uint32_t key = 0;
  if (lane < (uint32_t)NL) {
    const int32_t back = cache_candidate(dca, (int)lane);
    if (back > 0 && (uint32_t)back <= mb) {
      const uint64_t x = ldu64(data + pos) ^ ldu64(data + pos - back);
      uint32_t len = x ? ((uint32_t)(__ffsll((long long)x) - 1) >> 3) : CAPA;
      len = bmin(len, maxl);
      if (len == CAPA && maxl > CAPA) len = lane_lcp_ext(data + pos, (uint32_t)back, CAPA, maxl);
      if (len >= 3 || (len == 2 && lane < 2)) key = last_distance_key(ht, len, maxl, lane);
    }
  }
  key = __reduce_max_sync(FULL, key);
  Match f;
  f.len = 0; f.dist = 0; f.score = BRO_MIN_SCORE;
  if (key) {
    const uint32_t wi = last_distance_key_decode(key, &f.len);
    f.dist = (uint32_t)cache_candidate(dca, (int)wi);
    f.score = score_last_distance(ht, f.len, wi);
  }
  const uint32_t b = deep_best_warp<DEPTH>(A, P.abs_base + pos, rank, cpos, csig, s_back);
  const bool found = take_best_candidate(b, ht, P.lcap, data + pos, maxl, mb, D, warp_lcp_ext, key != 0, &f);
  *out = f;
  return found;
}

// (a 512-deep bucket holds 32 candidate registers per lane: at 8 CTAs per SM, i.e. 64 registers, that walk spilled 180 bytes;
// at 6 it takes 80 registers and spills 64 bytes, about what the 256-deep walk spills at 8)
template <int NL, int DEPTH>
__global__ void __launch_bounds__(PARSE_WARPS * 32, DEPTH > 256 ? 6 : 8) k_parse_ondemand(Workspace W, DeepArgs A) {
  const uint32_t u = blockIdx.x * PARSE_WARPS + (threadIdx.x >> 5);
  if (u >= W.num_units) return;
  const EncParams& P = W.P;
  const uint32_t s = u * P.unit, e = bmin(P.n, s + P.unit);
  uint32_t tail = 0, ncopy = 0, ncmd = 0;
  const bool D = P.use_dict != 0;
  int32_t dc[4] = {0x3fffffff, 0x3fffffff, 0x3fffffff, 0x3fffffff};
  const bool warm = (u % P.mb_units) != 0 && s >= BRO_WARMUP_BYTES;
  RawCmd* const out = W.raw + (size_t)u * (P.unit / 2 + 1);
  __shared__ uint32_t s_back_all[PARSE_WARPS][DeepSurvivors<DEPTH>::N];
  uint32_t* const s_back = s_back_all[threadIdx.x >> 5];
  const uint32_t FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x & 31;
  for (int phase = warm ? 0 : 1; phase < 2; ++phase) {
    const uint32_t rs = phase ? s : s - BRO_WARMUP_BYTES, re = phase ? e : s;
    RawCmd* const o = phase ? out : nullptr;
    // ranks of 64 consecutive positions ride in the lanes (two registers): the walk mostly moves a few bytes at a time, and the
    // second half is reloaded one half ahead of its use
    uint32_t rk_base = 0x80000000u, rk0 = 0, rk1 = 0;  // (no position is that large: the first query loads)
    auto rank_load = [&](uint32_t q) -> uint32_t { return q + lane < P.n ? __ldg(A.m.best + P.abs_base + q + lane) : 0u; };
    auto rank_of = [&](uint32_t q) -> uint32_t {
      uint32_t d = q - rk_base;
      if (d >= 64u) { rk_base = q; rk0 = rank_load(q); rk1 = rank_load(q + 32u); d = 0; }
      else if (d >= 32u) { rk_base += 32u; rk0 = rk1; rk1 = rank_load(rk_base + 32u); d -= 32u; }
      return __shfl_sync(FULL, rk0, (int)d);
    };
    auto rank_peek = [&](uint32_t q) -> uint32_t {  // rank of a position inside the window (0 outside: prefetch only)
      const uint32_t d = q - rk_base;
      const uint32_t v0 = __shfl_sync(FULL, rk0, (int)(d & 31u)), v1 = __shfl_sync(FULL, rk1, (int)(d & 31u));
      return d < 32u ? v0 : (d < 64u ? v1 : 0u);
    };
    auto find = [&](uint32_t q, uint32_t max_len, Match* m) {
      return find_match_ondemand<NL, DEPTH>(P, A, W.data, dc, q, max_len, D, rank_of(q), rank_peek(q + 1), s_back, m);
    };
    auto store = [&](uint32_t k, uint32_t ins, uint32_t len, uint32_t dist) {
      if (o && lane < 3) reinterpret_cast<uint32_t*>(o + k)[lane] = lane == 0 ? ins : (lane == 1 ? len : dist);
    };
    ncmd = parse_range(P, rs, re, dc, find, store, &tail, &ncopy);
  }
  if ((threadIdx.x & 31) == 0) {
    W.unit_ncmd[u] = ncmd;
    W.unit_tail[u] = tail;
    W.unit_ncopy[u] = ncopy;
  }
}

#ifndef PARSE_MIN_BLOCKS
#define PARSE_MIN_BLOCKS 10
#endif
// q7..q9 with the bucket candidates of every position found up front: one parse unit per warp, NL = n_last = 10 / 16
template <int NL>
__global__ void __launch_bounds__(PARSE_WARPS * 32, PARSE_MIN_BLOCKS) k_parse(Workspace W) {
  const uint32_t u = blockIdx.x * PARSE_WARPS + (threadIdx.x >> 5);
  if (u >= W.num_units) return;
  const EncParams& P = W.P;
  const uint32_t s = u * P.unit, e = bmin(P.n, s + P.unit);
  uint32_t tail, ncopy, ncmd;
  const uint32_t cu = P.unit / 2 + 1;
  const bool D = P.use_dict != 0;
  // phase 0: warm-up over the BRO_WARMUP_BYTES in front of the unit (commands discarded, only the distance cache is kept);
  // phase 1: the unit itself.  One loop body so that the parse code is instantiated once.
  int32_t dc[4] = {0x3fffffff, 0x3fffffff, 0x3fffffff, 0x3fffffff};
  const bool warm = (u % P.mb_units) != 0 && s >= BRO_WARMUP_BYTES;
  RawCmd* const out = W.raw + (size_t)u * cu;
  ncmd = 0;
  for (int phase = warm ? 0 : 1; phase < 2; ++phase) {
    const uint32_t rs = phase ? s : s - BRO_WARMUP_BYTES, re = phase ? e : s;
    ncmd = parse_unit_warp4<NL>(P, W.data, W.best, rs, re, phase ? out : nullptr, &tail, &ncopy, D, dc);
  }
  if ((threadIdx.x & 31) == 0) {
    W.unit_ncmd[u] = ncmd;
    W.unit_tail[u] = tail;
    W.unit_ncopy[u] = ncopy;
  }
}

__device__ __forceinline__ UnitView unit_view(const Workspace& W) {
  UnitView V;
  V.raw = W.raw; V.ncmd = W.unit_ncmd; V.tail = W.unit_tail;
  V.cu = W.P.unit / 2 + 1; V.unit = W.P.unit; V.n = W.P.n;
  return V;
}

// block-wide exclusive scan helper (blockDim.x == 1024), returns exclusive prefix and total via smem
__device__ __forceinline__ uint32_t block_excl_scan_1024(uint32_t v, uint32_t* s_warp, uint32_t* total) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= (uint32_t)o) x += y;
  }
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  if (wid == 0) {
    uint32_t w = s_warp[lane];
    uint32_t xs = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t y = __shfl_up_sync(0xffffffffu, xs, o);
      if (lane >= (uint32_t)o) xs += y;
    }
    s_warp[lane] = xs - w;
    if (lane == 31) s_warp[32] = xs;
  }
  __syncthreads();
  uint32_t r = s_warp[wid] + x - v;
  *total = s_warp[32];
  __syncthreads();
  return r;
}

// Metablock descriptors of a chunk: fixed spans of mb_units parse units.
__global__ void k_init_mb(Workspace W) {
  const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= W.num_mb) return;
  MBDesc d;
  memset(&d, 0, sizeof(d));
  d.u0 = m * W.P.mb_units;
  d.u1 = min(W.num_units, d.u0 + W.P.mb_units);
  d.start = d.u0 * W.P.unit;
  d.len = (uint32_t)min((uint64_t)W.P.n, (uint64_t)d.u1 * W.P.unit) - d.start;
  W.mb[m] = d;
}
// One CTA (1024 threads) per metablock: per-unit final command counts and literal counts -> exclusive scans.
__global__ void __launch_bounds__(1024) k_fin_count(Workspace W) {
  __shared__ uint32_t s_warp[33];
  const uint32_t m = blockIdx.x;
  MBDesc& mb = W.mb[m];
  const UnitView V = unit_view(W);
  uint32_t cmd_run = 0, lit_run = 0;
  for (uint32_t ub = mb.u0; ub < mb.u1; ub += 1024) {
    uint32_t u = ub + threadIdx.x;
    uint32_t nc = 0, nl = 0;
    if (u < mb.u1) {
      nc = unit_final_ncmd(V, mb.u0, mb.u1, u);
      uint32_t ulen = bmin(W.P.n, (u + 1) * W.P.unit) - u * W.P.unit;
      nl = ulen - W.unit_ncopy[u];
    }
    uint32_t tc, tl;
    uint32_t ec = block_excl_scan_1024(nc, s_warp, &tc);
    uint32_t el = block_excl_scan_1024(nl, s_warp, &tl);
    if (u < mb.u1) { W.unit_cmd_off[u] = cmd_run + ec; W.unit_lit_off[u] = lit_run + el; }
    cmd_run += tc;
    lit_run += tl;
  }
  if (threadIdx.x == 0) { mb.ncmd = cmd_run; mb.nlit = lit_run; mb.has_long = 0; }
}
// Incoming distance cache of raw command i of unit u: the last (up to) four distinct-run distances before it, looking
// back inside the unit and, if needed, into earlier units of the metablock (same rule as finalize_unit()).
__device__ __forceinline__ void lookback_cache(const UnitView& V, uint32_t u0, uint32_t u, uint32_t i, int32_t* dc) {
  dc[0] = dc[1] = dc[2] = dc[3] = 0x3fffffff;
  int k = 0;
  uint32_t last = 0;
  uint32_t v = u, idx = i;
  for (;;) {
    while (idx > 0 && k < 4) {
      --idx;
      if (len_is_dict(V.raw[(size_t)v * V.cu + idx].copy_len)) continue;  // not part of the distance sequence
      const uint32_t d = V.raw[(size_t)v * V.cu + idx].distance;
      if (d != last) { dc[k++] = (int32_t)d; last = d; }
    }
    if (k >= 4 || v == u0) break;
    --v;
    idx = V.ncmd[v];
  }
}

// Warp-parallel form of finalize_unit(): lanes take consecutive raw commands; positions / literal ranks / distance
// ranks come from warp scans, the distance cache from a short per-lane look-back.  Identical output.
__global__ void __launch_bounds__(PARSE_WARPS * 32) k_fin_write(Workspace W) {
  const uint32_t u = blockIdx.x * PARSE_WARPS + (threadIdx.x >> 5);
  if (u >= W.num_units) return;
  const uint32_t FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t m = u / W.P.mb_units;
  const MBDesc& mb = W.mb[m];
  const UnitView V = unit_view(W);
  const uint32_t u0 = mb.u0, u1 = mb.u1;
  GCmd* out = W.cmds + (size_t)m * W.cmd_cap + W.unit_cmd_off[u];
  const uint32_t ustart = u * V.unit;
  const uint32_t nraw = V.ncmd[u];
  const RawCmd* rc = V.raw + (size_t)u * V.cu;
  const bool absorbed = unit_absorbed(V, u0, u);
  const uint32_t carry = unit_carry_in(V, u0, u);
  uint32_t cont = 0;  // bytes absorbed from following units by the last command
  if (nraw) {
    for (uint32_t v = u + 1; v < u1 && unit_absorbed(V, u0, v); ++v) {
      cont += V.raw[(size_t)v * V.cu].copy_len;
      if (!(V.ncmd[v] == 1 && V.tail[v] == 0)) break;
    }
  }
  uint32_t lit_run = W.unit_lit_off[u], pos_run = ustart, nd_run = 0;
  const uint32_t skip = absorbed ? 1u : 0u;
  for (uint32_t base = 0; base < nraw; base += 32) {
    const uint32_t i = base + lane;
    const bool act = i < nraw;
    uint32_t ins_r = 0, len_r = 0, dist = 0;
    if (act) { ins_r = rc[i].insert_len; len_r = rc[i].copy_len; dist = rc[i].distance; }
    // exclusive warp scans of literals and of covered bytes
    const uint32_t bytes_r = len_bytes(len_r);
    uint32_t sl = ins_r, sp = ins_r + bytes_r;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t a1 = __shfl_up_sync(FULL, sl, o), a2 = __shfl_up_sync(FULL, sp, o);
      if (lane >= (uint32_t)o) { sl += a1; sp += a2; }
    }
    const uint32_t lit_before = lit_run + sl - ins_r, pos_before = pos_run + sp - (ins_r + bytes_r);
    const bool emit = act && !(i == 0 && absorbed);
    uint32_t cmd_prefix = 0, sym_nbits = 0, extra = 0, ins = ins_r, len = len_r;
    if (emit) {
      if (i == 0) ins += carry;
      if (i + 1 == nraw) len += cont;
      int32_t dc[4];
      lookback_cache(V, u0, u, i, dc);
      const uint32_t code = len_is_dict(len) ? dist + 15u : compute_distance_code(dist, dc);
      prefix_encode_copy_distance(code, &sym_nbits, &extra);
      cmd_prefix = combine_length_codes(insert_length_code(ins), copy_length_code(len_coded(len)), code == 0);
    }
    const uint32_t hd = __ballot_sync(FULL, emit && cmd_prefix >= 128);
    if (emit) {
      GCmd g;
      g.insert_len = ins;
      g.copy_len = len;
      g.dist_extra = extra;
      g.cmd_prefix = (uint16_t)cmd_prefix;
      g.dist_prefix = (uint16_t)sym_nbits;
      g.lit_idx = lit_before - (i == 0 ? carry : 0u);
      g.dist_idx = nd_run + __popc(hd & ((1u << lane) - 1u));
      g.pos = pos_before - (i == 0 ? carry : 0u);
      g.pad = u;
      out[i - skip] = g;
    }
    lit_run += __shfl_sync(FULL, sl, 31);
    pos_run += __shfl_sync(FULL, sp, 31);
    nd_run += __popc(hd);
  }
  if (lane == 0) {
    if (u + 1 == u1) {
      const uint32_t carry_out = V.tail[u] + (nraw == 0 ? carry : 0u);
      if (carry_out) {
        const uint32_t uend = bmin(V.n, ustart + V.unit);
        GCmd g;
        g.insert_len = carry_out;
        g.copy_len = 0;
        g.dist_extra = 0;
        g.dist_prefix = 0;
        g.cmd_prefix = (uint16_t)combine_length_codes(insert_length_code(carry_out), copy_length_code(4), false);
        g.lit_idx = lit_run + V.tail[u] - carry_out;
        g.dist_idx = nd_run;
        g.pos = uend - carry_out;
        g.pad = u;
        out[nraw - skip] = g;
      }
    }
    W.unit_ndist[u] = nd_run;
  }
}
// One CTA per metablock: scan distance-symbol counts over units and add the prefix to each command.
__global__ void __launch_bounds__(1024) k_fin_dist(Workspace W) {
  __shared__ uint32_t s_warp[33];
  const uint32_t m = blockIdx.x;
  MBDesc& mb = W.mb[m];
  uint32_t run = 0;
  for (uint32_t ub = mb.u0; ub < mb.u1; ub += 1024) {
    uint32_t u = ub + threadIdx.x;
    uint32_t nd = u < mb.u1 ? W.unit_ndist[u] : 0;
    uint32_t tot;
    uint32_t ex = block_excl_scan_1024(nd, s_warp, &tot);
    if (u < mb.u1) W.unit_dist_off[u] = run + ex;  // commands carry their unit in GCmd::pad and add this at use
    run += tot;
  }
  if (threadIdx.x == 0) mb.ndist = run;
}


// ---------------------------------------------------------------------------------------------------
// Long inserts.  A command with more than LONG_INS literals would serialise its thread in k_symbols / k_bitlen /
// k_emit_body (incompressible input is one 4 Mi-literal command per metablock), so those kernels skip its literals and
// the *_long kernels below finish them, one CTA per LONG_INS-literal segment.  Long commands are found through a table
// indexed by (pos - mb.start) / LONG_INS: two commands with more than LONG_INS literals never share a slot.
// ---------------------------------------------------------------------------------------------------
#define LONG_INS 512u
#define LONG_GRID 64u
__device__ __forceinline__ uint32_t block_excl_scan_256(uint32_t v, uint32_t* s_warp /*[9]*/, uint32_t* total) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= (uint32_t)o) x += y;
  }
  __syncthreads();
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  uint32_t woff = 0, tot = 0;
#pragma unroll
  for (uint32_t w = 0; w < 8; ++w) { const uint32_t t = s_warp[w]; if (w < wid) woff += t; tot += t; }
  *total = tot;
  return woff + x - v;
}
// Calls f(cmd_idx, g, slot, k) with the whole CTA (256 threads) for every segment k of every long command of metablock
// blockIdx.y that this CTA owns; segments are dealt round-robin over the LONG_GRID CTAs of the metablock.
template <typename F>
__device__ __forceinline__ void for_each_long_segment(const Workspace& W, F f) {
  __shared__ uint32_t s_mask[8];
  const uint32_t m = blockIdx.y;
  const MBDesc& mb = W.mb[m];
  if (!mb.has_long) return;
  const uint32_t nslots = (mb.len + LONG_INS - 1) / LONG_INS;
  const uint2* tab = W.long_tab + (size_t)m * W.long_cap;
  for (uint32_t sb = 0; sb < nslots; sb += 256) {
    const uint32_t s = sb + threadIdx.x;
    const uint32_t v = s < nslots ? tab[s].x : 0u;
    const uint32_t bal = __ballot_sync(0xffffffffu, v != 0);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_mask[threadIdx.x >> 5] = bal;
    __syncthreads();
    for (uint32_t w = 0; w < 8; ++w) {
      uint32_t mask = s_mask[w];
      while (mask) {
        const uint32_t slot = sb + w * 32 + (uint32_t)__ffs((int)mask) - 1u;
        mask &= mask - 1u;
        const uint32_t ci = tab[slot].x - 1u;
        const GCmd g = W.cmds[(size_t)m * W.cmd_cap + ci];
        const uint32_t nseg = (g.insert_len + LONG_INS - 1) / LONG_INS;
        for (uint32_t k = (blockIdx.x + LONG_GRID - slot % LONG_GRID) % LONG_GRID; k < nseg; k += LONG_GRID) f(ci, g, slot, k);
      }
    }
  }
}
__global__ void __launch_bounds__(256) k_symbols_long(Workspace W) {
  const uint32_t m = blockIdx.y;
  const MBDesc& mb = W.mb[m];
  const int id = mb.ctx_map_id;
  const uint8_t* d = W.data;
  for_each_long_segment(W, [&](uint32_t, const GCmd& g, uint32_t, uint32_t k) {
    uint16_t* ls = W.lit_syms + mb.start + g.lit_idx;
    for (uint32_t off = k * LONG_INS + threadIdx.x; off < min(g.insert_len, (k + 1) * LONG_INS); off += 256) {
      const uint32_t pos = g.pos + off;
      const uint8_t p1 = ((uint64_t)W.P.abs_base + pos >= 1) ? d[(int64_t)pos - 1] : 0, p2 = ((uint64_t)W.P.abs_base + pos >= 2) ? d[(int64_t)pos - 2] : 0;
      const uint32_t cx = (id && !(id >= CTXMAP_FULL_UTF8 && !W.P.ctx_model)) ? ctxmap_lookup(id, literal_context(id, p1, p2)) : 0u;
      ls[off] = (uint16_t)(d[pos] | (cx << 8));
    }
  });
}
__global__ void __launch_bounds__(256) k_bitlen_long(Workspace W) {
  __shared__ uint32_t s_warp[9];
  const uint32_t m = blockIdx.y;
  const MetaCodes mc = make_codes(W, m);
  for_each_long_segment(W, [&](uint32_t, const GCmd& g, uint32_t slot, uint32_t k) {
    CountWriter w;
    w.bits = 0;
    for (uint32_t off = k * LONG_INS + threadIdx.x; off < min(g.insert_len, (k + 1) * LONG_INS); off += 256)
      emit_one_literal(w, mc, g.lit_idx + off, W.data, g.pos + off, W.P.abs_base);
    uint32_t tot;
    block_excl_scan_256((uint32_t)w.bits, s_warp, &tot);
    if (threadIdx.x == 0) {
      W.seg_bits[(size_t)m * W.long_cap + slot + k] = tot;
      atomicAdd(&W.long_tab[(size_t)m * W.long_cap + slot].y, tot);
    }
  });
}

// ---------------------------------------------------------------------------------------------------
// Literal context decision: one CTA per metablock (encode.rs:1873-1927 in Q16).
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_ctx_decide(Workspace W) {
  __shared__ CtxSampleHist sh;
  const uint32_t m = blockIdx.x;
  MBDesc& mb = W.mb[m];
  uint32_t* raw = reinterpret_cast<uint32_t*>(&sh);
  for (uint32_t i = threadIdx.x; i < sizeof(CtxSampleHist) / 4; i += blockDim.x) raw[i] = 0;
  __syncthreads();
  const EncParams& P = W.P;
  if (P.hq_meta && P.hq_split) {  // ChooseContextMode (encode.rs:1357-1377), decided on the first 64 KiB
    if (threadIdx.x == 0) mb.ctx_map_id = hq_is_mostly_utf8(W.data + mb.start, bmin(mb.len, 65536u)) ? CTXMAP_FULL_UTF8 : CTXMAP_FULL_SIGNED;
    return;
  }
  if (!P.ctx_model || P.quality < 5 || mb.len < 64) {
    if (threadIdx.x == 0) mb.ctx_map_id = CTXMAP_NONE;
    return;
  }
  const bool complex_map = P.size_hint >= (1u << 20);
  const uint32_t nstrides = (mb.len - 64) / 4096 + 1;
  for (uint32_t s = threadIdx.x; s < nstrides; s += blockDim.x) {
    // one stride per thread into a private histogram would not fit; accumulate with shared atomics
    const uint8_t* d = W.data;
    uint32_t sp = mb.start + s * 4096;
    if (complex_map) {
      uint8_t prev2 = d[sp], prev1 = d[sp + 1];
      for (uint32_t pos = sp + 2; pos < sp + 64; ++pos) {
        uint8_t lit = d[pos];
        uint32_t cx = ctxmap_lookup(CTXMAP_COMPLEX13, context_utf8(prev1, prev2));
        atomicAdd(&sh.total, 1u);
        atomicAdd(&sh.combined[lit >> 3], 1u);
        atomicAdd(&sh.ctx[cx][lit >> 3], 1u);
        prev2 = prev1;
        prev1 = lit;
      }
    }
    uint32_t prev = (d[sp] >> 6) == 0 ? 0u : ((d[sp] >> 6) - 1u) * 3u;
    for (uint32_t pos = sp + 1; pos < sp + 64; ++pos) {
      uint32_t cl = d[pos] >> 6;
      uint32_t l = cl == 0 ? 0u : cl - 1u;
      atomicAdd(&sh.bigram[prev + l], 1u);
      prev = l * 3u;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) mb.ctx_map_id = ctx_decide_from_hist(P.quality, P.size_hint, &sh, W.lut);
}

// ---------------------------------------------------------------------------------------------------
// Symbol streams: one thread per command.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_symbols(Workspace W) {
  const uint32_t m = blockIdx.y;
  const MBDesc& mb = W.mb[m];
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= mb.ncmd) return;
  const GCmd c = W.cmds[(size_t)m * W.cmd_cap + i];
  W.cmd_syms[(size_t)m * W.cmd_cap + i] = c.cmd_prefix;
  const int id = mb.ctx_map_id;
  if (c.copy_len != 0 && c.cmd_prefix >= 128)  // quality >= 10: the distance context rides in bits 10..11
    W.dist_syms[(size_t)m * W.cmd_cap + c.dist_idx + W.unit_dist_off[c.pad]] =
        (uint16_t)((c.dist_prefix & 0x3ffu) | (id >= CTXMAP_FULL_UTF8 ? distance_context(c.cmd_prefix) << 10 : 0u));
  const uint8_t* d = W.data;
  uint16_t* ls = W.lit_syms + mb.start + c.lit_idx;
  if (c.insert_len > LONG_INS) {  // finished by k_symbols_long
    W.long_tab[(size_t)m * W.long_cap + (c.pos - mb.start) / LONG_INS].x = i + 1;
    W.mb[m].has_long = 1;
    return;
  }
  uint8_t p1 = ((uint64_t)W.P.abs_base + c.pos >= 1) ? d[(int64_t)c.pos - 1] : 0, p2 = ((uint64_t)W.P.abs_base + c.pos >= 2) ? d[(int64_t)c.pos - 2] : 0;
  for (uint32_t j = 0; j < c.insert_len; ++j) {
    uint8_t lit = d[c.pos + j];
    uint32_t cx = (id && !(id >= CTXMAP_FULL_UTF8 && !W.P.ctx_model)) ? ctxmap_lookup(id, literal_context(id, p1, p2)) : 0u;
    ls[j] = (uint16_t)(lit | (cx << 8));
    p2 = p1;
    p1 = lit;
  }
}

// ---------------------------------------------------------------------------------------------------
// Histograms / block split.  grid = (num_mb, 3 categories).
// ---------------------------------------------------------------------------------------------------
struct CatInfo {
  const uint16_t* syms;
  uint32_t count, A, nctx, min_block, thr_bits, max_types;
  uint8_t* types;
  uint32_t *lengths, *starts, *hist, *counts;  // counts -> {num_blocks, num_types}
};
__device__ __forceinline__ CatInfo cat_info(const Workspace& W, uint32_t m, int cat) {
  CatInfo c;
  const MBDesc& mb = W.mb[m];
  if (cat == 0) {
    c.syms = W.lit_syms + mb.start; c.count = mb.nlit; c.A = 256; c.nctx = ctxmap_num_contexts(mb.ctx_map_id);
    c.min_block = 512; c.thr_bits = 400; c.max_types = c.nctx == 1 ? 256u : 256u / c.nctx;
    c.types = W.lit_types + (size_t)m * W.lit_blk_cap; c.lengths = W.lit_lengths + (size_t)m * W.lit_blk_cap;
    c.starts = W.lit_starts + (size_t)m * W.lit_blk_cap;
    c.hist = W.lit_hist + (size_t)m * (W.max_lit_trees + 13) * 256; c.counts = W.split_counts + (size_t)m * 6;
  } else if (cat == 1) {
    c.syms = W.cmd_syms + (size_t)m * W.cmd_cap; c.count = mb.ncmd; c.A = 704; c.nctx = 1;
    c.min_block = 1024; c.thr_bits = 500; c.max_types = 256;
    c.types = W.cmd_types + (size_t)m * W.cmd_blk_cap; c.lengths = W.cmd_lengths + (size_t)m * W.cmd_blk_cap;
    c.starts = W.cmd_starts + (size_t)m * W.cmd_blk_cap;
    c.hist = W.cmd_hist + (size_t)m * (W.max_cmd_types + 1) * 704; c.counts = W.split_counts + (size_t)m * 6 + 2;
  } else {
    c.syms = W.dist_syms + (size_t)m * W.cmd_cap; c.count = mb.ndist; c.A = W.dist_A; c.nctx = 1;
    c.min_block = 512; c.thr_bits = 100; c.max_types = 256;
    c.types = W.dist_types + (size_t)m * W.dist_blk_cap; c.lengths = W.dist_lengths + (size_t)m * W.dist_blk_cap;
    c.starts = W.dist_starts + (size_t)m * W.dist_blk_cap;
    c.hist = W.dist_hist + (size_t)m * (W.max_dist_types + 1) * W.dist_A; c.counts = W.split_counts + (size_t)m * 6 + 4;
  }
  if (c.max_types > (cat == 0 ? W.max_lit_trees / c.nctx : (cat == 1 ? W.max_cmd_types : W.max_dist_types)))
    c.max_types = (cat == 0 ? W.max_lit_trees / c.nctx : (cat == 1 ? W.max_cmd_types : W.max_dist_types));
  return c;
}

// Greedy splitter: one CTA per (metablock, category); the symbol stream is consumed block by block, histograms
// live in global memory (L2 resident), entropies are reduced in parallel, thread 0 takes the decision with the
// same split_decide() the CPU model uses.
#define SPLIT_THREADS 512
#define SPLIT_WARPS (SPLIT_THREADS / 32)

// The three live histograms (pending block, last and second-last block type) stay in shared memory; the per-type slots
// in global memory are written through whenever a type's histogram changes and are never read back.  With literal
// contexts each warp owns one context, so a FinishBlock step costs one warp reduction instead of one per context.
#define SPLIT_SMEM_WORDS (3 * 13 * 256)
__global__ void __launch_bounds__(SPLIT_THREADS) k_split_greedy(Workspace W) {
  extern __shared__ uint32_t s_hist3[];             // [3][HA]
  __shared__ uint64_t s_part[3][SPLIT_WARPS];       // nctx == 1: sum c*log2(c) partials of pending, pending+last0, pending+last1
  __shared__ uint32_t s_cnt[3][SPLIT_WARPS];
  __shared__ uint64_t s_e[3][13];
  __shared__ SplitState st;
  __shared__ int s_action;
  __shared__ uint32_t s_nblocks, s_new_type;
  __shared__ uint32_t s_ic, s_i0, s_i1;             // buffer of the pending / last / second-last histogram (i0 may equal i1)
  const uint32_t m = blockIdx.x;
  const CatInfo c = cat_info(W, m, (int)blockIdx.y);
  const uint32_t A = c.A, nctx = c.nctx, HA = nctx * A;
  const uint32_t* lut = W.lut;
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    memset(&st, 0, sizeof(st));
    st.target_block_size = c.min_block;
    s_nblocks = 0;
    s_ic = 0; s_i0 = 1; s_i1 = 1;
  }
  for (uint32_t i = threadIdx.x; i < 3 * HA; i += SPLIT_THREADS) s_hist3[i] = 0;
  __syncthreads();
  uint32_t consumed = 0;
  for (;;) {
    const uint32_t target = st.target_block_size;
    const uint32_t remaining = c.count - consumed;
    const bool is_final = remaining < target;   // the last call takes whatever is left (possibly nothing)
    const uint32_t take = is_final ? remaining : target;
    const uint32_t nb = st.num_blocks;
    uint32_t* cur = s_hist3 + s_ic * HA;
    const uint32_t* l0 = s_hist3 + s_i0 * HA;
    const uint32_t* l1 = s_hist3 + s_i1 * HA;
    for (uint32_t i = threadIdx.x; i < take; i += SPLIT_THREADS) {
      uint32_t sv = c.syms[consumed + i];
      uint32_t sym = nctx == 1 ? sv : (sv & 0xFFu) + (sv >> 8) * A;
      atomicAdd(&cur[sym], 1u);
    }
    __syncthreads();
    consumed += take;
    if (nctx > 1) {  // A == 256: warp cx reduces context cx
      if (wid < nctx) {
        const uint32_t cx = wid;
        uint64_t a0 = 0, a1 = 0, a2 = 0;
        uint32_t t0 = 0, t1 = 0, t2 = 0;
#pragma unroll
        for (uint32_t r = 0; r < 8; ++r) {
          const uint32_t k = cx * 256u + r * 32u + lane;
          const uint32_t v = cur[k];
          if (v) { a0 += xlog2x_q16(lut, v); t0 += v; }
          if (nb) {
            const uint32_t v0 = v + l0[k], v1 = v + l1[k];
            if (v0) { a1 += xlog2x_q16(lut, v0); t1 += v0; }
            if (v1) { a2 += xlog2x_q16(lut, v1); t2 += v1; }
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          a0 += __shfl_xor_sync(0xffffffffu, a0, o); a1 += __shfl_xor_sync(0xffffffffu, a1, o);
          a2 += __shfl_xor_sync(0xffffffffu, a2, o); t0 += __shfl_xor_sync(0xffffffffu, t0, o);
          t1 += __shfl_xor_sync(0xffffffffu, t1, o); t2 += __shfl_xor_sync(0xffffffffu, t2, o);
        }
        if (lane < 3) s_e[lane][cx] = bits_entropy_q16(lane == 0 ? a0 : (lane == 1 ? a1 : a2), lane == 0 ? t0 : (lane == 1 ? t1 : t2), lut);
      }
    } else {
      uint64_t a0 = 0, a1 = 0, a2 = 0;
      uint32_t t0 = 0, t1 = 0, t2 = 0;
      for (uint32_t k = threadIdx.x; k < A; k += SPLIT_THREADS) {
        const uint32_t v = cur[k];
        if (v) { a0 += xlog2x_q16(lut, v); t0 += v; }
        if (nb) {
          const uint32_t v0 = v + l0[k], v1 = v + l1[k];
          if (v0) { a1 += xlog2x_q16(lut, v0); t1 += v0; }
          if (v1) { a2 += xlog2x_q16(lut, v1); t2 += v1; }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        a0 += __shfl_down_sync(0xffffffffu, a0, o); a1 += __shfl_down_sync(0xffffffffu, a1, o);
        a2 += __shfl_down_sync(0xffffffffu, a2, o); t0 += __shfl_down_sync(0xffffffffu, t0, o);
        t1 += __shfl_down_sync(0xffffffffu, t1, o); t2 += __shfl_down_sync(0xffffffffu, t2, o);
      }
      if (lane == 0) {
        s_part[0][wid] = a0; s_part[1][wid] = a1; s_part[2][wid] = a2;
        s_cnt[0][wid] = t0; s_cnt[1][wid] = t1; s_cnt[2][wid] = t2;
      }
      __syncthreads();
      if (threadIdx.x < 3) {
        const uint32_t q = threadIdx.x;
        uint64_t a = 0;
        uint32_t t = 0;
        for (int w = 0; w < SPLIT_WARPS; ++w) { a += s_part[q][w]; t += s_cnt[q][w]; }
        s_e[q][0] = bits_entropy_q16(a, t, lut);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t bs = take < c.min_block ? c.min_block : take;
      uint32_t old_types = st.num_types;
      SplitAction act = split_decide(st, nctx, c.max_types, (uint64_t)c.thr_bits << 16, c.min_block, s_e[0], s_e[1], s_e[2]);
      s_action = (int)act;
      uint32_t b = s_nblocks;
      if (act == SPLIT_FIRST) { c.types[b] = 0; c.lengths[b] = bs; s_nblocks = b + 1; s_new_type = 0; }
      else if (act == SPLIT_NEW_TYPE) { c.types[b] = (uint8_t)old_types; c.lengths[b] = bs; s_nblocks = b + 1; s_new_type = old_types; }
      else if (act == SPLIT_SECOND_LAST) { c.types[b] = (uint8_t)st.last_type[0]; c.lengths[b] = bs; s_nblocks = b + 1; }
      else { c.lengths[b - 1] += bs; }
    }
    __syncthreads();
    {
      const int act = s_action;
      const uint32_t ic = s_ic, i0 = s_i0, i1 = s_i1;
      if (act == SPLIT_FIRST || act == SPLIT_NEW_TYPE) {
        // the pending histogram becomes block type s_new_type: write it through, rotate the roles, take a free buffer
        uint32_t* g = c.hist + (size_t)s_new_type * HA;
        const uint32_t ni1 = act == SPLIT_FIRST ? ic : i0, ni0 = ic;
        uint32_t nic = 0;
        while (nic == ni0 || nic == ni1) ++nic;
        uint32_t* np = s_hist3 + nic * HA;
        for (uint32_t i = threadIdx.x; i < HA; i += SPLIT_THREADS) { g[i] = cur[i]; np[i] = 0; }
        __syncthreads();
        if (threadIdx.x == 0) { s_ic = nic; s_i0 = ni0; s_i1 = ni1; }
      } else {
        // merge the pending histogram into the (new) last type: after SPLIT_SECOND_LAST that is the old second-last
        const uint32_t ni0 = act == SPLIT_SECOND_LAST ? i1 : i0, ni1 = act == SPLIT_SECOND_LAST ? i0 : i1;
        uint32_t* dst = s_hist3 + ni0 * HA;
        uint32_t* g = c.hist + (size_t)st.last_type[0] * HA;
        for (uint32_t i = threadIdx.x; i < HA; i += SPLIT_THREADS) {
          const uint32_t v = dst[i] + cur[i];
          dst[i] = v; g[i] = v; cur[i] = 0;
        }
        __syncthreads();
        if (threadIdx.x == 0) { s_i0 = ni0; s_i1 = ni1; }
      }
    }
    __syncthreads();
    if (is_final) break;
  }
  if (threadIdx.x == 0) {
    uint32_t acc = 0;
    for (uint32_t b = 0; b < s_nblocks; ++b) { c.starts[b] = acc; acc += c.lengths[b]; }
    c.counts[0] = s_nblocks;
    c.counts[1] = st.num_types;
  }
}

// ---------------------------------------------------------------------------------------------------
// Header.  k_trees: one warp (lane 0) per prefix code of a metablock -- count smoothing, length-limited Huffman
// tree, canonical codes, serialised code description into a private slot.  k_header: one warp per metablock writes
// the metablock prologue (block-split codes, context maps) and splices the per-tree descriptions behind it.
// ---------------------------------------------------------------------------------------------------
#define TREE_SLOT_BYTES 1536
// header sections that depend only on the block splits are serialised by extra blocks of k_trees, concurrently with
// the prefix codes: 0..2 block-split codes (literal, command, distance), 3 literal context map, 4 distance context map
#define HDR_SECTIONS 5
#define SECT_BYTES 65536  // worst case: 16384 context-map symbols of <= 21 bits + their prefix code

// Warp-cooperative front end of huff_code_lengths(): the used symbols are compacted into ws->key with ballots and sorted by a
// bitonic network over shared memory (keys are unique, so any correct sort gives the order of the sequential specification);
// the two-queue merge and the depth sweep then run on lane 0.  Must be called by the whole warp.  Returns the number of used symbols.
__device__ __forceinline__ uint32_t huff_sorted_keys_warp(const uint32_t* counts, uint32_t length, uint64_t* keys /* smem, 1024 */) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t FULL = 0xffffffffu;
  uint32_t n = 0;
  for (uint32_t base = 0; base < length; base += 32) {
    const uint32_t i = base + lane;
    const uint32_t c = i < length ? counts[i] : 0u;
    const uint32_t bal = __ballot_sync(FULL, c != 0);
    if (c) keys[n + __popc(bal & ((1u << lane) - 1u))] = ((uint64_t)c << 16) | i;
    n += __popc(bal);
  }
  if (n < 2) { __syncwarp(); return n; }
  uint32_t np = 1;
  while (np < n) np <<= 1;
  for (uint32_t i = n + lane; i < np; i += 32) keys[i] = ~0ull;
  __syncwarp();
  for (uint32_t k = 2; k <= np; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t t = lane; t < (np >> 1); t += 32) {
        const uint32_t lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // index with bit j clear
        const uint32_t hi = lo | j;
        const bool up = (lo & k) == 0;
        const uint64_t a = keys[lo], b = keys[hi];
        if ((a > b) == up) { keys[lo] = b; keys[hi] = a; }
      }
      __syncwarp();
    }
  }
  return n;
}

__global__ void __launch_bounds__(32) k_trees(Workspace W) {
  __shared__ HuffWs ws_s;  // code construction / serialisation scratch in shared memory: the serial parts are latency bound
  __shared__ uint8_t s_depth[704];
  __shared__ uint16_t s_code[704];
  __shared__ uint32_t s_hist[704];
  const uint32_t m = blockIdx.y;
  const uint32_t lane = threadIdx.x;
  const MBDesc& mb = W.mb[m];
  const uint32_t nctx = ctxmap_num_contexts(mb.ctx_map_id);
  const uint32_t* cnt = W.split_counts + (size_t)m * 6;
  const bool full = mb.ctx_map_id >= CTXMAP_FULL_UTF8;  // quality >= 10: codes = clusters of the context maps
  const uint32_t nlit = full ? W.cm_counts[(size_t)m * 2] : cnt[1] * nctx, ncmd = cnt[3], ndist = full ? W.cm_counts[(size_t)m * 2 + 1] : cnt[5];
  uint32_t t = blockIdx.x;
  const uint32_t tree_cap_total = W.max_lit_trees + W.max_cmd_types + W.max_dist_types;
  if (t >= tree_cap_total) {  // header section (serial code, one lane)
    const uint32_t k = t - tree_cap_total;
    if (lane != 0 || k >= HDR_SECTIONS) return;
    BitWriter sw;
    sw.init(W.sect_bits + ((size_t)m * HDR_SECTIONS + k) * SECT_BYTES);
    SplitCode* sc = W.split_codes + (size_t)m * 3;
    if (k < 3) {
      SplitView v = make_view(W, m, (int)k);
      store_block_split_code(sw, v, sc + k, &ws_s);
    } else if (k == 3) {
      uint32_t* rle = W.ctxmap_ws + (size_t)m * (256 * 64 + 1024);
      if (full) store_context_map(sw, W.lit_cmap + (size_t)m * 256 * 64, cnt[1] << 6, nlit, rle, &ws_s);
      else if (mb.ctx_map_id == CTXMAP_NONE) store_trivial_context_map(sw, cnt[1], 6, &ws_s);
      else store_static_literal_context_map(sw, cnt[1], mb.ctx_map_id, rle, &ws_s);
    } else {
      if (full) store_context_map(sw, W.dist_cmap + (size_t)m * 256 * 4, cnt[5] << 2, ndist, W.ctxmap_ws + (size_t)m * (256 * 64 + 1024) + 256 * 64, &ws_s);
      else store_trivial_context_map(sw, cnt[5], 2, &ws_s);
    }
    sw.flush_partial();
    W.sect_nbits[(size_t)m * HDR_SECTIONS + k] = (uint32_t)sw.bit_pos();
    return;
  }
  if (t >= nlit + ncmd + ndist) return;
  const uint32_t slot = t;
  uint32_t* hist; uint8_t* depth; uint16_t* code; uint32_t A, alphabet = 0;
  if (t < nlit) {
    A = 256; hist = W.lit_hist + ((size_t)m * (W.max_lit_trees + 13) + t) * 256;
    depth = W.lit_depth + ((size_t)m * W.max_lit_trees + t) * 256; code = W.lit_code + ((size_t)m * W.max_lit_trees + t) * 256;
  } else if (t < nlit + ncmd) {
    t -= nlit; A = 704; hist = W.cmd_hist + ((size_t)m * (W.max_cmd_types + 1) + t) * 704;
    depth = W.cmd_depth + ((size_t)m * W.max_cmd_types + t) * 704; code = W.cmd_code + ((size_t)m * W.max_cmd_types + t) * 704;
  } else {
    t -= nlit + ncmd; A = W.dist_A; hist = W.dist_hist + ((size_t)m * (W.max_dist_types + 1) + t) * A;
    depth = W.dist_depth + ((size_t)m * W.max_dist_types + t) * A; code = W.dist_code + ((size_t)m * W.max_dist_types + t) * A;
    alphabet = distance_alphabet_size(mb.dist_params & 0xFFu, mb.dist_params >> 8);  // symbol width of the simple / one-symbol forms
  }
  const uint32_t tree_cap = W.max_lit_trees + W.max_cmd_types + W.max_dist_types;
  // == huff_build_and_store() with the sort done by the whole warp; everything is worked on in shared memory: the merge, the
  // smoothing scan and the run-length coding are chains of dependent accesses ==
  for (uint32_t i = lane; i < A; i += 32) { s_hist[i] = hist[i]; s_depth[i] = 0; s_code[i] = 0; }
  __syncwarp();
  if (lane == 0) huff_smooth_counts(A, s_hist);
  __syncwarp();
  uint32_t max_bits = 0;
  for (uint32_t c = (alphabet ? alphabet : A) - 1; c; c >>= 1) ++max_bits;
  const uint32_t used = huff_sorted_keys_warp(s_hist, A, ws_s.key);
  BitWriter bw;
  bw.init(W.tree_bits + ((size_t)m * tree_cap + slot) * TREE_SLOT_BYTES);
  if (lane == 0) {
    if (used <= 1) {
      bw.put(4, 1);
      bw.put(max_bits, used ? (uint32_t)(ws_s.key[0] & 0xFFFFu) : 0u);
    } else {
      huff_lengths_sorted(&ws_s, used, 15, s_depth);
      huff_depths_to_codes(s_depth, A, s_code);
      if (used > 4) huff_store_complex(bw, s_depth, A, &ws_s);
      else {  // simple code: symbols by code length, then by value (ws_s.key is sorted by count, so re-derive from the alphabet)
        uint32_t first4[4] = {0, 0, 0, 0}, k = 0;
        for (uint32_t i = 0; i < A && k < used; ++i) if (s_hist[i]) first4[k++] = i;
        for (uint32_t i = 1; i < used; ++i) {
          const uint32_t v = first4[i];
          uint32_t j = i;
          for (; j > 0 && s_depth[first4[j - 1]] > s_depth[v]; --j) first4[j] = first4[j - 1];
          first4[j] = v;
        }
        bw.put(2, 1);
        bw.put(2, used - 1);
        for (uint32_t i = 0; i < used; ++i) bw.put(max_bits, first4[i]);
        if (used == 4) bw.put(1, s_depth[first4[0]] == 1 ? 1u : 0u);
      }
    }
    bw.flush_partial();
    W.tree_nbits[(size_t)m * tree_cap + slot] = (uint32_t)bw.bit_pos();
  }
  __syncwarp();
  for (uint32_t i = lane; i < A; i += 32) { depth[i] = s_depth[i]; code[i] = s_code[i]; }
}

__device__ __forceinline__ void append_bits(BitWriter& bw, const uint8_t* src, uint32_t nbits) {
  uint32_t i = 0;
  for (; i + 32 <= nbits; i += 32) {
    uint32_t v = (uint32_t)src[i >> 3] | ((uint32_t)src[(i >> 3) + 1] << 8) | ((uint32_t)src[(i >> 3) + 2] << 16) |
                 ((uint32_t)src[(i >> 3) + 3] << 24);
    bw.put(32, v);
  }
  for (; i < nbits; i += 8) {
    uint32_t n = nbits - i < 8 ? nbits - i : 8;
    bw.put(n, src[i >> 3] & ((1u << n) - 1u));
  }
}

// k_header: lane 0 writes the metablock prologue and the block-split / context-map sections, then the whole warp splices the
// per-code descriptions behind them at bit granularity (32-bit chunks, atomicOr into the zeroed tail of the header buffer).
__global__ void __launch_bounds__(32) k_header(Workspace W) {
  const uint32_t m = blockIdx.x;
  const uint32_t lane = threadIdx.x;
  MBDesc& mb = W.mb[m];
  const uint32_t nctx = ctxmap_num_contexts(mb.ctx_map_id);
  SplitView lv = make_view(W, m, 0), cv = make_view(W, m, 1), dv = make_view(W, m, 2);
  uint8_t* hdr = W.hdr + (size_t)m * W.hdr_cap;
  uint64_t pos = 0;
  if (lane == 0) {
    BitWriter bw;
    bw.init(hdr);
    store_compressed_metablock_header(bw, false, mb.len);
    const uint8_t* sect = W.sect_bits + (size_t)m * HDR_SECTIONS * SECT_BYTES;
    const uint32_t* snb = W.sect_nbits + (size_t)m * HDR_SECTIONS;
    for (uint32_t k = 0; k < 3; ++k) append_bits(bw, sect + (size_t)k * SECT_BYTES, snb[k]);  // block-split codes
    bw.put(2, mb.dist_params & 0xFFu);                               // NPOSTFIX
    bw.put(4, (mb.dist_params >> 8) >> (mb.dist_params & 0xFFu));    // NDIRECT >> NPOSTFIX
    for (uint32_t i = 0; i < lv.num_types; ++i) bw.put(2, mb.ctx_map_id == CTXMAP_FULL_SIGNED ? 3 : 2);  // CONTEXT_SIGNED / CONTEXT_UTF8
    append_bits(bw, sect + (size_t)3 * SECT_BYTES, snb[3]);  // literal context map
    append_bits(bw, sect + (size_t)4 * SECT_BYTES, snb[4]);  // distance context map
    bw.flush_partial();
    pos = bw.bit_pos();
  }
  pos = __shfl_sync(0xffffffffu, pos, 0);
  const uint32_t tree_cap = W.max_lit_trees + W.max_cmd_types + W.max_dist_types;
  const bool full = mb.ctx_map_id >= CTXMAP_FULL_UTF8;
  const uint32_t ntrees = (full ? W.cm_counts[(size_t)m * 2] : lv.num_types * nctx) + cv.num_types + (full ? W.cm_counts[(size_t)m * 2 + 1] : dv.num_types);
  const uint32_t* tnb = W.tree_nbits + (size_t)m * tree_cap;
  uint64_t total = 0;
  for (uint32_t t = lane; t < ntrees; t += 32) total += tnb[t];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
  // zero everything behind the prologue's last (partial) byte up to the end of the spliced region, word by word
  {
    const uint64_t first_byte = (pos + 7) >> 3, last_byte = ((pos + total + 7) >> 3) + 8;
    for (uint64_t i = first_byte + lane; i < ((first_byte + 3) & ~3ull); i += 32) hdr[i] = 0;
    uint32_t* hw = reinterpret_cast<uint32_t*>(hdr);
    for (uint64_t w = ((first_byte + 3) >> 2) + lane; w < (last_byte + 3) >> 2; w += 32) hw[w] = 0;
  }
  __syncwarp();
  uint32_t* hw = reinterpret_cast<uint32_t*>(hdr);
  for (uint32_t t = 0; t < ntrees; ++t) {
    const uint32_t nb = tnb[t];
    const uint8_t* src = W.tree_bits + ((size_t)m * tree_cap + t) * TREE_SLOT_BYTES;
    for (uint32_t c = lane; c * 32 < nb; c += 32) {
      const uint32_t left = nb - c * 32;
      uint32_t v = (uint32_t)src[c * 4] | ((uint32_t)src[c * 4 + 1] << 8) | ((uint32_t)src[c * 4 + 2] << 16) | ((uint32_t)src[c * 4 + 3] << 24);
      if (left < 32) v &= (1u << left) - 1u;
      const uint64_t bp = pos + (uint64_t)c * 32;
      const uint32_t sh = (uint32_t)(bp & 31);
      atomicOr(&hw[bp >> 5], v << sh);
      if (sh) atomicOr(&hw[(bp >> 5) + 1], v >> (32 - sh));
    }
    pos += nb;
  }
  __syncwarp();
  if (lane == 0) mb.hdr_bits = (uint32_t)pos;
}

// ---------------------------------------------------------------------------------------------------
// Emission.
// ---------------------------------------------------------------------------------------------------
// k_bitlen: exact bit length of every command + exclusive prefix inside its 256-command tile; tile totals go to
// cmd_tile[]; k_bitscan turns the (few) tile totals of a metablock into tile offsets.
__global__ void __launch_bounds__(256) k_bitlen(Workspace W) {
  __shared__ uint32_t s_warp[8];
  const uint32_t m = blockIdx.y;
  const MBDesc& mb = W.mb[m];
  if (blockIdx.x * 256u >= mb.ncmd) return;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t bits = 0;
  if (i < mb.ncmd) {
    const MetaCodes mc = make_codes(W, m);
    const GCmd g = W.cmds[(size_t)m * W.cmd_cap + i];
    CountWriter w;
    w.bits = 0;
    const uint32_t lb = g.insert_len > LONG_INS ? W.long_tab[(size_t)m * W.long_cap + (g.pos - mb.start) / LONG_INS].y : NOT_LONG;
    emit_command(w, mc, g.as_cmd(), i, g.lit_idx, g.dist_idx + W.unit_dist_off[g.pad], W.data, g.pos, W.P.abs_base, lb);
    bits = (uint32_t)w.bits;
  }
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = bits;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= (uint32_t)o) x += y;
  }
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  uint32_t woff = 0;
  for (uint32_t w = 0; w < wid; ++w) woff += s_warp[w];
  if (i < mb.ncmd) W.cmd_bits[(size_t)m * W.cmd_cap + i] = woff + x - bits;
  if (threadIdx.x == 255) W.cmd_tile[(size_t)m * W.tile_cap + blockIdx.x] = woff + x;
}
// One CTA per metablock: exclusive scan of the tile totals (64-bit running sum), total -> body_bits.
__global__ void __launch_bounds__(1024) k_bitscan(Workspace W) {
  __shared__ uint32_t s_warp[33];
  const uint32_t m = blockIdx.x;
  MBDesc& mb = W.mb[m];
  const uint32_t ntiles = (mb.ncmd + 255) / 256;
  uint32_t* tiles = W.cmd_tile + (size_t)m * W.tile_cap;
  uint64_t run = 0;
  for (uint32_t base = 0; base < ntiles; base += 1024) {
    uint32_t i = base + threadIdx.x;
    uint32_t v = i < ntiles ? tiles[i] : 0;
    uint32_t tot;
    uint32_t ex = block_excl_scan_1024(v, s_warp, &tot);
    if (i < ntiles) tiles[i] = (uint32_t)(run + ex);  // the body of a metablock stays below 2^32 bits
    run += tot;
  }
  if (threadIdx.x == 0) mb.body_bits = run;
}

struct AtomicOrWriter {
  uint32_t* out;
  uint64_t word;
  uint64_t acc;
  uint32_t nacc;
  __device__ __forceinline__ void init(uint32_t* o, uint64_t bitpos) { out = o; word = bitpos >> 5; nacc = (uint32_t)(bitpos & 31); acc = 0; }
  __device__ __forceinline__ void put(uint32_t n, uint64_t v) {
    acc |= v << nacc;
    nacc += n;
    if (nacc >= 32) {
      atomicOr(&out[word++], (uint32_t)acc);
      acc >>= 32;
      nacc -= 32;
    }
  }
  __device__ __forceinline__ void flush() { if (nacc) atomicOr(&out[word], (uint32_t)acc); }
  __device__ __forceinline__ void skip(uint32_t n) {
    flush();
    init(out, word * 32 + nacc + n);
  }
};

// Single thread: raw/compressed decision per metablock, stream layout, stream header / trailer / padding bits.
__global__ void k_layout(Workspace W, int first, int last, int byte_align, uint64_t* total_after) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const EncParams& P = W.P;
  uint64_t pos = *W.total_bits;
  if (first) {
    AtomicOrWriter w;
    w.init(W.out, pos);
    if (P.lgwin == 16) { w.put(1, 0); pos += 1; }
    else if (P.lgwin == 17) { w.put(7, 1); pos += 7; }
    else if (P.lgwin > 17) { w.put(4, (uint64_t)(((P.lgwin - 17) << 1) | 1)); pos += 4; }
    else { w.put(7, (uint64_t)(((P.lgwin - 8) << 4) | 1)); pos += 7; }
    w.flush();
  }
  for (uint32_t m = 0; m < W.num_mb; ++m) {
    MBDesc& mb = W.mb[m];
    uint64_t comp_bits = (uint64_t)mb.hdr_bits + mb.body_bits;
    uint64_t raw_hdr = raw_metablock_header_bits(mb.len);
    uint64_t raw_bits = ((pos + raw_hdr + 7) & ~7ull) - pos + 8ull * mb.len;
    mb.raw = comp_bits > raw_bits ? 1u : 0u;
    mb.out_bitpos = pos;
    pos += mb.raw ? raw_bits : comp_bits;
  }
  if (last) {
    AtomicOrWriter t;
    t.init(W.out, pos);
    t.put(2, 3);  // ISLAST = 1, ISLASTEMPTY = 1
    t.flush();
    pos += 2;
  } else if (byte_align && (pos & 7)) {
    AtomicOrWriter t;  // empty metadata metablock (brotli_bit_stream.rs:2840-2845), then zero padding
    t.init(W.out, pos);
    t.put(6, 6);
    t.flush();
    pos = (pos + 6 + 7) & ~7ull;
  }
  *W.total_bits = pos;
  *total_after = pos;  // per-chunk copy: the host reads it while later chunks keep advancing total_bits
}

// Single thread, last launch of a stream-ordered call: the byte size of the range's output, from the end bit position of its last
// chunk (end_bits), or -- a call without chunks -- of the empty stream (encode.rs:1463-1467: one byte 6) or of nothing.
// trailer >= 0: one more byte behind the (byte-aligned) end, the ISLAST + ISLASTEMPTY byte of a byte-aligned framed stream.
__global__ void k_out_size(const uint64_t* end_bits, uint8_t* out, int empty_stream, uint64_t* out_size, int trailer) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (end_bits) {
    uint64_t n = (*end_bits + 7) >> 3;
    if (trailer >= 0) out[n++] = (uint8_t)trailer;
    *out_size = n;
    return;
  }
  if (empty_stream) out[0] = 6;
  *out_size = empty_stream ? 1 : 0;
}

// Single thread: the host-built prologue of a framed stream (B200Prologue, bro_capi.cu:write_prologue) into out, its data bytes
// (the first n2 input bytes of a catable stream) taken from `in`.  Then either the chunks continue behind it (total_bits = its
// bit length, so k_layout of the first chunk starts there) or, when it is the whole stream, its size goes to out_size.
__global__ void k_prologue(B200Prologue pro, const uint8_t* in, uint8_t* out, uint64_t* total_bits, uint64_t* out_size) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  for (uint32_t i = 0; i < pro.len; ++i) out[i] = pro.bytes[i];
  for (uint32_t i = 0; i < pro.n2; ++i) out[pro.data_off + i] = in[i];
  if (total_bits) *total_bits = 8ull * pro.len;
  if (out_size) *out_size = pro.len;
}

__global__ void __launch_bounds__(256) k_emit_header(Workspace W) {
  const uint32_t m = blockIdx.x;
  const MBDesc& mb = W.mb[m];
  if (mb.raw) return;
  const uint8_t* h = W.hdr + (size_t)m * W.hdr_cap;
  const uint32_t nbytes = (mb.hdr_bits + 7) / 8;
  // hdr_cap is a multiple of 4 and the buffer is zero beyond hdr_bits within the last byte
  for (uint32_t i = threadIdx.x; i * 4 < nbytes; i += blockDim.x) {
    uint32_t v = 0;
    for (uint32_t k = 0; k < 4; ++k) {
      uint32_t idx = i * 4 + k;
      uint32_t byte = idx < nbytes ? h[idx] : 0u;
      if (idx == nbytes - 1 && (mb.hdr_bits & 7)) byte &= (1u << (mb.hdr_bits & 7)) - 1u;
      v |= byte << (8 * k);
    }
    if (v == 0) continue;
    uint64_t bitpos = mb.out_bitpos + (uint64_t)i * 32;
    uint64_t word = bitpos >> 5;
    uint32_t sh = (uint32_t)(bitpos & 31);
    atomicOr(&W.out[word], v << sh);
    if (sh) atomicOr(&W.out[word + 1], v >> (32 - sh));
  }
}
__global__ void __launch_bounds__(256) k_emit_body(Workspace W) {
  const uint32_t m = blockIdx.y;
  const MBDesc& mb = W.mb[m];
  if (mb.raw) return;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= mb.ncmd) return;
  const MetaCodes mc = make_codes(W, m);
  const GCmd g = W.cmds[(size_t)m * W.cmd_cap + i];
  AtomicOrWriter w;
  w.init(W.out, mb.out_bitpos + mb.hdr_bits + W.cmd_tile[(size_t)m * W.tile_cap + (i >> 8)] + W.cmd_bits[(size_t)m * W.cmd_cap + i]);
  const uint32_t lb = g.insert_len > LONG_INS ? W.long_tab[(size_t)m * W.long_cap + (g.pos - mb.start) / LONG_INS].y : NOT_LONG;
  emit_command(w, mc, g.as_cmd(), i, g.lit_idx, g.dist_idx + W.unit_dist_off[g.pad], W.data, g.pos, W.P.abs_base, lb);
  w.flush();
}
// The literals of long inserts: CTA per segment, bit offsets from a block scan.
__global__ void __launch_bounds__(256) k_emit_long(Workspace W) {
  __shared__ uint32_t s_warp[9];
  __shared__ uint64_t s_base;
  const uint32_t m = blockIdx.y;
  const MBDesc& mb = W.mb[m];
  if (mb.raw) return;
  const MetaCodes mc = make_codes(W, m);
  for_each_long_segment(W, [&](uint32_t ci, const GCmd& g, uint32_t slot, uint32_t k) {
    uint32_t before = 0;  // literal bits of the segments in front of this one
    for (uint32_t j = threadIdx.x; j < k; j += 256) before += W.seg_bits[(size_t)m * W.long_cap + slot + j];
    uint32_t tot;
    block_excl_scan_256(before, s_warp, &tot);
    if (threadIdx.x == 0) {
      CountWriter h;
      h.bits = 0;
      emit_command_head(h, mc, g.as_cmd(), ci);
      s_base = mb.out_bitpos + mb.hdr_bits + W.cmd_tile[(size_t)m * W.tile_cap + (ci >> 8)] + W.cmd_bits[(size_t)m * W.cmd_cap + ci] + h.bits + tot;
    }
    const uint32_t off = k * LONG_INS + 2 * threadIdx.x;
    CountWriter c;
    c.bits = 0;
    for (uint32_t j = off; j < min(g.insert_len, off + 2); ++j) emit_one_literal(c, mc, g.lit_idx + j, W.data, g.pos + j, W.P.abs_base);
    const uint32_t ex = block_excl_scan_256((uint32_t)c.bits, s_warp, &tot);  // (also orders s_base)
    if (c.bits) {
      AtomicOrWriter w;
      w.init(W.out, s_base + ex);
      for (uint32_t j = off; j < min(g.insert_len, off + 2); ++j) emit_one_literal(w, mc, g.lit_idx + j, W.data, g.pos + j, W.P.abs_base);
      w.flush();
    }
    __syncthreads();
  });
}
__global__ void __launch_bounds__(256) k_emit_raw(Workspace W) {
  const uint32_t m = blockIdx.y;
  const MBDesc& mb = W.mb[m];
  if (!mb.raw) return;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    AtomicOrWriter w;
    w.init(W.out, mb.out_bitpos);
    uint32_t lg = mb.len == 1 ? 1u : log2_floor_nz(mb.len - 1) + 1u;
    uint32_t mnibbles = (lg < 16 ? 16u : lg + 3u) / 4u;
    w.put(1, 0);
    w.put(2, mnibbles - 4);
    w.put(mnibbles * 4, mb.len - 1);
    w.put(1, 1);
    w.flush();
  }
  const uint64_t byte0 = (mb.out_bitpos + raw_metablock_header_bits(mb.len) + 7) >> 3;
  uint8_t* ob = reinterpret_cast<uint8_t*>(W.out);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < mb.len; i += gridDim.x * blockDim.x)
    ob[byte0 + i] = W.data[mb.start + i];
}

}  // namespace bro

// bro_encoder.cu -- host orchestration of the GPU brotli compression path and its C ABI.
//
// One Encoder object = one GPU + one CUDA stream + a reusable device workspace.  A stream is compressed as a
// sequence of independent ranges ("chunks", <= 128 MiB) whose match search sees a left halo of the previous
// 2^lgwin bytes; every chunk runs  sort -> match -> parse -> finalise -> context -> symbols -> split -> header ->
// bit lengths -> layout -> emit  entirely on the device and appends its metablocks at the running bit position.
// No stage has a CPU fallback: if CUDA is unavailable every entry point fails.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "bro_kernels.cuh"
#include "bro_kernels_hq.cuh"
#include "bro_encoder.h"
#include "bro_dict_data.inc"  // generated at build time by gen_dict.py: kDictData, kDictHash

using namespace bro;

#define CUDA_OK(x)                                                                                   \
  do {                                                                                               \
    cudaError_t e_ = (x);                                                                            \
    if (e_ != cudaSuccess) {                                                                         \
      fprintf(stderr, "[brotli_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      return false;                                                                                  \
    }                                                                                                \
  } while (0)

namespace {

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  bool frozen = false;  // a captured CUDA graph points into the buffer: it may not be freed or moved
  bool ensure(size_t bytes) {
    if (bytes <= cap) return true;
    if (frozen) {
      fprintf(stderr, "[brotli_b200] workspace frozen by a CUDA graph capture cannot grow to %zu bytes\n", bytes);
      return false;
    }
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + (bytes >> 4) + 4096;
    if (cudaMalloc(&p, want) != cudaSuccess) {
      fprintf(stderr, "[brotli_b200] cudaMalloc(%zu) failed\n", want);
      return false;
    }
    cap = want;
    return true;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

constexpr uint32_t kPad = 512;                 // zero bytes after the input
constexpr uint32_t kChunk = BRO_CHUNK_BYTES;   // bytes per pipeline pass (one sort batch for lgwin <= 22)
constexpr uint32_t kBatchMax = 1u << 25;       // positions per sort batch (25-bit packed positions)
constexpr uint32_t kLookahead = 4096;          // input bytes past a chunk's end that must be resident before it runs
constexpr int kMaxLanes = 6;
static_assert((kBatchMax >> BEST_SLAB_BITS) <= BEST_MAX_SLABS, "a batch has more best[] slabs than cursors");

struct EventPool {
  std::vector<cudaEvent_t> ev;
  size_t used = 0;
  cudaEvent_t get(bool timing) {
    (void)timing;
    if (used == ev.size()) {
      cudaEvent_t e;
      cudaEventCreateWithFlags(&e, timing ? cudaEventDefault : cudaEventDisableTiming);
      ev.push_back(e);
    }
    return ev[used++];
  }
  void reserve(size_t n) {  // untimed events, so that a call inside a graph capture creates none
    while (ev.size() < n) {
      cudaEvent_t e;
      if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return;
      ev.push_back(e);
    }
  }
  void reset() { used = 0; }
  void destroy() { for (auto& e : ev) cudaEventDestroy(e); ev.clear(); used = 0; }
};

// One lane = one stream + the per-chunk workspace.  Consecutive chunks alternate between lanes so that the
// latency-bound stages of one chunk (block splitting, Huffman trees, layout) overlap the throughput-bound stages of
// the next one (sort, match, parse) and the host<->device copies.
struct Lane {
  cudaStream_t stream = nullptr;
  DevBuf arena;     // every region of the chunk workspace (layout_chunk)
  Workspace W{};    // the last chunk's workspace: the stage hooks read their results through it
  const uint32_t* slab_cursor = nullptr;  // the last chunk's last sort batch, when its best[] went through match_store:
  uint32_t slab_payload = 0;              //   its slab cursors and payload size (b200_stage_match_slabs)
  EventPool marks;  // timing marks: (event, stage that starts there); -1 ends the last stage
  std::vector<int> mark_stage;
  void release() {
    arena.release();
    marks.destroy();
    if (stream) cudaStreamDestroy(stream);
    stream = nullptr;
  }
};

// Hands out the regions of a lane's workspace from one allocation.  Pass 1 (base == nullptr) only sizes the layout, pass 2
// returns pointers into the arena.  Every region starts 256-byte aligned and is followed by a kGuard-byte gap, so that a small
// overrun lands in the gap instead of in the next region.  No region carries data from one chunk to the next: each chunk
// writes (or clears) a region before it reads it, so the layout may differ from chunk to chunk.
constexpr size_t kGuard = 4096;
struct Carve {
  uint8_t* base;
  size_t off = 0;
  template <class T> T* take(size_t count) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off = (off + count * sizeof(T) + kGuard + 255) & ~(size_t)255;
    return p;
  }
};

struct SortBufs {
  uint32_t *a, *b;  // ping-pong of the sort passes; the sorted positions land in b
  uint32_t* state;  // digit counts, tile counters and look-back words
};
// sort regions for batches of up to nb positions
SortBufs layout_sort(Carve& a, uint32_t nb) {
  SortBufs s;
  s.a = a.take<uint32_t>((size_t)nb + 16);  // (+ 64 bytes)
  s.b = a.take<uint32_t>((size_t)nb + 16);
  s.state = a.take<uint32_t>(sort_state_words((nb + SORT_TILE - 1) / SORT_TILE));
  return s;
}

// workspaces of the quality 10 / 11 histogram stage (BrotliSplitBlock + context-map clustering); W's capacities are set
void layout_hq_split(Carve& a, const EncParams& P, const Workspace& W, BsWs* B, CmWs* M) {
  const uint32_t NM = W.num_mb;
  const uint32_t mb_span = P.unit * P.mb_units;
  memset(B, 0, sizeof(*B));
  memset(M, 0, sizeof(*M));
  B->cap[0] = mb_span; B->cap[1] = W.cmd_cap; B->cap[2] = W.cmd_cap;
  B->maxb[0] = W.lit_blk_cap; B->maxb[1] = W.cmd_blk_cap; B->maxb[2] = W.dist_blk_cap;
  for (int i = 0; i < 3; ++i) B->segc[i] = B->cap[i] / BS_SEG + 1;
  B->cap_sum = B->cap[0] + B->cap[1] + B->cap[2];
  B->maxb_sum = B->maxb[0] + B->maxb[1] + B->maxb[2];
  B->segc_sum = B->segc[0] + B->segc[1] + B->segc[2];
  B->dist_A = W.dist_A;
  B->hist_stride = 100u * (256u + 704u + W.dist_A);
  B->bh_sum = B->maxb[0] * 256 + B->maxb[1] * 704 + B->maxb[2] * W.dist_A;
  B->nsurv_stride = std::max(B->maxb[0], std::max(B->maxb[1], B->maxb[2])) / 64 + 2;
  const size_t nb = (size_t)NM * B->maxb_sum;
  B->meta = a.take<BsMeta>((size_t)NM * 3);
  B->blockid = a.take<uint8_t>((size_t)NM * B->cap_sum + 64);
  B->signal = a.take<uint32_t>((size_t)NM * B->cap_sum * 4 + 16);  // (+ 64 bytes)
  B->hist = a.take<uint32_t>((size_t)NM * B->hist_stride);
  B->icost = a.take<uint32_t>((size_t)NM * B->hist_stride);
  B->firstpos = a.take<uint32_t>((size_t)NM * 3 * 128);
  B->fmap = a.take<uint8_t>((size_t)NM * B->segc_sum * 129);
  B->enter = B->fmap + (size_t)NM * B->segc_sum * 128;
  B->bstart = a.take<uint32_t>(nb + NM * 3 + 16);  // (+ 64 bytes)
  B->bh_in = a.take<uint32_t>((size_t)NM * B->bh_sum);
  B->bh_work = a.take<uint32_t>((size_t)NM * B->bh_sum);
  B->ccost = a.take<uint64_t>(nb * 2);
  B->bd = reinterpret_cast<int64_t*>(B->ccost + nb);
  B->csize = a.take<uint32_t>(nb * 4); B->hsym = B->csize + nb; B->clusters = B->hsym + nb; B->bj = B->clusters + nb;
  B->nsurv = a.take<uint32_t>((size_t)NM * 3 * B->nsurv_stride);
  const size_t nc = (size_t)NM * (CM_LIT_MAX + CM_DIST_MAX);
  const size_t hl = (size_t)NM * CM_LIT_MAX * 256, hd = (size_t)NM * CM_DIST_MAX * W.dist_A;
  M->in_lit = a.take<uint32_t>(hl + hd); M->in_dist = M->in_lit + hl;
  M->work_lit = a.take<uint32_t>(hl + hd); M->work_dist = M->work_lit + hl;
  M->cost = a.take<uint64_t>(nc * 2);
  M->bd = reinterpret_cast<int64_t*>(M->cost + nc);
  M->size = a.take<uint32_t>(nc * 4); M->sym = M->size + nc; M->clusters = M->sym + nc; M->bj = M->clusters + nc;
  M->nsurv = a.take<uint32_t>((size_t)NM * 2 * CM_NSURV_STRIDE);
  M->counts = W.cm_counts;
  M->lit_cmap = W.lit_cmap;
  M->dist_cmap = W.dist_cmap;
}

struct ChunkBufs {  // the regions of a chunk that Workspace does not point to
  SortBufs sort;
  uint2* stage;         // bucket depth 16 / 32: best[] records of a sort batch, slab-major (match_store)
  ZopfliArgs za;        // zopfli
  BsWs bs;              // hq_meta with hq_split
  CmWs cm;              //   "
  uint64_t* dist_cost;  //   "   [num_mb][64] cost of every (NPOSTFIX, NDIRECT)
};

// The workspace of one chunk of c bytes: W's capacities and every region of the lane's arena.  W and X start zeroed.
void layout_chunk(Carve& a, uint32_t c, const EncParams& P, Workspace* W, ChunkBufs* X) {
  const uint32_t mb_span = P.unit * P.mb_units;
  const uint32_t NU = (c + P.unit - 1) / P.unit;
  const uint32_t NM = (NU + P.mb_units - 1) / P.mb_units;
  const uint32_t cu = P.unit / 2 + 1;
  const uint32_t cmd_cap = mb_span / 2 + 2;
  const bool hq = P.zopfli, hq_split = P.hq_meta && P.hq_split;
  W->num_units = NU;
  W->num_mb = NM;
  W->cmd_cap = cmd_cap;
  W->lit_blk_cap = mb_span / 512 + 2;
  W->cmd_blk_cap = cmd_cap / 1024 + 2;
  W->dist_blk_cap = cmd_cap / 512 + 2;
  W->max_lit_trees = 256;
  W->max_cmd_types = 256;
  W->max_dist_types = 256;
  W->dist_A = hq_split ? BRO_DIST_A_MAX : 64u;
  W->hdr_cap = 384u << 10;
  W->tile_cap = cmd_cap / 256 + 2;
  W->long_cap = mb_span / LONG_INS + 1;
  if (!hq) {
    W->best = a.take<uint32_t>((size_t)c + 64);
    if (P.depth <= 32) X->stage = a.take<uint2>(c);  // a batch's payload is at most the chunk
  } else {
    W->hqm = a.take<HqMatch>(((size_t)c + 64) * HQ_MAXM);
    W->hqn = a.take<uint8_t>((size_t)c + 64);
    X->za.nodes = a.take<ZNode>((size_t)NU * (P.unit + 1));
    X->za.pre = a.take<uint32_t>((size_t)NU * (P.unit + 1));
    X->za.scratch = a.take<uint32_t>((size_t)NU * HQ_SCRATCH_WORDS);
  }
  W->raw = a.take<RawCmd>((size_t)NU * cu);
  uint32_t* up = a.take<uint32_t>((size_t)NU * 7);  // one [7][NU] block: b200_stage_hq copies the first three rows at once
  W->unit_ncmd = up; W->unit_tail = up + NU; W->unit_ncopy = up + 2 * (size_t)NU;
  W->unit_cmd_off = up + 3 * (size_t)NU; W->unit_lit_off = up + 4 * (size_t)NU; W->unit_ndist = up + 5 * (size_t)NU; W->unit_dist_off = up + 6 * (size_t)NU;
  W->cmds = a.take<GCmd>((size_t)NM * cmd_cap);
  W->cmd_bits = a.take<uint32_t>((size_t)NM * cmd_cap);
  W->cmd_tile = a.take<uint32_t>((size_t)NM * W->tile_cap);
  W->long_tab = a.take<uint2>((size_t)NM * W->long_cap);
  W->seg_bits = a.take<uint32_t>((size_t)NM * W->long_cap);
  W->lit_syms = a.take<uint16_t>((size_t)c + 64);
  W->cmd_syms = a.take<uint16_t>((size_t)NM * cmd_cap);
  W->dist_syms = a.take<uint16_t>((size_t)NM * cmd_cap);
  W->mb = a.take<MBDesc>(NM);
  const size_t blk_total = (size_t)W->lit_blk_cap + W->cmd_blk_cap + W->dist_blk_cap;
  uint8_t* t8 = a.take<uint8_t>((size_t)NM * blk_total);
  W->lit_types = t8; W->cmd_types = t8 + (size_t)NM * W->lit_blk_cap; W->dist_types = W->cmd_types + (size_t)NM * W->cmd_blk_cap;
  uint32_t* t32 = a.take<uint32_t>((size_t)NM * blk_total * 2);
  W->lit_lengths = t32; t32 += (size_t)NM * W->lit_blk_cap;
  W->lit_starts = t32; t32 += (size_t)NM * W->lit_blk_cap;
  W->cmd_lengths = t32; t32 += (size_t)NM * W->cmd_blk_cap;
  W->cmd_starts = t32; t32 += (size_t)NM * W->cmd_blk_cap;
  W->dist_lengths = t32; t32 += (size_t)NM * W->dist_blk_cap;
  W->dist_starts = t32;
  W->split_counts = a.take<uint32_t>((size_t)NM * 6);
  W->lit_hist = a.take<uint32_t>((size_t)NM * (W->max_lit_trees + 13) * 256);
  W->cmd_hist = a.take<uint32_t>((size_t)NM * (W->max_cmd_types + 1) * 704);
  W->dist_hist = a.take<uint32_t>((size_t)NM * (W->max_dist_types + 1) * W->dist_A);
  W->split_codes = a.take<SplitCode>((size_t)NM * 3);
  const size_t code_syms = (size_t)W->max_lit_trees * 256 + (size_t)W->max_cmd_types * 704 + (size_t)W->max_dist_types * W->dist_A;
  uint8_t* c8 = a.take<uint8_t>((size_t)NM * code_syms);
  W->lit_depth = c8; W->cmd_depth = c8 + (size_t)NM * W->max_lit_trees * 256;
  W->dist_depth = W->cmd_depth + (size_t)NM * W->max_cmd_types * 704;
  uint16_t* c16 = a.take<uint16_t>((size_t)NM * code_syms);
  W->lit_code = c16; W->cmd_code = c16 + (size_t)NM * W->max_lit_trees * 256;
  W->dist_code = W->cmd_code + (size_t)NM * W->max_cmd_types * 704;
  W->hdr = a.take<uint8_t>((size_t)NM * W->hdr_cap);
  W->ctxmap_ws = a.take<uint32_t>((size_t)NM * (256 * 64 + 1024));
  W->lit_cmap = a.take<uint8_t>((size_t)NM * (CM_LIT_MAX + CM_DIST_MAX));
  W->dist_cmap = W->lit_cmap + (size_t)NM * CM_LIT_MAX;
  W->cm_counts = a.take<uint32_t>((size_t)NM * 2);
  const size_t tree_cap = (size_t)W->max_lit_trees + W->max_cmd_types + W->max_dist_types;
  W->tree_bits = a.take<uint8_t>((size_t)NM * tree_cap * TREE_SLOT_BYTES);
  W->tree_nbits = a.take<uint32_t>((size_t)NM * tree_cap);
  W->sect_bits = a.take<uint8_t>((size_t)NM * HDR_SECTIONS * SECT_BYTES);
  W->sect_nbits = a.take<uint32_t>((size_t)NM * HDR_SECTIONS);
  X->sort = layout_sort(a, (uint32_t)std::min<uint64_t>((uint64_t)c + (1ull << P.lgwin) + 4096, kBatchMax));
  if (hq_split) {
    layout_hq_split(a, P, *W, &X->bs, &X->cm);
    X->dist_cost = a.take<uint64_t>((size_t)NM * 64);
  }
}

// bytes of lane arena a chunk of c bytes uses (the sizing pass of run_chunk)
size_t chunk_arena_bytes(const EncParams& P, uint32_t c) {
  Workspace W;
  ChunkBufs X;
  memset(&W, 0, sizeof(W));
  memset(&X, 0, sizeof(X));
  Carve sizing{nullptr};
  layout_chunk(sizing, c, P, &W, &X);
  return sizing.off;
}

// What one call compresses: its parameters, the span of the input that is staged on the device (the range and the window in
// front of it) and the range's chunks.
struct CallPlan {
  EncParams P;
  size_t base = 0, end = 0, staged = 0;  // absolute positions: staged = end - base bytes from base on
  size_t need = 0;                       // output bytes the chunks may touch (zeroed before they run)
  std::vector<std::pair<size_t, size_t>> chunks;  // (absolute start, length)
};

// The device memory and events a call uses, apart from the blocking path's d_out and pinned totals.
struct CallSizes {
  size_t data = 0, total = 0, events = 0, arena[kMaxLanes] = {};
  void cover(const CallSizes& o) {
    data = std::max(data, o.data);
    total = std::max(total, o.total);
    events = std::max(events, o.events);
    for (int i = 0; i < kMaxLanes; ++i) arena[i] = std::max(arena[i], o.arena[i]);
  }
};

bool on_device(const void* p, int device) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device;
}

}  // namespace

struct B200Encoder {
  int device = 0;
  bool ok = false;
  // configuration knobs (tests flip these)
  int ctx_model = 1, use_dict = 1, hq_split = 1, hq_levels = HQ_MAX_LEVELS;
  int q9_5 = 0;           // BROTLI_PARAM_Q9_5: quality 10 / 11 parse with the hash chains (default_enc_params)
  uint32_t hq_unit = 0;  // parse unit of the shortest-path parse (quality 10 / 11); 0 = 8 KiB at q10, 16 KiB at q11 (DESIGN.md)
  int num_lanes = 4;
  int ondemand = 1;       // q7..q9: search deep buckets where the parse stands (1) or for every position up front (0, A/B)
  Lane lanes[kMaxLanes];
  cudaStream_t s_in = nullptr, s_out = nullptr;  // copy streams
  DevBuf d_dict_words, d_dict_hash, d_dict_lutb, d_dict_lute, d_dict_trg, d_dict_tr;
  DevBuf d_data, d_lut, d_out, d_total;          // d_total: [0] running bit position, [1 + k] position after chunk k
  DevBuf d_probe;                                // b200_stage_match(search = 1): the on-demand search at every position
  uint32_t* od_probe = nullptr;                  // set only inside that hook: run_chunk launches k_od_probe into it
  uint64_t* h_total = nullptr;                   // pinned mirror of d_total[1 + k]
  size_t h_total_cap = 0;
  EventPool sync_events;
  cudaEvent_t ev_call = nullptr;  // end of the last stream-ordered call outside a capture: the next call starts behind it
  uint64_t data_base = 0;  // absolute stream position of d_data[0]
  float stage_ms[B200_NUM_STAGES];
  uint32_t launches = 0;
  bool timing = false;
  int num_sms = 0;

  bool init(int dev) {
    device = dev;
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
    // (descending stream priorities per lane, to stagger the chunks, were tried: slower than equal priority)
    for (auto& L : lanes) CUDA_OK(cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking));
    CUDA_OK(cudaStreamCreateWithFlags(&s_in, cudaStreamNonBlocking));
    CUDA_OK(cudaStreamCreateWithFlags(&s_out, cudaStreamNonBlocking));
    CUDA_OK(cudaEventCreateWithFlags(&ev_call, cudaEventDisableTiming));
    if (!d_lut.ensure(65536 * 4)) return false;
    std::vector<uint32_t> lut(65536);
    fill_log2_q16_lut(lut.data());
    CUDA_OK(cudaMemcpy(d_lut.p, lut.data(), 65536 * 4, cudaMemcpyHostToDevice));
    if (!d_dict_words.ensure(sizeof(kDictData) + 64) || !d_dict_hash.ensure(sizeof(kDictHash))) return false;
    CUDA_OK(cudaMemset(d_dict_words.p, 0, sizeof(kDictData) + 64));
    CUDA_OK(cudaMemcpy(d_dict_words.p, kDictData, sizeof(kDictData), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(d_dict_hash.p, kDictHash, sizeof(kDictHash), cudaMemcpyHostToDevice));
    if (!d_dict_lutb.ensure(sizeof(kDictLutBuckets)) || !d_dict_lute.ensure(sizeof(kDictLutEntries)) || !d_dict_trg.ensure(sizeof(kDictTrGroups)) ||
        !d_dict_tr.ensure(sizeof(kDictTransforms)))
      return false;
    CUDA_OK(cudaMemcpy(d_dict_lutb.p, kDictLutBuckets, sizeof(kDictLutBuckets), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(d_dict_lute.p, kDictLutEntries, sizeof(kDictLutEntries), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(d_dict_trg.p, kDictTrGroups, sizeof(kDictTrGroups), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(d_dict_tr.p, kDictTransforms, sizeof(kDictTransforms), cudaMemcpyHostToDevice));
    CUDA_OK(cudaDeviceSetLimit(cudaLimitStackSize, 4096));
    CUDA_OK(cudaFuncSetAttribute(k_split_greedy, cudaFuncAttributeMaxDynamicSharedMemorySize, SPLIT_SMEM_WORDS * 4));
    for (int i = 0; i < B200_NUM_STAGES; ++i) stage_ms[i] = 0;
    ok = true;
    return true;
  }
  void destroy() {
    cudaSetDevice(device);
    cudaDeviceSynchronize();
    for (auto& L : lanes) L.release();
    DevBuf* all[] = {&d_data, &d_lut, &d_out, &d_total, &d_probe, &d_dict_words, &d_dict_hash, &d_dict_lutb, &d_dict_lute, &d_dict_trg, &d_dict_tr};
    for (auto* b : all) b->release();
    if (h_total) cudaFreeHost(h_total);
    sync_events.destroy();
    if (ev_call) cudaEventDestroy(ev_call);
    if (s_in) cudaStreamDestroy(s_in);
    if (s_out) cudaStreamDestroy(s_out);
  }
  bool ensure_totals(size_t chunks) {
    if (!d_total.ensure((chunks + 2) * 8)) return false;
    if (chunks + 2 > h_total_cap) {
      if (h_total) cudaFreeHost(h_total);
      h_total = nullptr;
      h_total_cap = chunks + 64;
      CUDA_OK(cudaHostAlloc((void**)&h_total, h_total_cap * 8, cudaHostAllocDefault));
    }
    return true;
  }

  void fill_params(EncParams* P, int quality, int lgwin, uint64_t size_hint) const {
    default_enc_params(P, quality, lgwin, size_hint > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)size_hint, q9_5);
    P->ctx_model = ctx_model;
    P->use_dict = use_dict;
    P->hq_split = hq_split;
    if (P->zopfli) {
      P->hq_levels = hq_levels;
      if (hq_unit) {  // same metablock span
        const uint32_t span = P->unit * P->mb_units;
        P->unit = bmin(hq_unit, span);
        P->mb_units = span / P->unit;
      }
    }
  }

  void plan_call(CallPlan* c, int quality, int lgwin, uint64_t size_hint, size_t range_start, size_t range_len) const {
    fill_params(&c->P, quality, lgwin, size_hint);
    const size_t window = (size_t)1 << c->P.lgwin;
    c->base = range_start > window ? ((range_start - window) & ~(size_t)4095) : 0;
    c->end = range_start + range_len;
    c->staged = c->end - c->base;
    c->need = b200_max_compressed_size(range_len) + 64;
    c->chunks.clear();
    for (size_t done = 0; done < range_len;) {
      const size_t len = chunk_len_at(done, range_len);
      c->chunks.emplace_back(range_start + done, len);
      done += len;
    }
  }
  // chunk k runs on lane k % num_lanes; a call without chunks uses nothing
  CallSizes sizes_of(const CallPlan& c) const {
    CallSizes s;
    const size_t nchunks = c.chunks.size();
    if (!nchunks) return s;
    s.data = c.staged + kPad;
    s.total = (nchunks + 2) * 8;
    s.events = 3 * nchunks + kMaxLanes + 2;  // blocking: in / layout / done per chunk; async: in / layout per chunk, fork, joins
    for (size_t k = 0; k < nchunks; ++k) {
      size_t& a = s.arena[k % (size_t)num_lanes];
      a = std::max(a, chunk_arena_bytes(c.P, (uint32_t)c.chunks[k].second));
    }
    return s;
  }
  // Puts the buffers and events of s in place (grow), or only checks that they are (a call inside a graph capture may not
  // allocate).  Growing frees the old buffer, and cudaFree waits for the device.
  bool provide(const CallSizes& s, bool grow) {
    if (!grow) {
      if (d_data.cap < s.data || d_total.cap < s.total || sync_events.ev.size() < s.events) return false;
      for (int i = 0; i < kMaxLanes; ++i)
        if (lanes[i].arena.cap < s.arena[i]) return false;
      return true;
    }
    if (!d_data.ensure(s.data) || !d_total.ensure(s.total)) return false;
    for (int i = 0; i < kMaxLanes; ++i)
      if (!lanes[i].arena.ensure(s.arena[i])) return false;
    sync_events.reserve(s.events);
    return sync_events.ev.size() >= s.events;
  }
  // a captured graph holds pointers into these buffers from now on
  void freeze() {
    d_data.frozen = d_total.frozen = true;
    for (auto& L : lanes) L.arena.frozen = true;
  }

  // Enqueues on `stream` the stable sort of the batch positions 0..count-1 (input bytes at `data`, 4096-byte aligned and padded)
  // by the bucket key of `hash_type` (BRO_HASH_LEVEL0 + l: long-prefix level l); the sorted positions land in S.b.
  // Three launches: the digit counts, then one one-sweep pass per digit.
  template <bool LEVEL>
  void run_sort(cudaStream_t stream, const SortBufs& S, const uint8_t* data, uint32_t count, int hash_type, int key_bits) {
    SortArgs sa;
    sa.data = data;
    sa.count = count;
    sa.num_tiles = (count + SORT_TILE - 1) / SORT_TILE;
    sa.state = S.state;
    sa.hash_type = hash_type;
    sa.key_bits = key_bits;
    // counts, tile counters and look-back words start at zero for every sort (batches and chunks follow each other on the lane)
    cudaMemsetAsync(sa.state, 0, sort_state_words(sa.num_tiles) * 4, stream);
    sa.pass = 0;
    sa.in = nullptr;
    sa.outw = S.a;
    k_sort_count<LEVEL><<<std::min<uint32_t>(sa.num_tiles, (uint32_t)num_sms * 8), SORT_THREADS, 0, stream>>>(sa);
    k_sort_onesweep<LEVEL><<<sa.num_tiles, SORT_THREADS, 0, stream>>>(sa);
    sa.pass = 1;
    sa.in = S.a;
    sa.outw = S.b;
    k_sort_onesweep<LEVEL><<<sa.num_tiles, SORT_THREADS, 0, stream>>>(sa);
    launches += 3;
  }

  // BrotliSplitBlock + BrotliBuildMetaBlock's clustering for every metablock of the chunk (replaces k_split_greedy)
  bool run_hq_split(cudaStream_t st, const Workspace& W, const BsWs& B, const CmWs& M) {
    const uint32_t NM = W.num_mb;
    const dim3 g3(NM, 3), gx3(64, NM, 3), g2(NM, 2), gx2(64, NM, 2);
    k_bs_setup<<<g3, 128, 0, st>>>(W, B);
    k_bs_sample<<<dim3(32, NM, 3), 256, 0, st>>>(W, B);
    for (int it = 0; it < 3; ++it) {
      k_bs_icost<<<g3, 256, 0, st>>>(W, B);
      k_bs_forward<<<dim3(B.segc[0], NM, 3), 32, 0, st>>>(W, B);
      k_bs_bfunc<<<dim3(B.segc[0], NM, 3), 32, 0, st>>>(W, B);
      k_bs_bchain<<<g3, 32, 0, st>>>(W, B);
      k_bs_bwrite<<<dim3(B.segc[0], NM, 3), 32, 0, st>>>(W, B);
      k_bs_remap<<<g3, 256, 0, st>>>(W, B);
      k_bs_rehist<<<gx3, 256, 0, st>>>(W, B);
    }
    k_bs_blocks<<<g3, 1024, 0, st>>>(W, B);
    CUDA_OK(cudaMemsetAsync(B.bh_in, 0, (size_t)NM * B.bh_sum * 4, st));
    k_bs_bhist<<<gx3, 256, 0, st>>>(W, B);
    k_bs_cl_prepare<<<gx3, CL_WARPS * 32, 0, st>>>(W, B);
    k_bs_cl_batch<<<dim3(128, NM, 3), CLB_WARPS * 32, 0, st>>>(W, B);
    k_bs_cl_final<<<g3, CLB_WARPS * 32, 0, st>>>(W, B);
    k_bs_cl_assign<<<gx3, CL_WARPS * 32, 0, st>>>(W, B);
    k_bs_types<<<g3, 32, 0, st>>>(W, B);
    k_cm_zero<<<dim3(64, NM), 256, 0, st>>>(W, M);
    k_cm_hist<<<gx3, 256, 0, st>>>(W, M);
    k_cm_cl_prepare<<<gx2, CL_WARPS * 32, 0, st>>>(W, M);
    k_cm_cl_batch<<<dim3(256, NM, 2), CLB_WARPS * 32, 0, st>>>(W, M);
    k_cm_cl_final<<<g2, CLB_WARPS * 32, 0, st>>>(W, M);
    k_cm_cl_assign<<<gx2, CL_WARPS * 32, 0, st>>>(W, M);
    k_cm_reindex<<<g2, 256, 0, st>>>(W, M);
    k_cm_rebuild<<<gx2, 256, 0, st>>>(W, M);
    launches += 2 + 21 + 3 + 5 + 8;
    return true;
  }

  void mark(Lane& L, int stage) {
    if (!timing) return;
    cudaEventRecord(L.marks.get(true), L.stream);
    L.mark_stage.push_back(stage);
  }
  void reset_timings() {
    for (auto& L : lanes) { L.marks.reset(); L.mark_stage.clear(); }
  }
  // per-stage sums of event-bracketed time on each lane's own stream (with two lanes stages of different chunks overlap,
  // so the sum over stages can exceed the wall time)
  void collect_timings() {
    for (int i = 0; i < B200_NUM_STAGES; ++i) stage_ms[i] = 0;
    for (auto& L : lanes) {
      for (size_t i = 0; i + 1 < L.mark_stage.size(); ++i) {
        if (L.mark_stage[i] < 0) continue;
        float ms = 0;
        cudaEventElapsedTime(&ms, L.marks.ev[i], L.marks.ev[i + 1]);
        stage_ms[L.mark_stage[i]] += ms;
      }
    }
    reset_timings();
  }

  // Enqueues, on lane L, the compression of data[range_start, range_start + range_len) of the stream resident at d_data
  // (absolute positions); its metablocks are appended to the output at the running bit position.  `after_layout` (may
  // be null) is the previous chunk's layout event; `layout_done` is recorded when this chunk's layout is final.
  bool run_chunk(Lane& L, const EncParams& Pstream, uint32_t range_start, uint32_t range_len, uint32_t* d_outw,
                 uint64_t out_cap_bytes, bool first, bool last, bool byte_align_end, uint32_t chunk_idx,
                 cudaEvent_t after_layout, cudaEvent_t layout_done) {
    cudaStream_t stream = L.stream;
    Workspace W;
    ChunkBufs X;
    memset(&W, 0, sizeof(W));
    memset(&X, 0, sizeof(X));
    EncParams P = Pstream;
    P.n = range_len;
    P.abs_base = range_start;
    // the whole workspace is in place before the chunk's first launch: growing the arena (cudaFree) waits for the device
    Carve sizing{nullptr};
    layout_chunk(sizing, range_len, P, &W, &X);
    if (!L.arena.ensure(sizing.off)) return false;
    Carve carve{L.arena.as<uint8_t>()};
    layout_chunk(carve, range_len, P, &W, &X);
    W.P = P;
    W.lut = d_lut.as<uint32_t>();
    W.dict.words = d_dict_words.as<uint8_t>();
    W.dict.hash = d_dict_hash.as<uint16_t>();
    W.dict.lut_buckets = d_dict_lutb.as<uint16_t>();
    W.dict.lut_entries = d_dict_lute.as<uint32_t>();
    W.dict.tr_groups = d_dict_trg.as<uint8_t>();
    W.dict.transforms = d_dict_tr.as<uint8_t>();
    W.dict.num_tr_groups = BRO_DICT_NUM_TR_GROUPS;
    W.total_bits = d_total.as<uint64_t>();
    W.data = d_data.as<uint8_t>() + (range_start - data_base);
    W.out = d_outw;
    W.out_cap_bytes = out_cap_bytes;
    const uint8_t* d_all = d_data.as<uint8_t>() - data_base;  // indexable by absolute position >= data_base
    k_init_mb<<<(W.num_mb + 63) / 64, 64, 0, stream>>>(W);
    // the literal context decision needs the input only: it runs here, under the throughput-bound stages of the other lanes,
    // instead of in the latency-bound tail of the chunk
    k_ctx_decide<<<W.num_mb, 256, 0, stream>>>(W);
    // ---- sort + match, batch by batch ----
    const uint32_t window = 1u << P.lgwin;
    const uint32_t payload_max = kBatchMax - window - 4096;
    // q7..q9 and 9.5 (bucket depth >= 64): the parse searches the buckets on demand when the chunk is a single sort batch
    // (depth >= 128 -- q8, q9, 9.5 and the lgwin <= 16 configurations -- gains most on JSON logs and periodic data, where the walk
    // visits few positions; depth 64 (q7) and inputs of a few units are faster up front.  ondemand = 2 forces the on-demand path
    // for every deep configuration, 0 switches it off.)
    const bool od_shape = !P.zopfli && (P.depth == 64 || P.depth == 128 || P.depth == 256 || P.depth == 512) && range_len <= payload_max;
    const bool od = od_shape && (ondemand > 1 || (ondemand == 1 && P.depth >= 128 && range_len >= ((uint32_t)4 << 20)));
    DeepArgs da;
    memset(&da, 0, sizeof(da));
    L.slab_cursor = nullptr;
    for (uint64_t b0 = range_start; b0 < (uint64_t)range_start + range_len; b0 += payload_max) {
      const uint32_t b1 = (uint32_t)std::min<uint64_t>((uint64_t)range_start + range_len, b0 + payload_max);
      uint32_t origin = b0 > window ? (uint32_t)b0 - window : 0u;
      origin &= ~4095u;  // tile staging needs word alignment
      if (origin < data_base) origin = (uint32_t)data_base;
      const uint32_t count = b1 - origin;
      mark(L, B200_ST_SORT);
      run_sort<false>(stream, X.sort, d_all + origin, count, P.hash_type, P.key_bits);
      MatchArgs ma;
      ma.data = d_all;
      ma.sorted = X.sort.b;
      ma.count = count;
      ma.origin = origin;
      ma.payload_begin = (uint32_t)b0 - origin;
      ma.n = range_start + range_len;  // matches may not run past the end of this range
      ma.best = W.best - range_start;  // best[] is indexed by range-relative position
      ma.hash_type = P.hash_type;
      ma.key_bits = P.key_bits;
      ma.depth = P.depth;
      ma.lcap = P.lcap;
      ma.max_backward = P.max_backward;
      ma.dict = W.dict;
      ma.use_dict = P.use_dict;
      const BestStage bs{X.stage, X.sort.state + SORT_ST_SLAB};  // cursors zeroed by run_sort
      const size_t smem = (size_t)(MATCH_THREADS + P.depth) * 6 * 4;
      mark(L, B200_ST_MATCH);
      const uint32_t mgrid = (count + MATCH_THREADS - 1) / MATCH_THREADS;
      if (od) {  // ranks into best[], signatures into the free half of the sort ping-pong
        da.m = ma;
        da.sig = X.sort.a;
        k_rank_sig<<<(count + 255) / 256, 256, 0, stream>>>(ma, X.sort.a);
        if (od_probe) {  // stage hook only: the search of every position, while the ranks and signatures are intact
          const uint32_t pg = (range_len + 7) / 8;
          if (P.depth == 64) k_od_probe<64><<<pg, 256, 0, stream>>>(da, range_start, range_len, od_probe);
          else if (P.depth == 128) k_od_probe<128><<<pg, 256, 0, stream>>>(da, range_start, range_len, od_probe);
          else if (P.depth == 256) k_od_probe<256><<<pg, 256, 0, stream>>>(da, range_start, range_len, od_probe);
          else k_od_probe<512><<<pg, 256, 0, stream>>>(da, range_start, range_len, od_probe);
        }
      } else
      if (P.zopfli) {  // all matches of every position
        MatchAllArgs aa;
        aa.m = ma;
        aa.hqm = W.hqm - (size_t)range_start * HQ_MAXM;
        aa.hqn = W.hqn - range_start;
        aa.quality = P.quality;
        aa.level = 0;
        aa.last_pass = P.hq_levels == 0;
        if (P.depth != 256) { fprintf(stderr, "[brotli_b200] unsupported bucket depth %d\n", P.depth); return false; }
        k_match_all<256><<<mgrid, MATCH_THREADS, (size_t)(MATCH_THREADS + 256) * 3 * 4, stream>>>(aa);
        for (int lv = 0; lv < P.hq_levels; ++lv) {  // long-prefix levels: the batch re-sorted by the level's hash, lists merged
          run_sort<true>(stream, X.sort, d_all + origin, count, BRO_HASH_LEVEL0 + lv, P.key_bits);
          aa.level = lv;
          aa.last_pass = lv + 1 == P.hq_levels;
          k_match_level<HQ_LEVEL_DEPTH><<<mgrid, MATCH_THREADS, (size_t)(MATCH_THREADS + HQ_LEVEL_DEPTH) * 3 * 4, stream>>>(aa);
          launches += 1;
        }
      } else {
        switch (P.depth) {  // bucket depth = 1 << block_bits: 16 (q5) .. 256 (q9, and lgwin <= 16), 512 (quality 11 with Q9_5)
          case 16:
            k_match_shallow<16><<<mgrid, MATCH_THREADS, smem, stream>>>(ma, bs);
            break;
          case 32:
            k_match_shallow<32><<<mgrid, MATCH_THREADS, smem, stream>>>(ma, bs);
            break;
          case 64: k_match_deep<64><<<mgrid, MATCH_THREADS, smem, stream>>>(ma); break;
          case 128: k_match_deep<128><<<mgrid, MATCH_THREADS, smem, stream>>>(ma); break;
          case 256: k_match_deep<256><<<mgrid, MATCH_THREADS, smem, stream>>>(ma); break;
          case 512: k_match_deep<512><<<mgrid, MATCH_THREADS, smem, stream>>>(ma); break;
          default: fprintf(stderr, "[brotli_b200] unsupported bucket depth %d\n", P.depth); return false;
        }
        if (P.depth <= 32) {  // k_match_shallow left one record per payload position in X.stage
          const uint32_t payload = b1 - (uint32_t)b0;
          k_best_place<<<(payload + 255) / 256, 256, 0, stream>>>(X.stage, payload, ma.best);
          L.slab_cursor = bs.slab_cursor;
          L.slab_payload = payload;
          launches += 1;
        }
      }
      launches += 1;
    }
    mark(L, B200_ST_PARSE);
    if (P.zopfli) {  // shortest-path parse, one unit per warp
      for (int phase = 1; phase <= (P.quality >= 11 ? 2 : 1); ++phase) k_zopfli<<<W.num_units, 32, 0, stream>>>(W, X.za, phase);
    } else {  // greedy / lazy parse: fill_params gives n_last 4 at depth 16 / 32 (q5, q6), 10 at 64 / 128 (q7, q8), 16 at 256 / 512
      const uint32_t pg = (W.num_units + PARSE_WARPS - 1) / PARSE_WARPS;
      if (od && P.n_last == 10 && P.depth == 64) k_parse_ondemand<10, 64><<<pg, PARSE_WARPS * 32, 0, stream>>>(W, da);
      else if (od && P.n_last == 10 && P.depth == 128) k_parse_ondemand<10, 128><<<pg, PARSE_WARPS * 32, 0, stream>>>(W, da);
      else if (od && P.n_last == 16 && P.depth == 256) k_parse_ondemand<16, 256><<<pg, PARSE_WARPS * 32, 0, stream>>>(W, da);
      else if (od && P.n_last == 16 && P.depth == 512) k_parse_ondemand<16, 512><<<pg, PARSE_WARPS * 32, 0, stream>>>(W, da);
      else if (!od && P.n_last == 4) k_parse_pair<<<(W.num_units + 4 * PARSE_WARPS - 1) / (4 * PARSE_WARPS), PARSE_WARPS * 32, 0, stream>>>(W);
      else if (!od && P.n_last == 10) k_parse<10><<<pg, PARSE_WARPS * 32, 0, stream>>>(W);
      else if (!od && P.n_last == 16) k_parse<16><<<pg, PARSE_WARPS * 32, 0, stream>>>(W);
      else { fprintf(stderr, "[brotli_b200] unsupported parse shape: n_last %d, bucket depth %d\n", P.n_last, P.depth); return false; }
    }
    mark(L, B200_ST_FINALIZE);
    k_fin_count<<<W.num_mb, 1024, 0, stream>>>(W);
    k_fin_write<<<(W.num_units + PARSE_WARPS - 1) / PARSE_WARPS, PARSE_WARPS * 32, 0, stream>>>(W);
    k_fin_dist<<<W.num_mb, 1024, 0, stream>>>(W);
    if (P.hq_meta && P.hq_split) {  // NPOSTFIX / NDIRECT of every metablock (metablock.rs:152-207), commands re-coded
      k_dist_cost<<<dim3(64, W.num_mb), 256, 0, stream>>>(W, X.dist_cost);
      k_dist_apply<<<dim3(64, W.num_mb), 256, 0, stream>>>(W, X.dist_cost);
      launches += 2;
    }
    {
      dim3 g((W.cmd_cap + 255) / 256, W.num_mb);
      cudaMemsetAsync(W.long_tab, 0, (size_t)W.num_mb * W.long_cap * sizeof(uint2), stream);
      k_symbols<<<g, 256, 0, stream>>>(W);
      k_symbols_long<<<dim3(LONG_GRID, W.num_mb), 256, 0, stream>>>(W);
    }
    mark(L, B200_ST_SPLIT);
    {
      dim3 g(W.num_mb, 3);
      if (P.hq_meta && P.hq_split) { if (!run_hq_split(stream, W, X.bs, X.cm)) return false; }
      else k_split_greedy<<<g, SPLIT_THREADS, SPLIT_SMEM_WORDS * 4, stream>>>(W);
    }
    mark(L, B200_ST_HEADER);
    {
      dim3 g(W.max_lit_trees + W.max_cmd_types + W.max_dist_types + HDR_SECTIONS, W.num_mb);
      k_trees<<<g, 32, 0, stream>>>(W);
    }
    k_header<<<W.num_mb, 32, 0, stream>>>(W);
    mark(L, B200_ST_EMIT);
    {
      dim3 g((W.cmd_cap + 255) / 256, W.num_mb);
      k_bitlen_long<<<dim3(LONG_GRID, W.num_mb), 256, 0, stream>>>(W);
      k_bitlen<<<g, 256, 0, stream>>>(W);
      k_bitscan<<<W.num_mb, 1024, 0, stream>>>(W);
      if (after_layout) CUDA_OK(cudaStreamWaitEvent(stream, after_layout, 0));  // bit positions chain through the chunks
      k_layout<<<1, 32, 0, stream>>>(W, first ? 1 : 0, last ? 1 : 0, byte_align_end ? 1 : 0, d_total.as<uint64_t>() + 1 + chunk_idx);
      CUDA_OK(cudaEventRecord(layout_done, stream));
      k_emit_header<<<W.num_mb, 256, 0, stream>>>(W);
      k_emit_body<<<g, 256, 0, stream>>>(W);
      k_emit_long<<<dim3(LONG_GRID, W.num_mb), 256, 0, stream>>>(W);
      dim3 gr(64, W.num_mb);
      k_emit_raw<<<gr, 256, 0, stream>>>(W);
    }
    mark(L, -1);
    launches += 19;
    L.W = W;
    CUDA_OK(cudaGetLastError());
    return true;
  }
};

// ---------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------
extern "C" {

int b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}
// The quality the device path runs for a requested one (bro_parse.cuh: effective_quality)
int b200_effective_quality(int requested_quality) { return effective_quality(requested_quality); }

B200Encoder* b200_encoder_create(int device) {
  B200Encoder* e = new B200Encoder();
  if (!e->init(device)) {
    delete e;
    return nullptr;
  }
  return e;
}
int b200_encoder_device(const B200Encoder* e) { return e ? e->device : -1; }
void b200_encoder_destroy(B200Encoder* e) {
  if (!e) return;
  e->destroy();
  delete e;
}
int b200_encoder_set_option(B200Encoder* e, int option, uint32_t value) {
  if (!e) return 0;
  switch (option) {
    case B200_OPT_CTX_MODEL: e->ctx_model = (int)value; return 1;
    case B200_OPT_TIMING: e->timing = value != 0; return 1;
    case B200_OPT_DICT: e->use_dict = (int)value; return 1;
    case B200_OPT_ONDEMAND: e->ondemand = (int)value; return 1;
    case B200_OPT_HQ_LEVELS: e->hq_levels = value > HQ_MAX_LEVELS ? HQ_MAX_LEVELS : (int)value; return 1;
    case B200_OPT_HQ_SPLIT: e->hq_split = (int)value; return 1;
    case B200_OPT_HQ_UNIT: e->hq_unit = value; return 1;
    case B200_OPT_Q9_5: e->q9_5 = value != 0; return 1;
    case B200_OPT_LANES: e->num_lanes = value < 1 ? 1 : (value > (uint32_t)kMaxLanes ? kMaxLanes : (int)value); return 1;
  }
  return 0;
}

size_t b200_max_compressed_size(size_t n) { return n + (n >> 10) * 8 + 4096; }

// Stages the input of plan c on s_in and enqueues its chunks on the lanes; their metablocks are written into `out` (c.need
// bytes, zeroed here first).  The caller has made s_in wait for whatever the call is ordered after.  h_done (blocking path):
// each chunk's end bit position is copied to h_total[k] on its lane and h_done[k] is recorded behind it.
//
// Pipeline: the input is staged chunk by chunk on a copy stream and chunks alternate between the compute lanes.
// pro (device input only): the prologue of a framed stream goes in front, and the first chunk starts behind it.
static bool enqueue_range(B200Encoder* e, const CallPlan& c, const uint8_t* in, cudaMemcpyKind in_kind, uint8_t* out, bool first,
                          bool last, bool byte_align, std::vector<cudaEvent_t>* h_done, const B200Prologue* pro = nullptr,
                          const uint8_t* pro_in = nullptr) {
  const size_t nchunks = c.chunks.size();
  e->data_base = c.base;
  uint8_t* dd = e->d_data.as<uint8_t>();
  CUDA_OK(cudaMemsetAsync(out, 0, c.need, e->s_in));
  CUDA_OK(cudaMemsetAsync(e->d_total.p, 0, 8, e->s_in));
  if (pro) {
    k_prologue<<<1, 32, 0, e->s_in>>>(*pro, pro_in, out, e->d_total.as<uint64_t>(), nullptr);
    e->launches += 1;
  }
  CUDA_OK(cudaMemsetAsync(dd + c.staged, 0, kPad, e->s_in));
  cudaEvent_t prev_layout = nullptr;
  size_t copied = c.base;  // absolute position up to which the input is staged
  for (size_t k = 0; k < nchunks; ++k) {
    const size_t s = c.chunks[k].first, len = c.chunks[k].second;
    // stage the input this chunk can see: its window halo (first chunk), its own bytes, a short look-ahead
    const size_t upto = std::min(c.end, s + len + kLookahead);
    if (upto > copied) {
      CUDA_OK(cudaMemcpyAsync(dd + (copied - c.base), in + copied, upto - copied, in_kind, e->s_in));
      copied = upto;
    }
    cudaEvent_t ev_in = e->sync_events.get(false);
    CUDA_OK(cudaEventRecord(ev_in, e->s_in));
    Lane& L = e->lanes[k % (size_t)e->num_lanes];
    CUDA_OK(cudaStreamWaitEvent(L.stream, ev_in, 0));
    cudaEvent_t ev_layout = e->sync_events.get(false);
    const bool f = first && k == 0, l = k + 1 == nchunks;
    if (!e->run_chunk(L, c.P, (uint32_t)s, (uint32_t)len, reinterpret_cast<uint32_t*>(out), c.need, f, last && l, byte_align && l,
                      (uint32_t)k, prev_layout, ev_layout))
      return false;
    prev_layout = ev_layout;
    if (h_done) {
      CUDA_OK(cudaMemcpyAsync(e->h_total + k, e->d_total.as<uint64_t>() + 1 + k, 8, cudaMemcpyDeviceToHost, L.stream));
      (*h_done)[k] = e->sync_events.get(false);
      CUDA_OK(cudaEventRecord((*h_done)[k], L.stream));
    }
  }
  return true;
}

// Compresses [range_start, range_start+range_len) of an n-byte stream and returns when the output is in place.  in/out are
// device pointers when device_io != 0, host pointers otherwise.  first/last: emit stream header / final empty metablock;
// byte_align: end the range with a padding metablock so that ranges can be concatenated with memcpy.
//
// The stream is built in d_out; as each chunk finishes, the finished part of the output is copied to `out` while later chunks
// are still running.
static bool compress_range_impl(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, const uint8_t* in, size_t n,
                                size_t range_start, size_t range_len, bool first, bool last, bool byte_align, uint8_t* out,
                                size_t out_cap, size_t* out_size, int device_io, bool keep_on_device) {
  e->launches = 0;
  e->reset_timings();
  e->sync_events.reset();
  CallPlan c;
  e->plan_call(&c, quality, lgwin, size_hint ? size_hint : n, range_start, range_len);
  const size_t nchunks = c.chunks.size();
  // device_io: 0 host in / host out, 1 device in / device out, 2 host in / device out, 3 device in / host out
  const bool in_dev = device_io == 1 || device_io == 3, out_dev = device_io == 1 || device_io == 2;
  const cudaMemcpyKind in_kind = in_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  const cudaMemcpyKind out_kind = out_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  // the whole workspace is in place before the first launch: growing a buffer (cudaFree) waits for the device
  if (!e->provide(e->sizes_of(c), true) || !e->d_out.ensure(c.need) || !e->ensure_totals(nchunks)) return false;
  CUDA_OK(cudaStreamWaitEvent(e->s_in, e->ev_call, 0));  // behind the encoder's last stream-ordered call
  std::vector<cudaEvent_t> ev_done(nchunks);
  if (!enqueue_range(e, c, in, in_kind, e->d_out.as<uint8_t>(), first, last, byte_align, &ev_done)) return false;
  // drain: as each chunk finishes, every output byte below its end bit position is final
  size_t done_bytes = 0;
  for (size_t k = 0; k < nchunks; ++k) {
    if (cudaEventSynchronize(ev_done[k]) != cudaSuccess) {
      fprintf(stderr, "[brotli_b200] kernel failure: %s\n", cudaGetErrorString(cudaGetLastError()));
      return false;
    }
    const uint64_t tb = e->h_total[k];
    const size_t upto = k + 1 == nchunks ? (size_t)((tb + 7) >> 3) : (size_t)(tb >> 3);
    if (upto > out_cap) return false;
    if (!keep_on_device && upto > done_bytes)
      CUDA_OK(cudaMemcpyAsync(out + done_bytes, e->d_out.as<uint8_t>() + done_bytes, upto - done_bytes, out_kind, e->s_out));
    done_bytes = upto;
  }
  CUDA_OK(cudaStreamSynchronize(e->s_out));
  CUDA_OK(cudaStreamSynchronize(e->s_in));
  *out_size = done_bytes;
  if (e->timing) e->collect_timings();
  return true;
}

// The stream-ordered ending (b200_encoder_compress_range_async): the call forks from `st` into s_in (and through s_in's events
// into the lanes), joins back into `st` behind the last work of s_in and of every lane it used, and writes *out_size with one
// more launch on `st`.  Inside a capture it neither waits for nor records ev_call: a graph may not depend on work outside it.
static bool enqueue_async(B200Encoder* e, const CallPlan& c, const uint8_t* in, bool first, bool last, bool byte_align,
                          bool empty_stream, uint8_t* out, uint64_t* out_size, cudaStream_t st, bool capturing,
                          const B200Prologue* pro = nullptr, int trailer = -1, const uint8_t* pro_in = nullptr) {
  const size_t nchunks = c.chunks.size();
  cudaEvent_t fork = e->sync_events.get(false);
  CUDA_OK(cudaEventRecord(fork, st));
  CUDA_OK(cudaStreamWaitEvent(e->s_in, fork, 0));
  if (!capturing) CUDA_OK(cudaStreamWaitEvent(e->s_in, e->ev_call, 0));
  if (nchunks) {
    if (!enqueue_range(e, c, in, cudaMemcpyDeviceToDevice, out, first, last, byte_align, nullptr, pro, pro_in)) return false;
  } else {
    CUDA_OK(cudaMemsetAsync(out, 0, c.need, e->s_in));
  }
  cudaStream_t used[kMaxLanes + 1];
  size_t nused = 0;
  used[nused++] = e->s_in;
  for (size_t i = 0; i < std::min(nchunks, (size_t)e->num_lanes); ++i) used[nused++] = e->lanes[i].stream;
  for (size_t i = 0; i < nused; ++i) {
    cudaEvent_t join = e->sync_events.get(false);
    CUDA_OK(cudaEventRecord(join, used[i]));
    CUDA_OK(cudaStreamWaitEvent(st, join, 0));
  }
  k_out_size<<<1, 1, 0, st>>>(nchunks ? e->d_total.as<uint64_t>() + nchunks : nullptr, out, empty_stream ? 1 : 0, out_size, trailer);
  e->launches += 1;
  CUDA_OK(cudaGetLastError());
  if (!capturing) CUDA_OK(cudaEventRecord(e->ev_call, st));
  return true;
}

int b200_encoder_reserve(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, size_t n, size_t range_len) {
  if (!e || !e->ok || n >= 0xFFFFF000ull || range_len > n) return 0;
  if (cudaSetDevice(e->device) != cudaSuccess) return 0;
  // Every call with the same or smaller arguments must fit.  Workspaces grow with the range and the window, but not with the
  // quality or the size hint: smaller parse units (quality 10 against 11, small size hints at 10 / 11) need more per byte.  So
  // each quality family up to `quality` is sized at each size-hint class up to `size_hint`; the staged input is bounded over
  // every range start.  Quality 10 / 11 include their Q9_5 layout (the hash-chain regions next to the histogram-stage ones),
  // whatever the encoder's B200_OPT_Q9_5 is now, because the framed entry points set it per call.
  const uint64_t hint = size_hint ? size_hint : n;
  const int q_max = effective_quality(quality);
  const uint64_t hints[3] = {hint, std::min<uint64_t>(hint, 1u << 20), std::min<uint64_t>(hint, 256u << 10)};
  CallSizes s;
  const int saved_q95 = e->q9_5;
  for (int q : {5, 10, 11}) {
    if (q > q_max) break;
    for (int q95 = 0; q95 <= (q >= 10 ? 1 : 0); ++q95) {
      e->q9_5 = q95;
      for (uint64_t h : hints) {
        if (!h) continue;
        CallPlan c;
        e->plan_call(&c, q, lgwin, h, n - range_len, range_len);
        s.cover(e->sizes_of(c));
      }
    }
  }
  e->q9_5 = saved_q95;
  if (range_len) {
    EncParams P;
    e->fill_params(&P, quality, lgwin, hint);
    s.data = std::min<size_t>(n, range_len + ((size_t)1 << P.lgwin) + 4095) + kPad;
  }
  return e->provide(s, true) ? 1 : 0;
}

// b200_encoder_compress_range_async and, with a prologue / trailer / per-call options, b200_encoder_compress_framed_async
static int compress_async_impl(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, int ctx_model, int use_dict, int q9_5,
                               const uint8_t* in, size_t n, size_t range_start, size_t range_len, int first, int last, int byte_align,
                               const B200Prologue* pro, int trailer, uint8_t* out, size_t out_cap, uint64_t* out_size, void* stream) {
  if (!e || !e->ok || !out || !out_size) return 0;
  if (n >= 0xFFFFF000ull || range_start > n || range_len > n - range_start) return 0;  // 32-bit positions
  if (pro && (pro->len > sizeof(pro->bytes) || pro->data_off + pro->n2 > pro->len || pro->n2 > range_start)) return 0;
  const uint8_t* pro_in = pro ? in + range_start - pro->n2 : nullptr;  // the prologue's data bytes precede the range
  if (cudaSetDevice(e->device) != cudaSuccess) return 0;
  if (out_cap < b200_max_compressed_size(range_len) + 64 || (reinterpret_cast<uintptr_t>(out) & 3)) return 0;
  const bool reads_in = range_len || (pro && pro->n2);
  // (the pointer queries run in relaxed capture mode: under a global-mode capture on another stream they are no reason to fail)
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  if (cudaThreadExchangeStreamCaptureMode(&mode) != cudaSuccess) return 0;
  const bool placed = on_device(out, e->device) && on_device(out_size, e->device) && (!reads_in || on_device(in, e->device));
  cudaThreadExchangeStreamCaptureMode(&mode);
  if (!placed) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaStreamCaptureStatus cs;
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  if (cs == cudaStreamCaptureStatusInvalidated) return 0;
  const bool capturing = cs == cudaStreamCaptureStatusActive;
  if (pro && pro->complete) {  // the whole stream is prologue and trailer: nothing of the encoder is used
    k_prologue<<<1, 32, 0, st>>>(*pro, pro_in, out, nullptr, out_size);
    return cudaGetLastError() == cudaSuccess ? 1 : 0;
  }
  const int saved_ctx = e->ctx_model, saved_dict = e->use_dict, saved_q95 = e->q9_5;
  if (ctx_model >= 0) e->ctx_model = ctx_model;  // read into the call's parameters by plan_call, restored below
  if (use_dict >= 0) e->use_dict = use_dict;
  if (q9_5 >= 0) e->q9_5 = q9_5;
  CallPlan c;
  e->plan_call(&c, quality, lgwin, size_hint ? size_hint : n, range_start, range_len);
  e->ctx_model = saved_ctx;
  e->use_dict = saved_dict;
  e->q9_5 = saved_q95;
  if (pro && c.chunks.empty()) return 0;  // a prologue in front of nothing is a complete one
  if (!e->provide(e->sizes_of(c), !capturing)) {
    if (capturing) fprintf(stderr, "[brotli_b200] a call inside a CUDA graph capture needs b200_encoder_reserve first\n");
    return 0;
  }
  if (capturing) e->freeze();
  e->launches = 0;
  e->reset_timings();
  e->sync_events.reset();
  const bool timing = e->timing;
  e->timing = false;  // stage timing would read events back on the host
  const bool ok = enqueue_async(e, c, in, first != 0, last != 0, byte_align != 0, first && last && n == 0, out, out_size, st,
                                capturing, pro, trailer, pro_in);
  e->timing = timing;
  if (!ok) {
    if (!capturing) cudaDeviceSynchronize();  // leave no work in flight behind a failed call
    return 0;
  }
  return 1;
}

int b200_encoder_compress_range_async(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, const uint8_t* in, size_t n,
                                      size_t range_start, size_t range_len, int first, int last, int byte_align, uint8_t* out,
                                      size_t out_cap, uint64_t* out_size, void* stream) {
  return compress_async_impl(e, quality, lgwin, size_hint, -1, -1, -1, in, n, range_start, range_len, first, last, byte_align, nullptr, -1,
                             out, out_cap, out_size, stream);
}

int b200_encoder_compress_framed_async(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, int ctx_model, int use_dict,
                                       int q9_5, const uint8_t* in, size_t n, size_t range_start, size_t range_len, int first,
                                       int last, int byte_align, const B200Prologue* pro, int trailer, uint8_t* out, size_t out_cap,
                                       uint64_t* out_size, void* stream) {
  return compress_async_impl(e, quality, lgwin, size_hint, ctx_model, use_dict, q9_5, in, n, range_start, range_len, first, last, byte_align,
                             pro, trailer, out, out_cap, out_size, stream);
}

int b200_encoder_compress_range(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, const uint8_t* in, size_t n,
                                size_t range_start, size_t range_len, int first, int last, int byte_align, uint8_t* out,
                                size_t out_cap, size_t* out_size, int device_io) {
  if (!e || !e->ok || !out_size) return 0;
  if (n >= 0xFFFFF000ull) return 0;  // 32-bit positions
  if (cudaSetDevice(e->device) != cudaSuccess) return 0;
  if (n == 0 || range_len == 0) {
    if (first && last && n == 0) {  // encode.rs:1463-1467
      if (out_cap < 1) return 0;
      uint8_t b = 6;
      if (device_io == 1 || device_io == 2) { if (cudaMemcpy(out, &b, 1, cudaMemcpyHostToDevice) != cudaSuccess) return 0; }
      else out[0] = b;
      *out_size = 1;
      return 1;
    }
    *out_size = 0;
    return 1;
  }
  if (!compress_range_impl(e, quality, lgwin, size_hint, in, n, range_start, range_len, first != 0, last != 0, byte_align != 0,
                           out, out_cap, out_size, device_io, false)) {
    cudaDeviceSynchronize();  // leave no work in flight behind a failed call
    return 0;
  }
  return 1;
}

int b200_encoder_compress(B200Encoder* e, int quality, int lgwin, const uint8_t* in, size_t n, uint8_t* out, size_t out_cap,
                          size_t* out_size, int device_io) {
  return b200_encoder_compress_range(e, quality, lgwin, n, in, n, 0, n, 1, 1, 0, out, out_cap, out_size, device_io);
}

int b200_encoder_last_timings(B200Encoder* e, float* ms, uint32_t* launches) {
  if (!e) return 0;
  for (int i = 0; i < B200_NUM_STAGES; ++i) ms[i] = e->stage_ms[i];
  if (launches) *launches = e->launches;
  return 1;
}

// test hook (the hash-chain parse: quality 5..9, and 10 / 11 with B200_OPT_Q9_5): best[] of the match stage for the range
// [range_start, range_start + range_len) of an n-byte buffer (host in, host out; range_len <= one chunk, the bytes in front of the
// range are its window).  search = 0: the up-front kernels (k_match_shallow / k_match_deep), with the on-demand path switched off
// for the call.  search = 1: the on-demand search (k_rank_sig + deep_best_warp) at every position of the range; 0 is returned
// where that path does not run (depth < 64, or a chunk that needs more than one sort batch).
int b200_stage_match(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, const uint8_t* in, size_t n, size_t range_start,
                     size_t range_len, int search, uint32_t* best_out) {
  if (!e || !e->ok || n == 0 || n >= 0xFFFFF000ull || range_len == 0 || range_len > kChunk || range_start > n - range_len) return 0;
  if (search != 0 && search != 1) return 0;
  if (cudaSetDevice(e->device) != cudaSuccess) return 0;
  if (!size_hint) size_hint = n;
  EncParams P;
  e->fill_params(&P, quality, lgwin, size_hint);
  if (P.zopfli) return 0;
  if (search) {
    const uint64_t payload_max = kBatchMax - (1ull << P.lgwin) - 4096;
    if (P.depth < 64 || range_len > payload_max) return 0;
    if (!e->d_probe.ensure(range_len * 4)) return 0;
    e->od_probe = e->d_probe.as<uint32_t>();
  }
  const int ondemand = e->ondemand;
  e->ondemand = search ? 2 : 0;
  size_t got = 0;
  const bool ok = compress_range_impl(e, quality, lgwin, size_hint, in, n, range_start, range_len, true, true, false, nullptr,
                                      b200_max_compressed_size(range_len) + 64, &got, 0, true);
  e->ondemand = ondemand;
  e->od_probe = nullptr;
  if (!ok) {
    cudaDeviceSynchronize();
    return 0;
  }
  const void* src = search ? e->d_probe.p : (const void*)e->lanes[0].W.best;
  return cudaMemcpy(best_out, src, range_len * 4, cudaMemcpyDeviceToHost) == cudaSuccess;
}

// test hook: after b200_stage_match with the up-front kernels, the slab cursors of the range's last sort batch (records that
// match_store claimed in each slab) into cursors[] and the number of records each slab must receive into sizes[], at most cap
// of each.  Returns the number of slabs, 0 when the last call did not store through match_store.
int b200_stage_match_slabs(B200Encoder* e, uint32_t* cursors, uint32_t* sizes, uint32_t cap) {
  if (!e || !e->ok || cudaSetDevice(e->device) != cudaSuccess) return 0;
  const Lane& L = e->lanes[0];
  if (!L.slab_cursor) return 0;
  const uint32_t ns = (L.slab_payload + (1u << BEST_SLAB_BITS) - 1) >> BEST_SLAB_BITS;
  const uint32_t k = std::min(ns, cap);
  if (cudaMemcpy(cursors, L.slab_cursor, (size_t)k * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
  for (uint32_t s = 0; s < k; ++s) sizes[s] = std::min(1u << BEST_SLAB_BITS, L.slab_payload - (s << BEST_SLAB_BITS));
  return (int)ns;
}

// test hook (the shortest-path parse): matches per position, per-unit results and raw commands of an n-byte buffer (n <= one chunk)
int b200_stage_hq(B200Encoder* e, int quality, int lgwin, const uint8_t* in, size_t n, uint8_t* hqn, uint32_t* hqm, uint32_t* units,
                  uint32_t* raw) {
  if (!e || !e->ok || n == 0 || n > kChunk) return 0;
  EncParams P;
  e->fill_params(&P, quality, lgwin, n);
  if (!P.zopfli) return 0;
  if (cudaSetDevice(e->device) != cudaSuccess) return 0;
  size_t got = 0;
  if (!compress_range_impl(e, quality, lgwin, n, in, n, 0, n, true, true, false, nullptr, b200_max_compressed_size(n) + 64, &got, 0, true)) {
    cudaDeviceSynchronize();
    return 0;
  }
  const Workspace& W = e->lanes[0].W;
  const uint32_t nu = W.num_units;
  bool ok = cudaMemcpy(hqn, W.hqn, n, cudaMemcpyDeviceToHost) == cudaSuccess;
  ok = ok && cudaMemcpy(hqm, W.hqm, n * HQ_MAXM * 8, cudaMemcpyDeviceToHost) == cudaSuccess;
  ok = ok && cudaMemcpy(units, W.unit_ncmd, (size_t)nu * 3 * 4, cudaMemcpyDeviceToHost) == cudaSuccess;  // ncmd, tail, ncopy
  ok = ok && cudaMemcpy(raw, W.raw, (size_t)nu * (W.P.unit / 2 + 1) * 12, cudaMemcpyDeviceToHost) == cudaSuccess;
  return ok ? 1 : 0;
}

// test hook: the sorted positions of one sort batch covering an n-byte buffer (n <= 2^25), by the bucket key the quality /
// lgwin / size n configuration uses, or (level 0..2) by the key of that long-prefix level of quality 10 / 11
int b200_stage_sort(B200Encoder* e, int quality, int lgwin, const uint8_t* in, size_t n, int level, uint32_t* sorted_out) {
  if (!e || !e->ok || n == 0 || n > kBatchMax || level >= HQ_MAX_LEVELS) return 0;
  if (cudaSetDevice(e->device) != cudaSuccess) return 0;
  EncParams P;
  e->fill_params(&P, quality, lgwin, n);
  Lane& L = e->lanes[0];
  Carve sizing{nullptr};
  layout_sort(sizing, (uint32_t)n);
  if (!e->d_data.ensure(n + kPad) || !L.arena.ensure(sizing.off)) return 0;
  Carve carve{L.arena.as<uint8_t>()};
  const SortBufs S = layout_sort(carve, (uint32_t)n);
  e->data_base = 0;
  uint8_t* dd = e->d_data.as<uint8_t>();
  bool ok = cudaStreamWaitEvent(L.stream, e->ev_call, 0) == cudaSuccess &&
            cudaMemcpyAsync(dd, in, n, cudaMemcpyHostToDevice, L.stream) == cudaSuccess &&
            cudaMemsetAsync(dd + n, 0, kPad, L.stream) == cudaSuccess;
  if (!ok) return 0;
  if (level < 0) e->run_sort<false>(L.stream, S, dd, (uint32_t)n, P.hash_type, P.key_bits);
  else e->run_sort<true>(L.stream, S, dd, (uint32_t)n, BRO_HASH_LEVEL0 + level, P.key_bits);
  ok = cudaStreamSynchronize(L.stream) == cudaSuccess;
  return ok && cudaMemcpy(sorted_out, S.b, n * 4, cudaMemcpyDeviceToHost) == cudaSuccess;
}

// parse unit the shortest-path parse uses for this size hint with the encoder's current options (sizes the b200_stage_hq buffers)
uint32_t b200_hq_unit(B200Encoder* e, int quality, uint64_t size_hint) {
  if (!e) return 0;
  EncParams P;
  e->fill_params(&P, quality, 22, size_hint);
  return P.zopfli ? P.unit : 0;
}

}  // extern "C"

// bro_capi.cu -- the reference's C ABI (src/ffi/compressor.rs, src/ffi/multicompress/mod.rs) on top of the device
// encoder.  Host-side state machine only; every byte of compressed output is produced by the CUDA path.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "brotli_b200.h"
#include "bro_encoder.h"

namespace {

constexpr size_t BRO_CHUNK_BYTES_CAPI = (size_t)24 << 20;  // = BRO_CHUNK_BYTES of the device encoder

struct EncoderParams {  // the subset of BrotliEncoderParams (backward_references/mod.rs:71-125) this path consumes
  int quality = 11;     // defaults: encode.rs:318-357
  int lgwin = 22;
  int mode = 0;
  uint64_t size_hint = 0;
  int disable_ctx = 0;
  int no_dictionary = 0;
  int q9_5 = 0;         // BROTLI_PARAM_Q9_5 (encode.rs:221): quality 10 / 11 parse with the hash chains (bro_hq.cuh: default_enc_params)
  int catable = 0, appendable = 0, magic_number = 0, byte_align = 0, bare_stream = 0;
};

// Stream framing (encode.rs:559-568 SanitizeParams): catable implies appendable and no static dictionary; a bare stream is byte
// aligned; byte alignment only means something for appendable / bare streams.
void sanitize_framing(EncoderParams& p) {
  if (p.catable) { p.appendable = 1; p.no_dictionary = 1; }
  if (p.bare_stream) p.byte_align = 1;
  else if (!p.appendable) p.byte_align = 0;
}
bool framed(const EncoderParams& p) { return p.catable || p.appendable || p.magic_number || p.byte_align || p.bare_stream; }

// lgwin as the stream runs it: the window bits, the custom dictionary's share and the rebase window all use this value.
int window_bits(const EncoderParams& p) { return p.lgwin < 10 ? 10 : (p.lgwin > 24 ? 24 : p.lgwin); }
// The bytes kept in front of a position when input is handed over from a later base: the window and 64 KiB.
uint64_t rebase_window(const EncoderParams& p) { return ((uint64_t)1 << window_bits(p)) + 65536; }

// Applies one parameter; a value this path cannot honour leaves `p` unchanged and returns false (the reference's
// set_parameter returns false only after initialisation, encode.rs:289-295 -- here "accepted" also means "will act").
bool apply_param(EncoderParams& p, int key, uint32_t value) {
  EncoderParams q = p;
  switch (key) {
    case BROTLI_PARAM_MODE: if (value > 2) return false; q.mode = (int)value; break;
    case BROTLI_PARAM_QUALITY: q.quality = (int)value; break;
    case BROTLI_PARAM_LGWIN: q.lgwin = (int)value; break;
    case BROTLI_PARAM_LGBLOCK:  // 0 = automatic, else 16..24 (SanitizeParams encode.rs:570-585); the parse granularity is a
      if (!(value == 0 || (value >= 16 && value <= 24))) return false;  // device-side constant: a valid value changes nothing
      break;
    case BROTLI_PARAM_DISABLE_LITERAL_CONTEXT_MODELING: q.disable_ctx = (int)value; break;
    case BROTLI_PARAM_SIZE_HINT: q.size_hint = value; break;
    case BROTLI_PARAM_NO_DICTIONARY: q.no_dictionary = value != 0; break;
    case BROTLI_PARAM_LARGE_WINDOW: if (value != 0) return false; break;  // windows above 2^24 are not produced
    case BROTLI_PARAM_Q9_5: q.q9_5 = value != 0; break;
    // stream framing (encode.rs:264-283; acted on by compress_framed below)
    case BROTLI_PARAM_CATABLE: q.catable = value != 0; if (!q.appendable) q.appendable = value != 0; break;
    case BROTLI_PARAM_APPENDABLE: q.appendable = value != 0; break;
    case BROTLI_PARAM_MAGIC_NUMBER: q.magic_number = value != 0; break;
    case BROTLI_PARAM_BYTE_ALIGN: q.byte_align = value != 0; break;
    case BROTLI_PARAM_BARE_STREAM: q.bare_stream = value != 0; if (!q.byte_align) q.byte_align = value != 0; break;
    default:
      // research / divans knobs of the reference (stride, prior, cdf speeds ...) have no effect on this path
      if (!(key >= 151 && key <= 173)) return false;
  }
  p = q;
  return true;
}

bool parse_params(EncoderParams* p, size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values) {
  if (num_params && (!keys || !values)) return false;
  for (size_t i = 0; i < num_params; ++i)
    if (!apply_param(*p, (int)keys[i], values[i])) return false;
  return true;
}

struct DeviceGuard {  // every entry point leaves the caller's current CUDA device as it found it
  int prev = -1;
  DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// one lazily created encoder per device for the state-less entry points
std::mutex g_mu;
std::vector<B200Encoder*> g_encoders;
std::vector<std::mutex*> g_encoder_mu;

B200Encoder* shared_encoder(int device, std::mutex** mu) {
  std::lock_guard<std::mutex> lk(g_mu);
  int n = b200_device_count();
  if (n <= 0 || device >= n) return nullptr;
  if ((int)g_encoders.size() < n) {
    g_encoders.resize(n, nullptr);
    g_encoder_mu.resize(n, nullptr);
  }
  if (!g_encoders[device]) {
    g_encoders[device] = b200_encoder_create(device);
    g_encoder_mu[device] = new std::mutex();
  }
  *mu = g_encoder_mu[device];
  return g_encoders[device];
}

}  // namespace

// Stream state.  Input is buffered on the host; PROCESS turns it into output whenever kStreamPieceBytes are pending (the
// reference also emits as its blocks fill, encode.rs:2873-2995), FLUSH / FINISH emit whatever is pending.  Pieces end
// byte aligned (padding metablock), and only the last 2^lgwin bytes in front of the unflushed part are kept as match
// window, so a stream of any length needs a bounded buffer.  These decisions are stream_plan's (below), which the device
// stream (B200Stream) shares.
constexpr size_t kStreamPieceBytes = (size_t)4 * BRO_CHUNK_BYTES_CAPI;

// The custom dictionary rule (compressor.rs:162 / encode.rs:1205-1260): the last min(size, 2^lgwin - 16) bytes become window
// content in front of the stream (they occupy positions); a dictionary of at most one byte keeps nothing.  Returns the index
// of the first byte kept and sets the counters of the new stream.  The caller switches the static dictionary off.
static uint64_t stream_start(const EncoderParams& p, uint64_t size, B200StreamCounters* c) {
  memset(c, 0, sizeof(*c));
  if (size <= 1) return size;
  const uint64_t keep = std::min<uint64_t>(size, ((uint64_t)1 << window_bits(p)) - 16);
  c->dict_len = c->flushed = c->end = keep;
  return size - keep;
}

// One step of the stream (BrotliEncoderCompressStream with n new bytes): the emits to run, in order, and the counters after
// them.  An emit compresses [start, upto) against the bytes from `base` on (compress_framed, align_end) or is one end-of-stream
// byte; once it is done only the match window in front of the unflushed part is needed, from base_after on.
static void stream_plan(const EncoderParams& p, const B200StreamCounters& c0, int op, uint64_t n, std::vector<B200StreamEmit>* emits,
                        B200StreamCounters* next) {
  EncoderParams fp = p;
  sanitize_framing(fp);
  B200StreamCounters c = c0;
  c.end += n;
  const uint64_t window = rebase_window(p);
  const uint64_t hint = p.size_hint ? p.size_hint : c.end - c.dict_len;  // the input so far
  auto emit = [&](bool last, uint64_t upto) {
    B200StreamEmit m;
    memset(&m, 0, sizeof(m));
    m.start = c.flushed;
    m.upto = upto;
    m.base = m.base_after = c.base;
    m.size_hint = hint;
    m.first = !c.header_written;
    m.last = last;
    m.byte = -1;
    if (upto == c.flushed && !(framed(fp) && m.first)) {  // nothing to compress (only FINISH gets here)
      if (!last || (!m.first && fp.bare_stream)) return;
      m.byte = m.first ? 6 : 3;  // empty stream (encode.rs:1463) / ISLAST + ISLASTEMPTY after a byte-aligned flush
      c.header_written = 1;
      emits->push_back(m);
      return;
    }
    c.flushed = upto;
    c.header_written = 1;
    if (c.flushed > c.base + window) {  // keep only the match window in front of the unflushed part
      const uint64_t keep_from = (c.flushed - window) & ~(uint64_t)4095;
      if (keep_from > c.base) c.base = keep_from;
    }
    m.base_after = c.base;
    emits->push_back(m);
  };
  if (op == BROTLI_OPERATION_PROCESS) {
    while (c.end - c.flushed >= 2 * kStreamPieceBytes) emit(false, c.flushed + kStreamPieceBytes);  // keep one piece back for FINISH
  } else if (op == BROTLI_OPERATION_FLUSH) {
    if (c.flushed < c.end) emit(false, c.end);
  } else if (op == BROTLI_OPERATION_FINISH && !c.finished) {
    emit(true, c.end);
    c.finished = 1;
  }
  *next = c;
}

struct BrotliEncoderStateStruct {
  EncoderParams params;
  B200Encoder* enc = nullptr;
  brotli_alloc_func alloc_func = nullptr;  // compressor.rs:60-100: kept for BrotliEncoderMalloc* / Free*
  brotli_free_func free_func = nullptr;
  void* opaque = nullptr;
  std::vector<uint8_t> input;   // stream bytes [c.base, c.end)
  B200StreamCounters c{};       // offsets are absolute; the custom dictionary counts as positions (encode.rs:1247)
  std::vector<uint8_t> output;  // produced, not yet taken
  size_t out_pos = 0;
  uint64_t total_out = 0;       // bytes handed to the caller so far (total_out_, encode.rs:181)
  bool started = false;
};

struct BrotliEncoderWorkPoolStruct {
  size_t num_workers;
  std::vector<B200Encoder*> encoders;  // one per visible GPU
  std::vector<std::mutex*> mus;        // calls that share the pool are serialised per encoder (threading/mod.rs work pool)
};

// ---- stream framing (catable / appendable / magic_number / byte_align / bare_stream) ----
struct HostBits {  // LSB-first bit writer into a bounded host buffer
  uint8_t* out; size_t cap; uint64_t pos = 0; bool ok = true;
  void put(uint32_t nbits, uint64_t v) {
    for (uint32_t i = 0; i < nbits; ++i, ++pos) {
      if ((pos >> 3) >= cap) { ok = false; return; }
      if ((pos & 7) == 0) out[pos >> 3] = 0;
      out[pos >> 3] |= (uint8_t)(((v >> i) & 1u) << (pos & 7));
    }
  }
  void align() { while (ok && (pos & 7)) put(1, 0); }
  void bytes(const uint8_t* p, size_t n) { for (size_t i = 0; i < n; ++i) put(8, p[i]); }
};
static void put_window_bits(HostBits& w, int lgwin) {  // EncodeWindowBits encode.rs:600-627 (no large window)
  if (lgwin == 16) w.put(1, 0);
  else if (lgwin == 17) w.put(7, 1);
  else if (lgwin > 17) w.put(4, (uint64_t)(((lgwin - 17) << 1) | 1));
  else w.put(7, (uint64_t)(((lgwin - 8) << 4) | 1));
}
// The prologue of a framed stream of `len` bytes (p sanitised): [window bits unless catable && bare] [magic-number metadata
// metablock, brotli_bit_stream.rs:2869-2896] [catable: the first min(2, len) bytes as an uncompressed metablock,
// encode.rs:2285-2333 -- a stitched stream's literal contexts then never look into the previous file].  Zeros stand in for those
// bytes; *data_off / *n2: where they are and how many.
static void write_prologue(HostBits& w, const EncoderParams& p, size_t len, size_t* data_off, size_t* n2) {
  *data_off = 0;
  *n2 = 0;
  if (!(p.catable && p.bare_stream)) put_window_bits(w, window_bits(p));
  if (p.magic_number) {
    uint8_t sh[10]; size_t nsh = 0;
    for (uint64_t v = p.size_hint;;) {  // encode_base_128 brotli_bit_stream.rs:2855-2867
      sh[nsh] = (uint8_t)(v & 0x7f); v >>= 7;
      if (v) sh[nsh++] |= 0x80; else { ++nsh; break; }
      if (nsh == 10) break;
    }
    w.put(1, 0); w.put(2, 3); w.put(1, 0); w.put(2, 1); w.put(8, 3 + nsh);
    w.align();
    const uint8_t magic[4] = {0xe1, 0x97, (uint8_t)(p.catable ? 0x81 : (p.appendable ? 0x82 : 0x80)), 1 /* crate VERSION, lib.rs:67 */};
    w.bytes(magic, 4);
    w.bytes(sh, nsh);
  }
  if (p.catable && len) {
    *n2 = std::min<size_t>(2, len);
    w.put(1, 0); w.put(2, 0); w.put(16, *n2 - 1); w.put(1, 1);  // ISLAST 0, MNIBBLES 4, MLEN - 1, ISUNCOMPRESSED
    w.align();
    *data_off = (size_t)(w.pos >> 3);
    const uint8_t zeros[2] = {0, 0};
    w.bytes(zeros, *n2);
  }
}
// The end of a framed stream with nothing (left) to compress behind the prologue (WriteEmptyLastBlocksInternal
// encode.rs:1928-1940): last: [byte_align: padding metablock][unless bare: the empty last metablock]; else padding if asked.
static void write_empty_trailer(HostBits& w, const EncoderParams& p, bool last, bool align_end) {
  if (last) {
    if (p.byte_align && (w.pos & 7)) { w.put(6, 6); w.align(); }  // BrotliWritePaddingMetaBlock
    if (!p.bare_stream) { w.put(2, 3); w.align(); }
  } else if (align_end && (w.pos & 7)) { w.put(6, 6); w.align(); }
}

// How input bytes [a, b) become output: the prologue, the output of each device call in order, then the trailer byte.  Every
// entry point executes this plan: compress_framed on the host, b200_encoder_compress_params_async and the device stream.
struct FramedPlan {
  bool has_pro = false;
  B200Prologue pro{};                 // its n2 data bytes are zeros: the executor puts input bytes a, a + 1 there
  std::vector<B200FramedCall> calls;  // at least one: a complete prologue goes with one call that compresses nothing
  int trailer = -1;                   // appended behind the last call
  int ctx_model = 1, use_dict = 1;    // the encoder options of every call (catable switches the static dictionary off)
  int q9_5 = 0;
};

// first / last: the stream header / its end belong to [a, b); align_end: when not last, the output ends byte aligned.  A framed
// stream's header is a host-built prologue when it carries more than the window bits, or when there is nothing to compress; the
// device writes a plain 2-bit ending itself, a byte-aligned one ends with trailer byte 3.  Data metablocks never carry ISLAST on
// this path, so "appendable" (encode.rs:1973-1975) needs nothing more, and every metablock starts with an unknown distance cache,
// which is what catable's 0x7ffffff0 cache (encode.rs:693-703) asks for.  Positions inside the device encoder are 32-bit, so the
// body is cut into calls of at most kSpanPiece bytes, each handed over from a base at most one rebase window in front of it;
// calls in the middle end byte aligned.  Returns false when the output could not end on a byte boundary.
constexpr size_t kSpanPiece = (size_t)1 << 30;
static bool framed_plan(EncoderParams p, uint64_t a, uint64_t b, bool first, bool last, bool align_end, FramedPlan* f) {
  sanitize_framing(p);
  f->ctx_model = p.disable_ctx ? 0 : 1;
  f->use_dict = p.no_dictionary ? 0 : 1;
  f->q9_5 = p.q9_5;
  f->has_pro = framed(p) && ((first && (p.magic_number || p.catable)) || a == b);
  uint64_t body_a = a;
  if (f->has_pro) {
    HostBits w{f->pro.bytes, sizeof(f->pro.bytes)};
    size_t data_off = 0, n2 = 0;
    if (first) write_prologue(w, p, b - a, &data_off, &n2);
    body_a += n2;
    if (body_a == b) write_empty_trailer(w, p, last, align_end);
    if (!w.ok || (w.pos & 7)) return false;
    f->pro.len = (uint32_t)(w.pos >> 3);
    f->pro.data_off = (uint32_t)data_off;
    f->pro.n2 = (uint32_t)n2;
    f->pro.complete = body_a == b;
  }
  const bool dev_first = first && !f->has_pro, dev_last = last && !p.byte_align && !p.bare_stream;
  const bool dev_align = last ? p.byte_align != 0 : align_end;
  if (body_a < b && last && p.byte_align && !p.bare_stream) f->trailer = 3;  // ISLAST + ISLASTEMPTY on a byte boundary
  const uint64_t window = rebase_window(p);
  for (uint64_t s = body_a;;) {
    const uint64_t e = std::min<uint64_t>(b, s + kSpanPiece);
    const bool l = e == b;
    // once a full window precedes `s`, min(position, 2^lgwin - 16) is the same in rebased coordinates
    f->calls.push_back(B200FramedCall{s > window ? ((s - window) & ~(uint64_t)4095) : 0, s, e, dev_first && s == body_a,
                                      dev_last && l, l ? (dev_align && !dev_last) : true});
    if (l) return true;
    s = e;
  }
}

// Compresses input[a, b) into out (host): framed_plan's prologue with its data bytes, each call through the blocking device path,
// then the trailer byte.
static bool compress_framed(B200Encoder* enc, const EncoderParams& p, uint64_t hint, const uint8_t* input, size_t a, size_t b,
                            bool first, bool last, bool align_end, uint8_t* out, size_t out_cap, size_t* out_size) {
  FramedPlan f;
  if (!framed_plan(p, a, b, first, last, align_end, &f) || f.pro.len > out_cap) return false;
  std::copy(f.pro.bytes, f.pro.bytes + f.pro.len, out);
  std::copy(input + a, input + a + f.pro.n2, out + f.pro.data_off);
  size_t off = f.pro.len;
  b200_encoder_set_option(enc, B200_OPT_CTX_MODEL, f.ctx_model);
  b200_encoder_set_option(enc, B200_OPT_DICT, f.use_dict);
  b200_encoder_set_option(enc, B200_OPT_Q9_5, f.q9_5);
  for (const B200FramedCall& c : f.calls) {
    size_t got = 0;
    if (!b200_encoder_compress_range(enc, p.quality, p.lgwin, hint, input + c.rebase, c.end - c.rebase, c.start - c.rebase,
                                     c.end - c.start, c.first, c.last, c.byte_align, out + off, out_cap - off, &got, 0))
      return false;
    off += got;
  }
  if (f.trailer >= 0) {
    if (off >= out_cap) return false;
    out[off++] = (uint8_t)f.trailer;
  }
  *out_size = off;
  return true;
}

// Enqueues call i of plan f over `in` on the device, stream-ordered: a kernel writes the prologue in front of the first call's
// output (its data bytes are the input in front of that call's range), and the trailer byte follows the last.
static int enqueue_framed_call(B200Encoder* e, const EncoderParams& p, uint64_t hint, const FramedPlan& f, size_t i, const uint8_t* in,
                               uint8_t* out, size_t out_cap, uint64_t* out_size, void* stream) {
  const B200FramedCall& c = f.calls[i];
  return b200_encoder_compress_framed_async(e, p.quality, p.lgwin, hint, f.ctx_model, f.use_dict, f.q9_5, in + c.rebase, c.end - c.rebase,
                                            c.start - c.rebase, c.end - c.start, c.first, c.last, c.byte_align,
                                            (f.has_pro && i == 0) ? &f.pro : nullptr, i + 1 == f.calls.size() ? f.trailer : -1, out,
                                            out_cap, out_size, stream);
}

extern "C" {

uint32_t BrotliEncoderVersion(void) { return 0x08000004u; /* tracks crate 8.0.4 */ }

size_t BrotliEncoderMaxCompressedSize(size_t input_size) {  // encode.rs:1277-1299, the reference's arithmetic as it stands
  const size_t magic_size = 16;
  const size_t num_large_blocks = input_size >> 14;
  const size_t tail = input_size - (num_large_blocks << 24);  // wraps, as the reference's wrapping_sub does
  const size_t tail_overhead = tail > ((size_t)1 << 20) ? 4 : 3;
  const size_t overhead = 2 + 4 * num_large_blocks + tail_overhead + 1;
  const size_t result = input_size + overhead;
  if (input_size == 0) return 1 + magic_size;
  return result < input_size ? 0 : result + magic_size;
}
size_t BrotliEncoderMaxCompressedSizeMulti(size_t input_size, size_t num_threads) {  // encode.rs:1273-1275
  return BrotliEncoderMaxCompressedSize(input_size) + num_threads * 8;
}

BrotliEncoderState* BrotliEncoderCreateInstance(brotli_alloc_func alloc_func, brotli_free_func free_func, void* opaque) {
  DeviceGuard dg;
  if (alloc_func && !free_func) return nullptr;  // "either both alloc and free must exist or neither" (compressor.rs:84)
  if (alloc_func) {  // honour "allocator returns NULL => NULL instance" (compressor.rs:97-99, :452-473)
    void* probe = alloc_func(opaque, sizeof(BrotliEncoderStateStruct));
    if (!probe) return nullptr;
    free_func(opaque, probe);
  }
  B200Encoder* enc = b200_encoder_create(0);
  if (!enc) return nullptr;
  BrotliEncoderStateStruct* s = new (std::nothrow) BrotliEncoderStateStruct();
  if (!s) { b200_encoder_destroy(enc); return nullptr; }
  s->enc = enc;
  s->alloc_func = alloc_func;
  s->free_func = free_func;
  s->opaque = opaque;
  return s;
}
void BrotliEncoderDestroyInstance(BrotliEncoderState* s) {
  if (!s) return;
  DeviceGuard dg;
  b200_encoder_destroy(s->enc);
  delete s;
}
BROTLI_BOOL BrotliEncoderSetParameter(BrotliEncoderState* s, BrotliEncoderParameter p, uint32_t value) {
  if (!s || s->started) return BROTLI_FALSE;  // encode.rs:289-295
  return apply_param(s->params, (int)p, value) ? BROTLI_TRUE : BROTLI_FALSE;
}
// compressor.rs:162 / encode.rs:1205-1260: the dictionary rule of stream_start, the static dictionary is switched off.
// Ignored once input was consumed.
void BrotliEncoderSetCustomDictionary(BrotliEncoderState* s, size_t size, const uint8_t* dict) {
  if (!s || s->started || s->c.dict_len != 0) return;
  s->params.no_dictionary = 1;
  if (size <= 1 || !dict) return;
  const uint64_t from = stream_start(s->params, size, &s->c);
  s->input.assign(dict + from, dict + size);
}
uint8_t* BrotliEncoderMallocU8(BrotliEncoderState* s, size_t size) {  // compressor.rs:359-371
  if (s && s->alloc_func) return (uint8_t*)s->alloc_func(s->opaque, size);
  return (uint8_t*)calloc(size ? size : 1, 1);
}
void BrotliEncoderFreeU8(BrotliEncoderState* s, uint8_t* data, size_t size) {  // :373-388
  (void)size;
  if (s && s->free_func) s->free_func(s->opaque, data);
  else free(data);
}
size_t* BrotliEncoderMallocUsize(BrotliEncoderState* s, size_t size) {  // :390-403
  if (s && s->alloc_func) return (size_t*)s->alloc_func(s->opaque, size * sizeof(size_t));
  return (size_t*)calloc(size ? size : 1, sizeof(size_t));
}
void BrotliEncoderFreeUsize(BrotliEncoderState* s, size_t* data, size_t size) {  // :404-419
  (void)size;
  if (s && s->free_func) s->free_func(s->opaque, data);
  else free(data);
}

// Runs one emit of stream_plan and appends its output to the output queue.
static bool state_emit(BrotliEncoderStateStruct* s, const B200StreamEmit& m) {
  if (m.byte >= 0) {
    s->output.push_back((uint8_t)m.byte);
    s->c.header_written = 1;
    return true;
  }
  const uint64_t len = m.upto - m.start;
  size_t cap = b200_max_compressed_size(len) + 64, got = 0;
  size_t old = s->output.size();
  s->output.resize(old + cap);
  // positions are relative to `base`: once a prefix has been dropped at least a full window precedes `start`, so the
  // window limit min(position, 2^lgwin - 16) is the same in both coordinate systems
  bool ok = compress_framed(s->enc, s->params, m.size_hint, s->input.data(), (size_t)(m.start - m.base), (size_t)(m.upto - m.base),
                            m.first != 0, m.last != 0, true, s->output.data() + old, cap, &got);
  if (!ok) { s->output.resize(old); return false; }
  s->output.resize(old + got);
  s->c.flushed = m.upto;
  s->c.header_written = 1;
  if (m.base_after > s->c.base) {  // keep only the match window in front of the unflushed part
    s->input.erase(s->input.begin(), s->input.begin() + (size_t)(m.base_after - s->c.base));
    s->c.base = m.base_after;
  }
  return true;
}

BROTLI_BOOL BrotliEncoderCompressStream(BrotliEncoderState* s, BrotliEncoderOperation op, size_t* available_in,
                                        const uint8_t** next_in, size_t* available_out, uint8_t** next_out, size_t* total_out) {
  if (!s || !available_in || !available_out) return BROTLI_FALSE;
  if (op == BROTLI_OPERATION_EMIT_METADATA) return BROTLI_FALSE;  // not on this path
  DeviceGuard dg;
  const size_t n = *available_in;
  if (n) {
    if (s->c.finished || !next_in || !*next_in) return BROTLI_FALSE;
    s->started = true;
    s->input.insert(s->input.end(), *next_in, *next_in + n);
    *next_in += n;
    *available_in = 0;
  }
  std::vector<B200StreamEmit> plan;
  B200StreamCounters next;
  stream_plan(s->params, s->c, (int)op, n, &plan, &next);
  if ((op == BROTLI_OPERATION_FLUSH && s->c.flushed < next.end) || (op == BROTLI_OPERATION_FINISH && !s->c.finished)) s->started = true;
  s->c.end = next.end;
  for (const B200StreamEmit& m : plan)
    if (!state_emit(s, m)) return BROTLI_FALSE;
  s->c.finished = next.finished;
  size_t avail = s->output.size() - s->out_pos;
  if (avail && *available_out && next_out && *next_out) {
    size_t n = std::min(avail, *available_out);
    memcpy(*next_out, s->output.data() + s->out_pos, n);
    *next_out += n;
    *available_out -= n;
    s->out_pos += n;
    s->total_out += n;
  }
  if (total_out) *total_out = (size_t)s->total_out;  // the cumulative count is assigned (encode.rs:1591-1593, :2824-2826)
  if (s->out_pos == s->output.size()) { s->output.clear(); s->out_pos = 0; }
  return BROTLI_TRUE;
}
// compressor.rs:260-278: same call with the buffer pointers passed by value and no total_out
BROTLI_BOOL BrotliEncoderCompressStreaming(BrotliEncoderState* s, BrotliEncoderOperation op, size_t* available_in,
                                           const uint8_t* input_buf, size_t* available_out, uint8_t* output_buf) {
  return BrotliEncoderCompressStream(s, op, available_in, &input_buf, available_out, &output_buf, nullptr);
}
BROTLI_BOOL BrotliEncoderIsFinished(BrotliEncoderState* s) { return (s && s->c.finished && s->out_pos == s->output.size()) ? 1 : 0; }
BROTLI_BOOL BrotliEncoderHasMoreOutput(BrotliEncoderState* s) { return (s && s->out_pos < s->output.size()) ? 1 : 0; }
const uint8_t* BrotliEncoderTakeOutput(BrotliEncoderState* s, size_t* size) {  // encode.rs:3006-3027
  if (!s || !size) return nullptr;
  size_t avail = s->output.size() - s->out_pos;
  size_t n = *size ? std::min(*size, avail) : avail;  // *size == 0 asks for everything that is available
  const uint8_t* p = s->output.data() + s->out_pos;   // (the reference returns its next_out pointer even when n == 0)
  if (n == 0) { *size = 0; return avail ? p : nullptr; }
  s->out_pos += n;
  s->total_out += n;
  *size = n;
  return p;
}

BROTLI_BOOL BrotliEncoderCompress(int quality, int lgwin, BrotliEncoderMode mode, size_t input_size, const uint8_t* input,
                                  size_t* encoded_size, uint8_t* encoded) {
  (void)mode;
  if (!encoded_size || *encoded_size == 0) return BROTLI_FALSE;  // encode.rs:1459-1462
  const size_t out_cap = *encoded_size;
  if (input_size == 0) { encoded[0] = 6; *encoded_size = 1; return BROTLI_TRUE; }
  DeviceGuard dg;
  std::mutex* mu = nullptr;
  B200Encoder* enc = shared_encoder(0, &mu);
  if (!enc) { *encoded_size = 0; return BROTLI_FALSE; }
  size_t got = 0;
  bool ok;
  {
    std::lock_guard<std::mutex> lk(*mu);
    EncoderParams p;
    p.quality = quality;
    p.lgwin = lgwin;
    ok = compress_framed(enc, p, input_size, input, 0, input_size, true, true, false, encoded, out_cap, &got);
  }
  if (!ok) {  // no CPU-produced stream, ever: a device failure (or a too-small output buffer) is reported as failure
    *encoded_size = 0;
    return BROTLI_FALSE;
  }
  *encoded_size = got;
  return BROTLI_TRUE;
}

// One complete stream of the n device bytes at `in`, stream-ordered on `stream`: framed_plan(0, n, first, last) -- which
// BrotliEncoderCompressStream with one FINISH runs -- enqueued as its one device call.
int b200_encoder_compress_params_async(B200Encoder* e, size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values,
                                       const uint8_t* in, size_t n, uint8_t* out, size_t out_cap, uint64_t* out_size, void* stream) {
  if (!e) return 0;
  if (n >= kSpanPiece) return 0;  // one call: longer inputs are cut into several (a catable body starts two bytes in)
  if (out_cap < b200_max_compressed_size(n) + 64) return 0;
  EncoderParams p;
  FramedPlan f;
  if (!parse_params(&p, num_params, keys, values) || !framed_plan(p, 0, n, true, true, true, &f)) return 0;
  return enqueue_framed_call(e, p, p.size_hint ? p.size_hint : n, f, 0, in, out, out_cap, out_size, stream);
}

// ---- multi ----
static std::atomic<uint32_t> g_last_multi_mask{0};  // bit d set: device d compressed at least one shard of the last multi call
uint32_t b200_last_multi_device_mask(void) { return g_last_multi_mask.load(); }

static int32_t compress_multi_impl(const std::vector<B200Encoder*>& encs, const std::vector<std::mutex*>& mus, size_t num_params,
                                   const BrotliEncoderParameter* keys, const uint32_t* values, size_t input_size,
                                   const uint8_t* input, size_t* encoded_size, uint8_t* encoded, size_t desired_num_threads) {
  if (!encoded_size || encs.empty() || desired_num_threads == 0) return 0;  // multicompress/mod.rs:106-108
  EncoderParams p;
  for (size_t i = 0; i < num_params; ++i)
    if (!apply_param(p, (int)keys[i], values[i])) return 0;  // a parameter this path cannot honour fails the call
  size_t shards = std::min<size_t>(desired_num_threads, 16);  // MAX_THREADS, fixed_queue.rs:1
  if (input_size == 0) {
    EncoderParams fp = p;
    sanitize_framing(fp);
    if (framed(fp)) {  // header / magic number / trailer of an empty framed stream
      uint8_t tmp[64];
      size_t got = 0;
      if (!compress_framed(encs[0], p, 0, input, 0, 0, true, true, false, tmp, sizeof(tmp), &got) || got > *encoded_size) return 0;
      memcpy(encoded, tmp, got);
      *encoded_size = got;
      return 1;
    }
    if (*encoded_size < 1) return 0;
    encoded[0] = 6;
    *encoded_size = 1;
    return 1;
  }
  if (shards > input_size) shards = input_size;
  std::vector<std::vector<uint8_t>> outs(shards);
  std::vector<int> oks(shards, 0);
  const size_t ngpu = encs.size();
  g_last_multi_mask.store(0);
  auto work = [&](size_t g) {  // one host thread per GPU walks its shards in order
    DeviceGuard dg;
    if (g < shards) g_last_multi_mask.fetch_or(1u << (b200_encoder_device(encs[g]) & 31));
    for (size_t i = g; i < shards; i += ngpu) {
      size_t a = i * input_size / shards, b = (i + 1) * input_size / shards;  // get_range threading/mod.rs:333
      size_t cap = b200_max_compressed_size(b - a) + 16 * ((b - a) / kSpanPiece + 1) + 64, got = 0;
      outs[i].resize(cap);
      std::lock_guard<std::mutex> lk(*mus[g]);
      // compress_part threading/mod.rs:337-383: size_hint = shard length
      uint64_t hint = p.size_hint ? p.size_hint : (b - a);
      oks[i] = compress_framed(encs[g], p, hint, input, a, b, i == 0, i + 1 == shards, true, outs[i].data(), cap, &got) ? 1 : 0;
      outs[i].resize(oks[i] ? got : 0);
    }
  };
  std::vector<std::thread> th;
  for (size_t g = 1; g < std::min(ngpu, shards); ++g) th.emplace_back(work, g);
  work(0);
  for (auto& t : th) t.join();  // always join every worker, first error wins (threading/mod.rs:565-660)
  size_t total = 0;
  for (size_t i = 0; i < shards; ++i) {
    if (!oks[i]) return 0;
    total += outs[i].size();
  }
  if (total > *encoded_size) return 0;  // BrotliEncoderThreadError::InsufficientOutputSpace
  size_t off = 0;
  for (size_t i = 0; i < shards; ++i) {  // shards end byte aligned: concatenation is a plain copy
    memcpy(encoded + off, outs[i].data(), outs[i].size());
    off += outs[i].size();
  }
  *encoded_size = total;
  return 1;
}

int32_t BrotliEncoderCompressMulti(size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values, size_t input_size,
                                   const uint8_t* input, size_t* encoded_size, uint8_t* encoded, size_t desired_num_threads,
                                   brotli_alloc_func alloc_func, brotli_free_func free_func, void** alloc_opaque_per_thread) {
  (void)alloc_func; (void)free_func; (void)alloc_opaque_per_thread;
  DeviceGuard dg;
  int n = b200_device_count();
  if (n <= 0) return 0;
  std::vector<B200Encoder*> encs;
  std::vector<std::mutex*> mus;
  for (int d = 0; d < n; ++d) {
    std::mutex* mu = nullptr;
    B200Encoder* e = shared_encoder(d, &mu);
    if (!e) return 0;
    encs.push_back(e);
    mus.push_back(mu);
  }
  return compress_multi_impl(encs, mus, num_params, keys, values, input_size, input, encoded_size, encoded, desired_num_threads);
}

BrotliEncoderWorkPool* BrotliEncoderCreateWorkPool(size_t num_workers, brotli_alloc_func alloc_func, brotli_free_func free_func,
                                                   void** alloc_opaque_per_thread) {
  if (alloc_func) {  // NULL-returning allocator => NULL pool (multicompress/test.rs)
    void* probe = alloc_func(alloc_opaque_per_thread ? alloc_opaque_per_thread[0] : nullptr, 64);
    if (!probe) return nullptr;
    if (free_func) free_func(alloc_opaque_per_thread ? alloc_opaque_per_thread[0] : nullptr, probe);
  }
  DeviceGuard dg;
  int n = b200_device_count();
  if (n <= 0) return nullptr;
  BrotliEncoderWorkPoolStruct* pool = new (std::nothrow) BrotliEncoderWorkPoolStruct();
  if (!pool) return nullptr;
  pool->num_workers = num_workers;
  size_t want = std::max<size_t>(1, std::min<size_t>(num_workers ? num_workers : 1, (size_t)n));
  for (size_t d = 0; d < want; ++d) {
    B200Encoder* e = b200_encoder_create((int)d);
    if (!e) {
      BrotliEncoderDestroyWorkPool(pool);
      return nullptr;
    }
    pool->encoders.push_back(e);
    pool->mus.push_back(new std::mutex());
  }
  return pool;
}
void BrotliEncoderDestroyWorkPool(BrotliEncoderWorkPool* pool) {
  if (!pool) return;
  DeviceGuard dg;
  for (auto* e : pool->encoders) b200_encoder_destroy(e);
  for (auto* m : pool->mus) delete m;
  delete pool;
}
int32_t BrotliEncoderCompressWorkPool(BrotliEncoderWorkPool* pool, size_t num_params, const BrotliEncoderParameter* keys,
                                      const uint32_t* values, size_t input_size, const uint8_t* input, size_t* encoded_size,
                                      uint8_t* encoded, size_t desired_num_threads, brotli_alloc_func alloc_func,
                                      brotli_free_func free_func, void** alloc_opaque_per_thread) {
  (void)alloc_func; (void)free_func; (void)alloc_opaque_per_thread;
  if (!pool) return BrotliEncoderCompressMulti(num_params, keys, values, input_size, input, encoded_size, encoded,
                                               desired_num_threads, nullptr, nullptr, nullptr);
  DeviceGuard dg;
  return compress_multi_impl(pool->encoders, pool->mus, num_params, keys, values, input_size, input, encoded_size, encoded,
                             desired_num_threads);
}

}  // extern "C"

// ---- device-resident streams (b200_stream_*): stream_plan's emits, compressed and appended on the device ----

// One piece of a device stream onto the caller's output, stream-ordered: out[*cursor, *cursor + size) = src[0, size) and the
// cursor advances; size is *d_size (src != nullptr), 1 (the single byte `byte`) or 0 (the call only reports the status).  A piece
// that does not fit in out_cap is not written at all and fails the stream: state[0] = 2, and a failed stream appends nothing more.
// *status = state[0] afterwards.  Every block reads the cursor before it counts itself done in state[1]; the last block moves the
// cursor and resets the count.  The copy writes aligned 32-bit words of the output, each put together from two words of the
// source (4-byte aligned, readable up to size + 8 bytes), and single bytes at the two ends.
__global__ void __launch_bounds__(256) k_stream_append(const uint8_t* src, const uint64_t* d_size, int byte, uint8_t* out,
                                                      uint64_t out_cap, uint64_t* cursor, int32_t* status, uint32_t* state) {
  __shared__ uint64_t s_at, s_n;
  __shared__ int s_ok;
  if (threadIdx.x == 0) {
    s_at = *cursor;
    s_n = src ? *d_size : (byte >= 0 ? 1 : 0);
    s_ok = state[0] == 0 && s_at <= out_cap && s_n <= out_cap - s_at;
  }
  __syncthreads();
  const uint64_t at = s_at, n = s_n;
  if (s_ok && n) {
    uint8_t* dst = out + at;
    if (!src) {
      if (blockIdx.x == 0 && threadIdx.x == 0) dst[0] = (uint8_t)byte;
    } else {
      const uint32_t d = (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 3);  // dst[0] is byte d of the first output word
      uint32_t* dw = reinterpret_cast<uint32_t*>(dst - d);
      const uint32_t* sw = reinterpret_cast<const uint32_t*>(src);
      const uint64_t nw = (d + n + 3) >> 2;
      for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < nw; k += (uint64_t)gridDim.x * blockDim.x) {
        // output word k holds source bytes [4k - d, 4k - d + 4): the high bytes of source word k - 1, the low bytes of word k
        const uint32_t v = __funnelshift_l(k ? sw[k - 1] : 0u, sw[k], 8 * d);
        const int64_t r = 4 * (int64_t)k - d;
        if (r >= 0 && r + 4 <= (int64_t)n) {
          dw[k] = v;
        } else {
          for (int j = 0; j < 4; ++j)
            if (r + j >= 0 && r + j < (int64_t)n) dst[r + j] = (uint8_t)(v >> (8 * j));
        }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&state[1], 1u) == gridDim.x - 1) {
      if (s_ok) *cursor = at + n;
      else if (state[0] == 0) state[0] = 2;
      state[1] = 0;
      *status = (int32_t)state[0];
    }
  }
}

struct B200Stream {
  B200Encoder* enc = nullptr;
  int device = 0;
  EncoderParams params;                  // as applied, the custom dictionary's "no static dictionary" included
  B200StreamCounters c{};
  uint8_t* win[2] = {nullptr, nullptr};  // window buffers of win_cap bytes; win[cur][0] holds stream byte win_base
  size_t win_cap = 0;
  int cur = 0;
  uint64_t win_base = 0;
  uint8_t* scratch = nullptr;            // the compressed bytes of one piece
  size_t scratch_cap = 0;
  uint64_t* d_word = nullptr;            // [0] the piece's size; [1] k_stream_append's state: failed, blocks done (2 x u32)
  cudaStream_t last = nullptr;           // the CUDA stream of the last call: b200_stream_destroy frees there
  cudaEvent_t ev_done = nullptr;         // the end of the last call
  bool failed = false;                   // a device failure inside a call: later calls are refused
};

namespace {

bool on_gpu(const void* p, int device) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device;
}

bool stream_capturing(cudaStream_t st) {  // true also when the status cannot be read: the call is then refused
  cudaStreamCaptureStatus cs;
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) {
    cudaGetLastError();
    return true;
  }
  return cs != cudaStreamCaptureStatusNone;
}

// The framing of one emit of stream_plan: its range of the window buffer, whose first byte is stream offset m.base.
bool plan_emit(const EncoderParams& p, const B200StreamEmit& m, FramedPlan* f) {
  return framed_plan(p, m.start - m.base, m.upto - m.base, m.first != 0, m.last != 0, true, f);
}

// The input bytes the output of call i stands for: its range and, for the first call, the prologue's data bytes.
size_t call_piece(const FramedPlan& f, size_t i) { return (size_t)(f.calls[i].end - f.calls[i].start) + (i ? 0 : f.pro.n2); }

// Output bound of one call: the slack b200_encoder_compress_framed_async asks for, plus a prologue and a trailer byte.
size_t piece_bound(size_t piece) { return b200_max_compressed_size(piece) + 64 + sizeof(B200Prologue::bytes) + 1; }

// Output bound and largest piece of one emit.
size_t emit_bound(const EncoderParams& p, const B200StreamEmit& m, size_t* max_piece) {
  if (m.byte >= 0) return 1;
  FramedPlan f;
  if (!plan_emit(p, m, &f)) return 0;  // the call then fails before it appends anything
  size_t bound = 0;
  for (size_t i = 0; i < f.calls.size(); ++i) {
    *max_piece = std::max(*max_piece, call_piece(f, i));
    bound += piece_bound(call_piece(f, i));
  }
  return bound;
}

// Makes room for n more bytes behind the stream's end.  The kept bytes [base, end) move to the front through the other buffer
// (a copy between two distinct buffers: overlapping copies are undefined), or into a larger one.  All stream-ordered on st.
bool stream_room(B200Stream* s, uint64_t n, cudaStream_t st) {
  if (s->c.end + n - s->win_base <= s->win_cap) return true;
  const uint64_t live = s->c.end - s->c.base, want = live + n;
  const uint8_t* from = s->win[s->cur] + (s->c.base - s->win_base);
  if (want > s->win_cap) {
    const size_t cap = (size_t)(want + std::max<uint64_t>(want / 2, (uint64_t)1 << 20));
    void* p = nullptr;
    if (cudaMallocAsync(&p, cap, st) != cudaSuccess) return false;
    if (live && cudaMemcpyAsync(p, from, live, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return false;
    for (uint8_t*& w : s->win) {
      if (w) cudaFreeAsync(w, st);
      w = nullptr;
    }
    s->win[0] = static_cast<uint8_t*>(p);
    s->cur = 0;
    s->win_cap = cap;
  } else {
    const int to = s->cur ^ 1;
    if (!s->win[to] && cudaMallocAsync((void**)&s->win[to], s->win_cap, st) != cudaSuccess) return false;
    if (live && cudaMemcpyAsync(s->win[to], from, live, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return false;
    s->cur = to;
  }
  s->win_base = s->c.base;
  return true;
}

bool stream_append(B200Stream* s, const uint8_t* src, int byte, size_t bound, uint8_t* out, size_t out_cap, uint64_t* cursor,
                   int32_t* status, cudaStream_t st) {
  const size_t words = bound / 4 + 2;
  const unsigned blocks = (unsigned)std::min<size_t>(std::max<size_t>(1, (words + 255) / 256), 1056);  // 8 per SM at most
  k_stream_append<<<blocks, 256, 0, st>>>(src, s->d_word, byte, out, out_cap, cursor, status, reinterpret_cast<uint32_t*>(s->d_word + 1));
  return cudaGetLastError() == cudaSuccess;
}

// Runs one emit on the device: each call of its plan into the scratch buffer, then appended to the caller's output.
bool stream_run_emit(B200Stream* S, const B200StreamEmit& m, uint8_t* out, size_t out_cap, uint64_t* cursor, int32_t* status,
                     cudaStream_t st) {
  if (m.byte >= 0) return stream_append(S, nullptr, m.byte, 1, out, out_cap, cursor, status, st);
  FramedPlan f;
  if (!plan_emit(S->params, m, &f)) return false;
  const uint8_t* in = S->win[S->cur] + (m.base - S->win_base);
  for (size_t i = 0; i < f.calls.size(); ++i)
    if (!enqueue_framed_call(S->enc, S->params, m.size_hint, f, i, in, S->scratch, S->scratch_cap, S->d_word, st) ||
        !stream_append(S, S->scratch, -1, piece_bound(call_piece(f, i)), out, out_cap, cursor, status, st))
      return false;
  return true;
}

bool valid_op(int op) {
  return op == BROTLI_OPERATION_PROCESS || op == BROTLI_OPERATION_FLUSH || op == BROTLI_OPERATION_FINISH;
}

}  // namespace

extern "C" {

B200Stream* b200_stream_create(B200Encoder* e, size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values,
                               const uint8_t* d_dict, size_t dict_len, void* stream) {
  EncoderParams p;
  if (!e || (dict_len && !d_dict) || !parse_params(&p, num_params, keys, values)) return nullptr;
  DeviceGuard dg;
  const int device = b200_encoder_device(e);
  if (cudaSetDevice(device) != cudaSuccess) return nullptr;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (stream_capturing(st)) return nullptr;
  if (dict_len > 1 && !on_gpu(d_dict, device)) return nullptr;
  B200Stream* S = new (std::nothrow) B200Stream();
  if (!S) return nullptr;
  S->enc = e;
  S->device = device;
  S->last = st;
  uint64_t from = 0;
  if (d_dict) {  // BrotliEncoderSetCustomDictionary
    p.no_dictionary = 1;
    from = stream_start(p, dict_len, &S->c);
  }
  S->params = p;
  const uint64_t keep = S->c.end;
  S->c.end = 0;  // the window starts empty and receives the dictionary
  bool ok = cudaEventCreateWithFlags(&S->ev_done, cudaEventDisableTiming) == cudaSuccess &&
            cudaMallocAsync((void**)&S->d_word, 16, st) == cudaSuccess && cudaMemsetAsync(S->d_word, 0, 16, st) == cudaSuccess &&
            stream_room(S, keep, st);
  if (ok && keep) ok = cudaMemcpyAsync(S->win[S->cur], d_dict + from, keep, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
  S->c.end = keep;
  if (ok) ok = cudaEventRecord(S->ev_done, st) == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    b200_stream_destroy(S);
    return nullptr;
  }
  return S;
}

size_t b200_stream_output_bound(const B200Stream* S, BrotliEncoderOperation op, size_t n) {
  if (!S || S->failed || S->c.finished || !valid_op(op)) return 0;
  std::vector<B200StreamEmit> plan;
  B200StreamCounters next;
  stream_plan(S->params, S->c, (int)op, n, &plan, &next);
  size_t bound = 0, max_piece = 0;
  for (const B200StreamEmit& m : plan) bound += emit_bound(S->params, m, &max_piece);
  return bound;
}

int b200_stream_compress_async(B200Stream* S, BrotliEncoderOperation op, const uint8_t* d_in, size_t n, uint8_t* out, size_t out_cap,
                               uint64_t* d_out_size, int32_t* d_status, void* stream) {
  if (!S || S->failed || S->c.finished || !valid_op(op) || !out || !d_out_size || !d_status || (n && !d_in)) return 0;
  DeviceGuard dg;
  if (cudaSetDevice(S->device) != cudaSuccess) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (stream_capturing(st)) return 0;
  // (the pointer queries run in relaxed capture mode: under a global-mode capture on another stream they are no reason to fail)
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  if (cudaThreadExchangeStreamCaptureMode(&mode) != cudaSuccess) return 0;
  const bool placed = on_gpu(out, S->device) && on_gpu(d_out_size, S->device) && on_gpu(d_status, S->device) &&
                      (!n || on_gpu(d_in, S->device));
  cudaThreadExchangeStreamCaptureMode(&mode);
  if (!placed) return 0;
  std::vector<B200StreamEmit> plan;
  B200StreamCounters next;
  stream_plan(S->params, S->c, (int)op, n, &plan, &next);
  size_t max_piece = 0;
  for (const B200StreamEmit& m : plan) emit_bound(S->params, m, &max_piece);
  S->last = st;
  bool ok = cudaStreamWaitEvent(st, S->ev_done, 0) == cudaSuccess && stream_room(S, n, st);
  const size_t need = (b200_max_compressed_size(max_piece) + 128 + 15) & ~(size_t)15;
  if (ok && !plan.empty() && need > S->scratch_cap) {  // the old scratch is freed behind the work that reads it
    void* p = nullptr;
    ok = cudaMallocAsync(&p, need, st) == cudaSuccess;
    if (ok) {
      if (S->scratch) cudaFreeAsync(S->scratch, st);
      S->scratch = static_cast<uint8_t*>(p);
      S->scratch_cap = need;
    }
  }
  if (ok && n) ok = cudaMemcpyAsync(S->win[S->cur] + (S->c.end - S->win_base), d_in, n, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
  for (size_t i = 0; ok && i < plan.size(); ++i) ok = stream_run_emit(S, plan[i], out, out_cap, d_out_size, d_status, st);
  if (ok && plan.empty()) ok = stream_append(S, nullptr, -1, 0, out, out_cap, d_out_size, d_status, st);
  if (!ok) {  // part of the call may be enqueued: fail the stream on the device too, so that its status reads 2
    cudaGetLastError();
    S->failed = true;
    cudaMemsetAsync(S->d_word + 1, 2, 1, st);
    stream_append(S, nullptr, -1, 0, out, out_cap, d_out_size, d_status, st);
    cudaGetLastError();
    return 0;
  }
  S->c = next;
  cudaEventRecord(S->ev_done, st);
  return 1;
}

void b200_stream_destroy(B200Stream* S) {
  if (!S) return;
  DeviceGuard dg;
  cudaSetDevice(S->device);
  for (void* p : {(void*)S->win[0], (void*)S->win[1], (void*)S->scratch, (void*)S->d_word})
    if (p) cudaFreeAsync(p, S->last);
  if (S->ev_done) cudaEventDestroy(S->ev_done);
  cudaGetLastError();
  delete S;
}

int b200_stage_framed_plan(size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values, uint64_t a, uint64_t b,
                           int first, int last, int align_end, uint8_t* prologue, int32_t* prologue_info, B200FramedCall* calls,
                           size_t max_calls, size_t* num_calls, int32_t* trailer) {
  EncoderParams p;
  FramedPlan f;
  if (!prologue || !prologue_info || !num_calls || !trailer || b < a || !parse_params(&p, num_params, keys, values) ||
      !framed_plan(p, a, b, first != 0, last != 0, align_end != 0, &f) || f.calls.size() > max_calls || !calls)
    return 0;
  memcpy(prologue, f.pro.bytes, sizeof(f.pro.bytes));
  const int32_t info[4] = {f.has_pro ? (int32_t)f.pro.len : -1, (int32_t)f.pro.data_off, (int32_t)f.pro.n2, (int32_t)f.pro.complete};
  memcpy(prologue_info, info, sizeof(info));
  std::copy(f.calls.begin(), f.calls.end(), calls);
  *num_calls = f.calls.size();
  *trailer = f.trailer;
  return 1;
}

int b200_stage_stream_start(size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values, uint64_t dict_size,
                            B200StreamCounters* c, uint64_t* dict_from) {
  EncoderParams p;
  if (!c || !parse_params(&p, num_params, keys, values)) return 0;
  const uint64_t from = stream_start(p, dict_size, c);
  if (dict_from) *dict_from = from;
  return 1;
}

int b200_stage_stream_plan(size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values, const B200StreamCounters* c,
                           int op, uint64_t n, B200StreamEmit* emits, size_t max_emits, size_t* num_emits, B200StreamCounters* next) {
  EncoderParams p;
  if (!c || !next || !num_emits || !valid_op(op) || (n && c->finished) || !parse_params(&p, num_params, keys, values)) return 0;
  std::vector<B200StreamEmit> plan;
  stream_plan(p, *c, op, n, &plan, next);
  if (plan.size() > max_emits || (plan.size() && !emits)) return 0;
  std::copy(plan.begin(), plan.end(), emits);
  *num_emits = plan.size();
  return 1;
}

}  // extern "C"

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
    // stream framing (encode.rs:264-283; acted on by compress_framed below)
    case BROTLI_PARAM_CATABLE: q.catable = value != 0; if (!q.appendable) q.appendable = value != 0; break;
    case BROTLI_PARAM_APPENDABLE: q.appendable = value != 0; break;
    case BROTLI_PARAM_MAGIC_NUMBER: q.magic_number = value != 0; break;
    case BROTLI_PARAM_BYTE_ALIGN: q.byte_align = value != 0; break;
    case BROTLI_PARAM_BARE_STREAM: q.bare_stream = value != 0; if (!q.byte_align) q.byte_align = value != 0; break;
    default:
      // research / divans knobs of the reference (stride, prior, cdf speeds ...) have no effect on this path
      if (!(key >= 150 && key <= 173)) return false;
  }
  p = q;
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
// window, so a stream of any length needs a bounded buffer.
constexpr size_t kStreamPieceBytes = (size_t)4 * BRO_CHUNK_BYTES_CAPI;
struct BrotliEncoderStateStruct {
  EncoderParams params;
  B200Encoder* enc = nullptr;
  brotli_alloc_func alloc_func = nullptr;  // compressor.rs:60-100: kept for BrotliEncoderMalloc* / Free*
  brotli_free_func free_func = nullptr;
  void* opaque = nullptr;
  std::vector<uint8_t> input;   // stream bytes [base, base + input.size())
  uint64_t base = 0;            // absolute stream offset of input[0] (multiple of 4096)
  uint64_t flushed = 0;         // absolute offset up to which the stream has been turned into output
  uint64_t dict_len = 0;        // custom dictionary bytes in front of the stream (they count as positions, encode.rs:1247)
  std::vector<uint8_t> output;  // produced, not yet taken
  size_t out_pos = 0;
  uint64_t total_out = 0;       // bytes handed to the caller so far (total_out_, encode.rs:181)
  bool started = false, finished = false, header_written = false;
};

struct BrotliEncoderWorkPoolStruct {
  size_t num_workers;
  std::vector<B200Encoder*> encoders;  // one per visible GPU
  std::vector<std::mutex*> mus;        // calls that share the pool are serialised per encoder (threading/mod.rs work pool)
};

// Compresses input[a, b) of an n-byte stream into out (host).  Positions inside the device encoder are 32-bit, so the
// span is cut into pieces of at most kSpanPiece bytes, each handed over relative to a base at most one window in front of
// it; pieces in the middle end byte aligned.  first/last: stream header / final empty metablock belong to this span;
// align_end: a span that is not last ends byte aligned.
constexpr size_t kSpanPiece = (size_t)1 << 30;
static bool compress_span(B200Encoder* enc, const EncoderParams& p, uint64_t hint, const uint8_t* input, size_t a, size_t b,
                          bool first, bool last, bool align_end, uint8_t* out, size_t out_cap, size_t* out_size) {
  const int lw = p.lgwin < 10 ? 10 : (p.lgwin > 24 ? 24 : p.lgwin);
  const size_t window = ((size_t)1 << lw) + 65536;
  size_t off = 0;
  b200_encoder_set_option(enc, B200_OPT_CTX_MODEL, p.disable_ctx ? 0 : 1);
  b200_encoder_set_option(enc, B200_OPT_DICT, p.no_dictionary ? 0 : 1);
  for (size_t s = a; s < b || s == a;) {
    const size_t e = std::min(b, s + kSpanPiece);
    // once a full window precedes `s`, min(position, 2^lgwin - 16) is the same in rebased coordinates
    const size_t rb = s > window ? ((s - window) & ~(size_t)4095) : 0;
    size_t got = 0;
    const bool f = first && s == a, l = e == b;
    if (!b200_encoder_compress_range(enc, p.quality, p.lgwin, hint, input + rb, e - rb, s - rb, e - s, f ? 1 : 0,
                                     (last && l) ? 1 : 0, (l ? (align_end && !last) : true) ? 1 : 0, out + off, out_cap - off, &got, 0))
      return false;
    off += got;
    if (e == b) break;
    s = e;
  }
  *out_size = off;
  return true;
}

// ---- stream framing around compress_span (catable / appendable / magic_number / byte_align / bare_stream) ----
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
// encode.rs:2285-2333].  data: those first bytes, or nullptr to leave zeros in their place (the device copies them in);
// *data_off / *n2: where they are and how many.  Shared by compress_framed and b200_encoder_compress_params_async.
static void write_prologue(HostBits& w, const EncoderParams& p, size_t len, const uint8_t* data, size_t* data_off, size_t* n2) {
  const int lw = p.lgwin < 10 ? 10 : (p.lgwin > 24 ? 24 : p.lgwin);
  *data_off = 0;
  *n2 = 0;
  if (!(p.catable && p.bare_stream)) put_window_bits(w, lw);
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
    w.bytes(data ? data : zeros, *n2);
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
// Compresses input[a, b) like compress_span and wraps it in the framing `p` asks for:
//   first: [window bits unless catable && bare] [magic-number metadata metablock, brotli_bit_stream.rs:2869-2896]
//          [catable: the first min(2, len) bytes as an uncompressed metablock, encode.rs:2285-2333 -- a stitched stream's literal
//          contexts then never look into the previous file]
//   last:  [byte_align: padding metablock][unless bare: the empty last metablock]  (WriteEmptyLastBlocksInternal encode.rs:1928-1940)
// Data metablocks never carry ISLAST on this path, so "appendable" (encode.rs:1973-1975) needs nothing more, and every
// metablock starts with an unknown distance cache, which is what catable's 0x7ffffff0 cache (encode.rs:693-703) asks for.
static bool compress_framed(B200Encoder* enc, EncoderParams p, uint64_t hint, const uint8_t* input, size_t a, size_t b, bool first,
                            bool last, bool align_end, uint8_t* out, size_t out_cap, size_t* out_size) {
  sanitize_framing(p);
  if (!framed(p)) return compress_span(enc, p, hint, input, a, b, first, last, align_end, out, out_cap, out_size);
  HostBits w{out, out_cap};
  size_t body_a = a;
  bool dev_first = first;
  if (first && (p.magic_number || p.catable || a == b)) {
    dev_first = false;
    size_t data_off, n2;
    write_prologue(w, p, b - a, input + a, &data_off, &n2);
    body_a += n2;
  }
  if (!w.ok) return false;
  size_t off = (size_t)(w.pos >> 3);
  if (body_a < b) {
    if (w.pos & 7) return false;  // cannot happen: a prologue in front of data ends with a byte-aligned metablock
    // the device writes the plain 2-bit trailer itself when no alignment is asked for
    const bool dev_last = last && !p.byte_align && !p.bare_stream;
    const bool dev_align = last ? (p.byte_align != 0) : align_end;
    size_t got = 0;
    if (!compress_span(enc, p, hint, input, body_a, b, dev_first, dev_last, dev_align, out + off, out_cap - off, &got)) return false;
    off += got;
    if (last && p.byte_align && !p.bare_stream) {
      if (off >= out_cap) return false;
      out[off++] = 3;  // ISLAST + ISLASTEMPTY on a byte boundary
    }
    *out_size = off;
    return true;
  }
  // nothing (left) to compress: the trailer follows the prologue directly
  write_empty_trailer(w, p, last, align_end);
  if (!w.ok || (w.pos & 7)) return false;
  *out_size = (size_t)(w.pos >> 3);
  return true;
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
// compressor.rs:162 / encode.rs:1205-1260: the last min(size, 2^lgwin - 16) dictionary bytes become window content in
// front of the stream (they occupy positions), the static dictionary is switched off.  Ignored once input was consumed.
void BrotliEncoderSetCustomDictionary(BrotliEncoderState* s, size_t size, const uint8_t* dict) {
  if (!s || s->started || s->dict_len != 0) return;
  s->params.no_dictionary = 1;
  if (size <= 1 || !dict) return;
  const int lw = s->params.lgwin < 10 ? 10 : (s->params.lgwin > 24 ? 24 : s->params.lgwin);
  const size_t max_dict = ((size_t)1 << lw) - 16;
  if (size > max_dict) { dict += size - max_dict; size = max_dict; }
  s->input.assign(dict, dict + size);
  s->dict_len = size;
  s->flushed = size;
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

// Compresses the stream bytes [flushed, upto) and appends the result to the output queue.
static bool state_emit(BrotliEncoderStateStruct* s, bool last, uint64_t upto) {
  const uint64_t start = s->flushed, len = upto - start;
  const bool first = !s->header_written;
  EncoderParams fp = s->params;
  sanitize_framing(fp);
  if (len == 0 && !(framed(fp) && first)) {
    if (last) {
      if (first) s->output.push_back(6);        // empty stream, encode.rs:1463
      else if (!fp.bare_stream) s->output.push_back(3);  // ISLAST + ISLASTEMPTY after a byte-aligned flush
      s->header_written = true;
    }
    return true;
  }
  size_t cap = b200_max_compressed_size(len) + 64, got = 0;
  size_t old = s->output.size();
  s->output.resize(old + cap);
  uint64_t hint = s->params.size_hint ? s->params.size_hint : s->base + s->input.size() - s->dict_len;
  // positions are relative to `base`: once a prefix has been dropped at least a full window precedes `start`, so the
  // window limit min(position, 2^lgwin - 16) is the same in both coordinate systems
  bool ok = compress_framed(s->enc, s->params, hint, s->input.data(), (size_t)(start - s->base), (size_t)(upto - s->base), first, last,
                            true, s->output.data() + old, cap, &got);
  if (!ok) { s->output.resize(old); return false; }
  s->output.resize(old + got);
  s->flushed = upto;
  s->header_written = true;
  // keep only the match window in front of the unflushed part
  int lw = s->params.lgwin < 10 ? 10 : (s->params.lgwin > 24 ? 24 : s->params.lgwin);
  const uint64_t window = ((uint64_t)1 << lw) + 65536;
  if (s->flushed > s->base + window) {
    const uint64_t keep_from = (s->flushed - window) & ~(uint64_t)4095;
    if (keep_from > s->base) {
      s->input.erase(s->input.begin(), s->input.begin() + (size_t)(keep_from - s->base));
      s->base = keep_from;
    }
  }
  return true;
}

BROTLI_BOOL BrotliEncoderCompressStream(BrotliEncoderState* s, BrotliEncoderOperation op, size_t* available_in,
                                        const uint8_t** next_in, size_t* available_out, uint8_t** next_out, size_t* total_out) {
  if (!s || !available_in || !available_out) return BROTLI_FALSE;
  if (op == BROTLI_OPERATION_EMIT_METADATA) return BROTLI_FALSE;  // not on this path
  DeviceGuard dg;
  if (*available_in) {
    if (s->finished || !next_in || !*next_in) return BROTLI_FALSE;
    s->started = true;
    s->input.insert(s->input.end(), *next_in, *next_in + *available_in);
    *next_in += *available_in;
    *available_in = 0;
  }
  const uint64_t end = s->base + s->input.size();
  while (op == BROTLI_OPERATION_PROCESS && end - s->flushed >= 2 * kStreamPieceBytes) {  // keep one piece back for FINISH
    if (!state_emit(s, false, s->flushed + kStreamPieceBytes)) return BROTLI_FALSE;
  }
  if (op == BROTLI_OPERATION_FLUSH && s->flushed < end) {
    s->started = true;
    if (!state_emit(s, false, end)) return BROTLI_FALSE;
  } else if (op == BROTLI_OPERATION_FINISH && !s->finished) {
    s->started = true;
    if (!state_emit(s, true, end)) return BROTLI_FALSE;
    s->finished = true;
  }
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
BROTLI_BOOL BrotliEncoderIsFinished(BrotliEncoderState* s) { return (s && s->finished && s->out_pos == s->output.size()) ? 1 : 0; }
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
    ok = compress_span(enc, p, input_size, input, 0, input_size, true, true, false, encoded, out_cap, &got);
  }
  if (!ok) {  // no CPU-produced stream, ever: a device failure (or a too-small output buffer) is reported as failure
    *encoded_size = 0;
    return BROTLI_FALSE;
  }
  *encoded_size = got;
  return BROTLI_TRUE;
}

// One complete stream of the n device bytes at `in`, stream-ordered on `stream`: the bytes of compress_framed(first, last) --
// which BrotliEncoderCompressStream with one FINISH runs -- with the prologue written by a kernel and the body compressed behind it.
int b200_encoder_compress_params_async(B200Encoder* e, size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values,
                                       const uint8_t* in, size_t n, uint8_t* out, size_t out_cap, uint64_t* out_size, void* stream) {
  if (!e || (num_params && (!keys || !values))) return 0;
  if (n >= kSpanPiece) return 0;  // one span piece: longer inputs are cut into pieces by compress_span
  if (out_cap < b200_max_compressed_size(n) + 64) return 0;
  EncoderParams p;
  for (size_t i = 0; i < num_params; ++i)
    if (!apply_param(p, (int)keys[i], values[i])) return 0;
  sanitize_framing(p);
  const uint64_t hint = p.size_hint ? p.size_hint : n;
  const int ctx = p.disable_ctx ? 0 : 1, dict = p.no_dictionary ? 0 : 1;
  if (!framed(p))
    return b200_encoder_compress_framed_async(e, p.quality, p.lgwin, hint, ctx, dict, in, n, 0, n, 1, 1, 0, nullptr, -1, out, out_cap,
                                              out_size, stream);
  B200Prologue pro;
  memset(&pro, 0, sizeof(pro));
  HostBits w{pro.bytes, sizeof(pro.bytes)};
  size_t body_a = 0, data_off = 0, n2 = 0;
  const bool has_prologue = p.magic_number || p.catable || n == 0;
  if (has_prologue) write_prologue(w, p, n, nullptr, &data_off, &n2);
  body_a = n2;
  if (!w.ok) return 0;
  pro.data_off = (uint32_t)data_off;
  pro.n2 = (uint32_t)n2;
  if (body_a < n) {  // as compress_framed: the device writes the plain trailer itself unless the stream ends byte aligned
    if (w.pos & 7) return 0;
    pro.len = (uint32_t)(w.pos >> 3);
    const bool dev_last = !p.byte_align && !p.bare_stream;
    return b200_encoder_compress_framed_async(e, p.quality, p.lgwin, hint, ctx, dict, in, n, body_a, n - body_a, has_prologue ? 0 : 1,
                                              dev_last ? 1 : 0, p.byte_align ? 1 : 0, has_prologue ? &pro : nullptr,
                                              (p.byte_align && !p.bare_stream) ? 3 : -1, out, out_cap, out_size, stream);
  }
  write_empty_trailer(w, p, true, true);
  if (!w.ok || (w.pos & 7)) return 0;
  pro.len = (uint32_t)(w.pos >> 3);
  pro.complete = 1;
  return b200_encoder_compress_framed_async(e, p.quality, p.lgwin, hint, ctx, dict, in, n, n, 0, 0, 0, 0, &pro, -1, out, out_cap,
                                            out_size, stream);
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

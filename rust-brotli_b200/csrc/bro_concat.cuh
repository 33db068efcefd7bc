// bro_concat.cuh -- the stream stitcher of the reference (BroCatli, src/concat/mod.rs), restated once as __host__ __device__
// code.  The host Broccoli C ABI (bro_broccoli.cu) drives it over caller buffers of any size; the device splice
// (b200_concat_async, bro_concat.cu) runs the same state machine per stream with a recording sink to plan its copy.
//
// Output bound.  Every stream's bytes are emitted at most once, minus its window bits and the final ISLAST+ISLASTEMPTY pair that
// is stripped from it; the metablock header behind a spliced stream's window bits is re-emitted at the previous stream's end bit
// (realign_header: ceil((lbo + varlen - wbits) / 8) <= ceil(varlen / 8) + 1 bytes with lbo <= 7, wbits >= 1, and the first of
// them is the previous stream's last partial byte), so a stream never grows.  What is added on top: the seeded header of a
// window-size instance (<= 2 bytes), or the single ';' of an instance that emitted nothing.  One exception to "+ 2": a
// window-size instance of lgwin 10..15 or 17 whose every stream was dropped finishes with 3 bytes (append_eof on a two-byte
// tail, mod.rs:567-580, followed by the emitting loop of :585-594).  So the output is at most sum(sizes) + 3 bytes.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "bro_common.cuh"

namespace bro {
namespace cat {

// BroCatliResult (mod.rs:3-13); kPanic: where the reference panics (its FFI then returns 127 and keeps the previous state)
enum : int {
  kSuccess = 0,
  kNeedsMoreInput = 1,
  kNeedsMoreOutput = 2,
  kNotCraftedForAppend = 124,
  kInvalidWindowSize = 125,
  kWindowSizeLarger = 126,
  kNotCraftedForConcatenation = 127,
  kPanic = -1,
};
constexpr int kHeaderBytes = 5;  // NUM_STREAM_HEADER_BYTES, mod.rs:15

// NewStreamData::sufficient (mod.rs:31-36): 4 header bytes, or 5 when the first byte could open a large-window header
BRO_HD bool header_sufficient(const uint8_t* b, int nread) { return (nread == 4 && (b[0] & 127) != 17) || nread == 5; }

// parse_window_size (mod.rs:39-71): window size and header length in bits; false if the header is not one.  Reads b[1] only for
// the 14-bit large-window header; callers hold >= 4 bytes.
BRO_HD bool parse_window_size(const uint8_t* b, int* ws, int* bits) {
  if ((b[0] & 1) == 0) { *ws = 16; *bits = 1; return true; }
  const int lo4 = b[0] & 15;
  if (lo4 >= 3 && (lo4 & 1)) { *ws = 18 + (lo4 - 3) / 2; *bits = 4; return true; }
  switch (b[0] & 127) {
    case 0x71: *ws = 15; *bits = 7; return true;
    case 0x61: *ws = 14; *bits = 7; return true;
    case 0x51: *ws = 13; *bits = 7; return true;
    case 0x41: *ws = 12; *bits = 7; return true;
    case 0x31: *ws = 11; *bits = 7; return true;
    case 0x21: *ws = 10; *bits = 7; return true;
    case 0x01: *ws = 17; *bits = 7; return true;
    default: break;
  }
  if (b[0] & 0x80) return false;
  const int r = b[1] & 0x3f;
  if (r < 10 || r > 30) return false;
  *ws = r; *bits = 14;
  return true;
}

// detect_varlen_offset (mod.rs:73-120): bit offset behind the header of the first metablock, which must be an empty last one, a
// metadata block or an uncompressed one (the payload is then byte aligned); -1 otherwise.  ISLAST with data falls through to
// MNIBBLES as in the reference.  Bytes past `n` read as zero.
BRO_HD int detect_varlen_offset(const uint8_t* b, int n) {
  int ws, offset;
  if (!parse_window_size(b, &ws, &offset)) return -1;
  uint64_t bytes = 0;
  for (int i = 0; i < n; ++i) bytes |= (uint64_t)b[i] << (i * 8);
  bytes >>= offset;
  offset += 1;
  if (bytes & 1) {  // ISLAST
    bytes >>= 1;
    offset += 1;
    if (bytes & 1) return offset;  // ISLASTEMPTY
  }
  bytes >>= 1;
  uint64_t mnibbles = bytes & 3;
  bytes >>= 2;
  offset += 2;
  if (mnibbles == 3) {  // metadata block
    if (bytes & 1) return -1;  // reserved bit
    bytes >>= 1;
    offset += 1;
    const int skip = (int)(bytes & 3);
    offset += 2 + skip * 8;
    return offset;
  }
  mnibbles += 4;
  offset += (int)mnibbles * 4;
  bytes >>= mnibbles * 4;
  offset += 1;
  return (bytes & 1) ? offset : -1;  // ISUNCOMPRESSED
}

// flush_previous_stream's bit rule (mod.rs:289-310): masks the final ISLAST + ISLASTEMPTY pair out of the last `len` (1 or 2)
// bytes in lb and returns the bit index where the stream now ends (0..14), or -1 when the two highest set bits are not 1 1.
BRO_HD int strip_last_empty(uint8_t lb[2], int len) {
  uint32_t v = (uint32_t)lb[0] | ((uint32_t)lb[1] << 8);
  const int max = len * 8;
  int index = max - 1;
  for (int i = 0; i < max; ++i) {
    index = max - 1 - i;
    if ((1u << index) & v) break;
  }
  if (index == 0) return -1;
  if ((v >> (index - 1)) != 3) return -1;
  index -= 1;
  v &= (1u << index) - 1;
  lb[0] = (uint8_t)v;
  lb[1] = (uint8_t)(v >> 8);
  return index;
}

// The realigned header (mod.rs:357-405): the new stream's metablock header bits [wbits, varlen) placed behind the `lbo` bits of
// `last`, then the header's whole bytes from ceil(varlen / 8) on.  Returns the byte count (out[0] included), or -1 when the
// header reaches past the bytes read (-2: where the reference would panic).
BRO_HD int realign_header(const uint8_t* hdr, int nread, int wbits, int varlen, int lbo, uint8_t last, uint8_t out[kHeaderBytes + 1]) {
  out[0] = last;
  for (int i = 1; i <= kHeaderBytes; ++i) out[i] = 0;
  uint64_t bits = 0;
  for (int i = 0; i < nread; ++i) bits |= (uint64_t)hdr[i] << (i * 8);
  bits >>= wbits;
  bits &= ((uint64_t)1 << (varlen - wbits)) - 1;
  const int var_len_bytes = (varlen - wbits + 7) / 8;
  if (var_len_bytes > kHeaderBytes) return -2;  // cannot happen (varlen - wbits <= 33); the reference would index past its array
  for (int bi = 0; bi < var_len_bytes; ++bi) {
    const uint64_t cur = bits >> (bi * 8);
    out[bi] |= (uint8_t)((cur & (((uint64_t)1 << (8 - lbo)) - 1)) << lbo);
    out[bi + 1] = (uint8_t)(cur >> (8 - lbo));
  }
  const int dst = (lbo + varlen - wbits + 7) / 8, src = (varlen + 7) / 8;
  if (src > nread) return -1;
  const int whole = nread - src;
  for (int i = 0; i < whole; ++i) out[dst + i] = hdr[src + i];
  return dst + whole;
}

// try_new_with_window_size (mod.rs:231-272): the bytes of an empty stream with that window (window bits, then 1 1); false for a
// size the reference refuses.  Sizes above 24 take the large-window header.
BRO_HD bool seed_window(int ws, uint8_t lb[2], int* len) {
  if (ws > 24) { lb[0] = 17; lb[1] = (uint8_t)(ws | 64 | 128); *len = 2; return true; }
  if (ws == 16) { lb[0] = 1 | 2 | 4; lb[1] = 0; *len = 1; return true; }
  if (ws > 17) { lb[0] = (uint8_t)((3 + (ws - 18) * 2) | (16 | 32)); lb[1] = 0; *len = 1; return true; }
  uint8_t b0;
  switch (ws) {
    case 15: b0 = 0x71; break;
    case 14: b0 = 0x61; break;
    case 13: b0 = 0x51; break;
    case 12: b0 = 0x41; break;
    case 11: b0 = 0x31; break;
    case 10: b0 = 0x21; break;
    case 17: b0 = 0x01; break;
    default: return false;
  }
  lb[0] = (uint8_t)(b0 | 0x80); lb[1] = 1; *len = 2;
  return true;
}

// The BroCatli state (mod.rs:124-134, :17-22) as plain data.  stream() / finish() write through an output sink:
//   avail() bytes of room, put(b), copy(src, n) (n input bytes, in order), unput() (takes the last put byte back and returns it).
struct Catli {
  uint8_t last_bytes[2];
  uint8_t last_bytes_len;
  uint8_t last_byte_sanitized;
  uint8_t any_bytes_emitted;
  uint8_t last_byte_bit_offset;
  uint8_t window_size;
  uint8_t pending;                 // new_stream_pending.is_some()
  uint8_t pend_bytes[kHeaderBytes];
  uint8_t pend_read;
  uint8_t pend_has_written;        // num_bytes_written.is_some()
  uint8_t pend_written;

  BRO_HD void init() {  // BroCatli::new (mod.rs:137-139)
    last_bytes[0] = last_bytes[1] = 0;
    last_bytes_len = last_byte_sanitized = any_bytes_emitted = last_byte_bit_offset = window_size = 0;
    pending = 0;
    for (int i = 0; i < kHeaderBytes; ++i) pend_bytes[i] = 0;
    pend_read = pend_has_written = pend_written = 0;
  }
  BRO_HD bool init_window(int ws) {  // try_new_with_window_size; on refusal the state is BroCatli::new
    init();
    int len = 0;
    if (!seed_window(ws, last_bytes, &len)) return false;
    last_bytes_len = (uint8_t)len;
    window_size = (uint8_t)ws;
    return true;
  }
  BRO_HD void new_brotli_file() {  // mod.rs:274-276: pending header bytes of a stream not yet sufficient are dropped
    pending = 1;
    for (int i = 0; i < kHeaderBytes; ++i) pend_bytes[i] = 0;
    pend_read = 0;
    pend_has_written = 0;
    pend_written = 0;
  }

  template <class Out>
  BRO_HD int flush_previous_stream(Out& out) {  // mod.rs:277-329
    if (last_byte_sanitized) return kSuccess;
    if (last_bytes_len == 0) { last_byte_sanitized = 1; return kSuccess; }
    uint8_t lb[2] = {last_bytes[0], last_bytes[1]};
    int index = strip_last_empty(lb, last_bytes_len);
    if (index < 0) return kNotCraftedForAppend;
    last_bytes[0] = lb[0];
    last_bytes[1] = lb[1];
    if (index >= 8) {
      if (out.avail() == 0) return kNeedsMoreOutput;
      out.put(last_bytes[0]);
      last_bytes[0] = last_bytes[1];
      any_bytes_emitted = 1;
      index -= 8;
      last_bytes_len -= 1;
    }
    last_byte_bit_offset = (uint8_t)index;
    last_byte_sanitized = 1;
    return kSuccess;
  }

  template <class Out>
  BRO_HD int shift_and_check_new_stream_header(Out& out) {  // mod.rs:331-449
    if (!pend_has_written) {
      int ws, wbits;
      if (!parse_window_size(pend_bytes, &ws, &wbits)) return kInvalidWindowSize;
      if (window_size == 0) {  // first stream: copied as it is
        window_size = (uint8_t)ws;
        if (last_byte_bit_offset != 0) return kPanic;
        out.put(pend_bytes[0]);
        pend_has_written = 1;
        pend_written = 1;
        any_bytes_emitted = 1;
      } else {
        if (ws > window_size) return kWindowSizeLarger;
        const int varlen = detect_varlen_offset(pend_bytes, pend_read);
        if (varlen < 0) return kNotCraftedForConcatenation;
        uint8_t re[kHeaderBytes + 1];
        const int cnt = realign_header(pend_bytes, pend_read, wbits, varlen, last_byte_bit_offset, last_bytes[0], re);
        if (cnt < 0) return cnt == -2 ? kPanic : kNotCraftedForConcatenation;
        out.put(re[0]);
        any_bytes_emitted = 1;
        pend_read = (uint8_t)(cnt - 1);
        pend_has_written = 1;
        pend_written = 0;
        for (int i = 0; i < kHeaderBytes; ++i) pend_bytes[i] = re[i + 1];
      }
    } else if (window_size == 0) {
      return kPanic;
    }
    size_t to_copy = (size_t)(pend_read - pend_written);
    if (out.avail() < to_copy) to_copy = out.avail();
    for (size_t i = 0; i < to_copy; ++i) out.put(pend_bytes[pend_written + i]);
    if (to_copy) any_bytes_emitted = 1;
    pend_written = (uint8_t)(pend_written + to_copy);
    if (pend_written != pend_read) return kNeedsMoreOutput;  // (the pending header stays as it is now)
    pending = 0;
    last_byte_sanitized = 0;
    last_byte_bit_offset = 0;
    last_bytes[1] = 0;
    last_bytes[0] = out.unput();  // the last byte may still have to carry the end of the stream
    last_bytes_len = 1;
    return kSuccess;
  }

  template <class Out>
  BRO_HD int stream(const uint8_t* in, size_t in_len, size_t* in_off, Out& out) {  // mod.rs:450-566
    if (pending) {
      const int fr = flush_previous_stream(out);
      if (fr != kSuccess) return fr;
      if (pend_read < kHeaderBytes) {
        size_t to_copy = (size_t)(kHeaderBytes - pend_read);
        if (in_len - *in_off < to_copy) to_copy = in_len - *in_off;
        for (size_t i = 0; i < to_copy; ++i) pend_bytes[pend_read + i] = in[*in_off + i];
        *in_off += to_copy;
        pend_read = (uint8_t)(pend_read + to_copy);
      }
      if (!header_sufficient(pend_bytes, pend_read)) return kNeedsMoreInput;
      if (out.avail() == 0) return kNeedsMoreOutput;
      const int sr = shift_and_check_new_stream_header(out);
      if (sr != kSuccess) return sr;
      if (out.avail() == 0) return kNeedsMoreOutput;
    }
    if (last_bytes_len != 2) {
      if (out.avail() == 0) return kNeedsMoreOutput;
      if (in_len == *in_off) return kNeedsMoreInput;
      last_bytes[last_bytes_len] = in[(*in_off)++];
      last_bytes_len += 1;
      if (last_bytes_len != 2) {
        if (out.avail() == 0) return kNeedsMoreOutput;
        if (in_len == *in_off) return kNeedsMoreInput;
        last_bytes[last_bytes_len] = in[(*in_off)++];
        last_bytes_len += 1;
      }
    }
    if (out.avail() == 0) return kNeedsMoreOutput;
    if (in_len == *in_off) return kNeedsMoreInput;
    size_t to_copy = in_len - *in_off;
    if (out.avail() < to_copy) to_copy = out.avail();
    if (to_copy == 1) {
      out.put(last_bytes[0]);
      last_bytes[0] = last_bytes[1];
      last_bytes[1] = in[(*in_off)++];
      return out.avail() == 0 ? kNeedsMoreOutput : kNeedsMoreInput;
    }
    out.put(last_bytes[0]);
    out.put(last_bytes[1]);
    const size_t a = *in_off;
    last_bytes[0] = in[a + to_copy - 2];
    last_bytes[1] = in[a + to_copy - 1];
    out.copy(in + a, to_copy - 2);
    *in_off = a + to_copy;
    return out.avail() == 0 ? kNeedsMoreOutput : kNeedsMoreInput;
  }

  BRO_HD void append_eof_metablock_to_last_bytes() {  // mod.rs:567-580 (a two-byte tail loses bit 16: the reference's u16)
    uint32_t v = (uint32_t)last_bytes[0] | ((uint32_t)last_bytes[1] << 8);
    const int bit_end = (last_bytes_len - 1) * 8 + last_byte_bit_offset;
    v = (v | (3u << bit_end)) & 0xffffu;
    last_bytes[0] = (uint8_t)v;
    last_bytes[1] = (uint8_t)(v >> 8);
    last_byte_sanitized = 0;
    last_byte_bit_offset += 2;
    if (last_byte_bit_offset >= 8) {
      last_byte_bit_offset -= 8;
      last_bytes_len += 1;
    }
  }

  template <class Out>
  BRO_HD int finish(Out& out) {  // mod.rs:581-604
    if (last_byte_sanitized && last_bytes_len != 0) append_eof_metablock_to_last_bytes();
    while (last_bytes_len != 0) {
      if (out.avail() == 0) return kNeedsMoreOutput;
      out.put(last_bytes[0]);
      last_bytes_len -= 1;
      last_bytes[0] = last_bytes[1];
      any_bytes_emitted = 1;
    }
    if (!any_bytes_emitted) {
      if (out.avail() == 0) return kNeedsMoreOutput;
      any_bytes_emitted = 1;
      out.put(';');
    }
    return kSuccess;
  }

  // serialize_to_buffer / deserialize_from_buffer (mod.rs:141-221) over the first 21 bytes of a zeroed buffer
  BRO_HD void serialize(uint8_t* buf) const {
    buf[0] = last_bytes[0];
    buf[1] = last_bytes[1];
    buf[8] = last_bytes_len;
    buf[9] = (uint8_t)((last_byte_sanitized ? 1 : 0) | (pending ? 1 << 6 : 0) | (any_bytes_emitted ? 1 << 5 : 0));
    buf[10] = last_byte_bit_offset;
    buf[11] = window_size;
    if (pending) {
      if (pend_has_written) buf[9] |= 1 << 7;
      buf[12] = pend_read;
      buf[13] = pend_has_written ? pend_written : 0;
      for (int i = 0; i < kHeaderBytes; ++i) buf[16 + i] = pend_bytes[i];
    }
  }
  BRO_HD bool deserialize(const uint8_t* buf) {
    const uint8_t len = buf[8], lbo = buf[10], ws = buf[11];
    const bool has_pending = (buf[9] & (1 << 6)) != 0, has_written = (buf[9] & (1 << 7)) != 0;
    if (len > 2 || lbo >= 8) return false;
    if (ws != 0) {
      uint8_t tmp[2];
      int tl;
      if (!seed_window(ws, tmp, &tl)) return false;
    }
    if (has_pending) {
      if (buf[12] > kHeaderBytes) return false;
      if (has_written && buf[13] > buf[12]) return false;
    }
    last_bytes[0] = buf[0];
    last_bytes[1] = buf[1];
    last_bytes_len = len;
    last_byte_sanitized = (buf[9] & 1) ? 1 : 0;
    any_bytes_emitted = (buf[9] & (1 << 5)) ? 1 : 0;
    last_byte_bit_offset = lbo;
    window_size = ws;
    pending = has_pending ? 1 : 0;
    pend_read = buf[12];
    pend_has_written = has_written ? 1 : 0;
    pend_written = has_written ? buf[13] : 0;
    for (int i = 0; i < kHeaderBytes; ++i) pend_bytes[i] = buf[16 + i];
    return true;
  }
};

}  // namespace cat
}  // namespace bro

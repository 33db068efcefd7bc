// bro_broccoli.cu -- the reference's Broccoli C ABI (src/ffi/broccoli.rs) over the shared splice rules of bro_concat.cuh.
// Host code: the state is unpacked from the caller's BroccoliState, advanced over the caller's buffers and packed back, as the
// reference does with BroCatli::{deserialize_from_buffer, serialize_to_buffer}.  Where the reference panics (an unreadable
// state, an assertion), its FFI catches the panic, leaves the state and the pointers as they were and returns 127: so does this.
#include <cstring>

#include "broccoli.h"
#include "bro_concat.cuh"

namespace {

using bro::cat::Catli;

struct HostOut {  // output sink of Catli over a caller buffer (__host__ __device__ only because Catli's methods are)
  uint8_t* p;
  size_t cap, pos = 0;
  BRO_HD size_t avail() const { return cap - pos; }
  BRO_HD void put(uint8_t b) { p[pos++] = b; }
  BRO_HD void copy(const uint8_t* src, size_t n) {
    if (n) memcpy(p + pos, src, n);
    pos += n;
  }
  BRO_HD uint8_t unput() { return p[--pos]; }
};

BroccoliState pack(const Catli& c) {
  BroccoliState s;
  s.unused = nullptr;
  memset(s.data, 0, sizeof(s.data));
  c.serialize(s.data);
  return s;
}

BroccoliResult result(int code) {
  return static_cast<BroccoliResult>(code == bro::cat::kPanic ? bro::cat::kNotCraftedForConcatenation : code);
}

}  // namespace

static_assert(sizeof(BroccoliState) == 256, "the C header's layout: void* + 248 bytes");

extern "C" {

BroccoliState BroccoliCreateInstance(void) {
  Catli c;
  c.init();
  return pack(c);
}

BroccoliState BroccoliCreateInstanceWithWindowSize(uint8_t window_size) {
  Catli c;
  if (!c.init_window(window_size)) c.init();
  return pack(c);
}

void BroccoliDestroyInstance(BroccoliState state) { (void)state; }

void BroccoliNewBrotliFile(BroccoliState* state) {
  Catli c;
  if (!state || !c.deserialize(state->data)) return;
  c.new_brotli_file();
  *state = pack(c);
}

BroccoliResult BroccoliConcatStream(BroccoliState* state, size_t* available_in, const uint8_t** input_buf_ptr, size_t* available_out,
                                    uint8_t** output_buf_ptr) {
  Catli c;
  if (!state || !available_in || !input_buf_ptr || !available_out || !output_buf_ptr || !c.deserialize(state->data))
    return BroccoliBrotliFileNotCraftedForConcatenation;
  const uint8_t* in = *available_in ? *input_buf_ptr : nullptr;
  HostOut out{*available_out ? *output_buf_ptr : nullptr, *available_out};
  size_t in_off = 0;
  const int r = c.stream(in, *available_in, &in_off, out);
  if (r == bro::cat::kPanic) return result(r);
  *input_buf_ptr += in_off;
  *output_buf_ptr += out.pos;
  *available_in -= in_off;
  *available_out -= out.pos;
  *state = pack(c);
  return result(r);
}

BroccoliResult BroccoliConcatStreaming(BroccoliState* state, size_t* available_in, const uint8_t* input_buf_ptr, size_t* available_out,
                                       uint8_t* output_buf_ptr) {
  return BroccoliConcatStream(state, available_in, &input_buf_ptr, available_out, &output_buf_ptr);
}

BroccoliResult BroccoliConcatFinish(BroccoliState* state, size_t* available_out, uint8_t** output_buf) {
  Catli c;
  if (!state || !available_out || !output_buf || !c.deserialize(state->data)) return BroccoliBrotliFileNotCraftedForConcatenation;
  HostOut out{*available_out ? *output_buf : nullptr, *available_out};
  const int r = c.finish(out);
  *output_buf += out.pos;
  *available_out -= out.pos;
  *state = pack(c);
  return result(r);
}

BroccoliResult BroccoliConcatFinished(BroccoliState* state, size_t* available_out, uint8_t* output_buf) {
  return BroccoliConcatFinish(state, available_out, &output_buf);
}

}  // extern "C"

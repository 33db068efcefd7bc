/* broccoli.h -- C ABI of the stream stitcher, with the names, values and layout of the reference's c/brotli/broccoli.h
 * (dropbox/rust-brotli 8.0.4, src/ffi/broccoli.rs).  It splices brotli streams made with BROTLI_PARAM_CATABLE (or
 * APPENDABLE for the first one) into one standard stream, byte for byte as the reference's BroCatli (src/concat/mod.rs) does,
 * with the same result codes for every split of input and output buffers.
 *
 * These functions are host code.  They splice through a two-byte look-behind over caller buffers of any size and hold no
 * compression arithmetic, so they need no CUDA device and never touch one.  For streams already on the GPU see
 * b200_concat_async in brotli_b200.h, which produces the same bytes as the sequence CreateInstance, then NewBrotliFile +
 * ConcatStream over each stream, then ConcatFinish.
 *
 * BroccoliState is plain data: the whole splice state is serialised into `data` (the first 21 bytes, as the reference's
 * serialize_to_buffer lays them out); `unused` is always NULL.  It is returned and destroyed by value and may be copied freely.
 */
#ifndef BROTLI_BROCCOLI_H
#define BROTLI_BROCCOLI_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct BroccoliState_ {
  void* unused;
  unsigned char data[248];
} BroccoliState;

typedef enum BroccoliResult_ {
  BroccoliSuccess = 0,
  BroccoliNeedsMoreInput = 1,
  BroccoliNeedsMoreOutput = 2,
  BroccoliBrotliFileNotCraftedForAppend = 124,
  BroccoliInvalidWindowSize = 125,
  BroccoliWindowSizeLargerThanPreviousFile = 126,
  BroccoliBrotliFileNotCraftedForConcatenation = 127
} BroccoliResult;

/* broccoli.rs:56 */
BroccoliState BroccoliCreateInstance(void);
/* broccoli.rs:60-65: an instance whose output starts as an empty stream of that window; every stream must have a window no
 * larger.  A size the reference refuses (below 10) gives a default instance. */
BroccoliState BroccoliCreateInstanceWithWindowSize(uint8_t window_size);
/* broccoli.rs:67: nothing to release */
void BroccoliDestroyInstance(BroccoliState state);
/* broccoli.rs:70: the following bytes start a new stream; header bytes of a stream still too short to splice are dropped */
void BroccoliNewBrotliFile(BroccoliState* state);
/* broccoli.rs:82: consumes input, produces output, advances both pointers and decrements both counts */
BroccoliResult BroccoliConcatStream(BroccoliState* state, size_t* available_in, const uint8_t** input_buf_ptr, size_t* available_out,
                                    uint8_t** output_buf_ptr);
/* broccoli.rs:110: the same with the buffer pointers passed by value */
BroccoliResult BroccoliConcatStreaming(BroccoliState* state, size_t* available_in, const uint8_t* input_buf_ptr, size_t* available_out,
                                       uint8_t* output_buf_ptr);
/* broccoli.rs:133: writes the end of the spliced stream (a single ';' if nothing was ever written) */
BroccoliResult BroccoliConcatFinish(BroccoliState* state, size_t* available_out, uint8_t** output_buf);
/* broccoli.rs:156: the same with the output pointer passed by value */
BroccoliResult BroccoliConcatFinished(BroccoliState* state, size_t* available_out, uint8_t* output_buf);

#ifdef __cplusplus
}
#endif
#endif /* BROTLI_BROCCOLI_H */

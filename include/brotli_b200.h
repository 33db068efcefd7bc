/* brotli_b200.h -- C ABI of the GPU-native (CUDA, H100) brotli compression path.
 *
 * This library is a drop-in for the COMPRESSION entry points that the reference (dropbox/rust-brotli 8.0.4)
 * exports from its cdylib; each declaration cites the reference interface it replaces.  The reference's stream concatenator
 * (Broccoli) is declared in broccoli.h; its device counterpart b200_concat_async is below.  Decompression and the CLI are out of
 * scope (SURVEY.md section 8).  All pointers are plain host
 * pointers unless a function says otherwise; no CUDA or torch types appear in any signature.
 *
 * Failure behaviour mirrors the reference: functions return BROTLI_FALSE / NULL / 0 on any error (including
 * "no usable CUDA device" -- there is no CPU fallback), and never abort the process
 * (src/ffi/compressor.rs:253-256, :419-422).
 */
#ifndef BROTLI_B200_H_
#define BROTLI_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BROTLI_BOOL int
#define BROTLI_TRUE 1
#define BROTLI_FALSE 0

/* c/brotli/encode.h ; src/enc/encode.rs BrotliEncoderMode */
typedef enum BrotliEncoderMode { BROTLI_MODE_GENERIC = 0, BROTLI_MODE_TEXT = 1, BROTLI_MODE_FONT = 2 } BrotliEncoderMode;

/* src/enc/encode.rs:1380-1385 */
typedef enum BrotliEncoderOperation {
  BROTLI_OPERATION_PROCESS = 0,
  BROTLI_OPERATION_FLUSH = 1,
  BROTLI_OPERATION_FINISH = 2,
  BROTLI_OPERATION_EMIT_METADATA = 3
} BrotliEncoderOperation;

/* src/enc/parameters.rs:1-32 (same numeric values as c/brotli/encode.h) */
typedef enum BrotliEncoderParameter {
  BROTLI_PARAM_MODE = 0,
  BROTLI_PARAM_QUALITY = 1,
  BROTLI_PARAM_LGWIN = 2,
  BROTLI_PARAM_LGBLOCK = 3,
  BROTLI_PARAM_DISABLE_LITERAL_CONTEXT_MODELING = 4,
  BROTLI_PARAM_SIZE_HINT = 5,
  BROTLI_PARAM_LARGE_WINDOW = 6,
  BROTLI_PARAM_Q9_5 = 150,
  BROTLI_METABLOCK_CALLBACK = 151,
  BROTLI_PARAM_STRIDE_DETECTION_QUALITY = 152,
  BROTLI_PARAM_HIGH_ENTROPY_DETECTION_QUALITY = 153,
  BROTLI_PARAM_LITERAL_BYTE_SCORE = 154,
  BROTLI_PARAM_CDF_ADAPTATION_DETECTION = 155,
  BROTLI_PARAM_PRIOR_BITMASK_DETECTION = 156,
  BROTLI_PARAM_SPEED = 157,
  BROTLI_PARAM_SPEED_MAX = 158,
  BROTLI_PARAM_CM_SPEED = 159,
  BROTLI_PARAM_CM_SPEED_MAX = 160,
  BROTLI_PARAM_SPEED_LOW = 161,
  BROTLI_PARAM_SPEED_LOW_MAX = 162,
  BROTLI_PARAM_CM_SPEED_LOW = 164,
  BROTLI_PARAM_CM_SPEED_LOW_MAX = 165,
  BROTLI_PARAM_AVOID_DISTANCE_PREFIX_SEARCH = 166,
  BROTLI_PARAM_CATABLE = 167,
  BROTLI_PARAM_APPENDABLE = 168,
  BROTLI_PARAM_MAGIC_NUMBER = 169,
  BROTLI_PARAM_NO_DICTIONARY = 170,
  BROTLI_PARAM_FAVOR_EFFICIENCY = 171,
  BROTLI_PARAM_BYTE_ALIGN = 172,
  BROTLI_PARAM_BARE_STREAM = 173
} BrotliEncoderParameter;

typedef void* (*brotli_alloc_func)(void* opaque, size_t size);
typedef void (*brotli_free_func)(void* opaque, void* address);

typedef struct BrotliEncoderStateStruct BrotliEncoderState;
typedef struct BrotliEncoderWorkPoolStruct BrotliEncoderWorkPool;

/* ---- single stream: src/ffi/compressor.rs ---- */
/* :72  BrotliEncoderCreateInstance.  Host-side bookkeeping uses alloc_func when given; device memory is owned by the state. */
BrotliEncoderState* BrotliEncoderCreateInstance(brotli_alloc_func alloc_func, brotli_free_func free_func, void* opaque);
/* :115 BrotliEncoderSetParameter (refused after the first byte was consumed, encode.rs:289-295).  Also refused
 * (BROTLI_FALSE, state unchanged): a value this path cannot honour -- LARGE_WINDOW != 0, LGBLOCK outside 0 / 16..24.
 * Framing parameters act as in the reference (encode.rs:264-283, :559-568, :1928-1940, :2258-2333): CATABLE (first two bytes as an
 * uncompressed metablock, no static dictionary, implies APPENDABLE), APPENDABLE, MAGIC_NUMBER (metadata metablock e1 97 8x,
 * VERSION, size hint), BYTE_ALIGN (padding metablock in front of the final empty one), BARE_STREAM (no final metablock; with
 * CATABLE no window bits either).  Streams made with CATABLE go through the reference's BroCatli (src/concat/mod.rs).
 * QUALITY: 5..9 run the hash-chain family, 10 and 11 the optimal-parse family; values below 5 run as 5 (the q0..q4
 * hashers are not built) -- b200_effective_quality() reports the quality that will really be used.
 * Q9_5 ("quality 9.5", encode.rs:834-893): quality 10 / 11 parse with the hash chains (10: H9; 11: H5 / H6 with 512-deep buckets)
 * and keep their metablock builder (context mode, block split, clustered context maps, distance parameters); at every quality
 * it lowers the size hint above which H6 is chosen from 4 MiB to 1 MiB.  The one-shot BrotliEncoderCompress never sets it.
 * The other research knobs (151..173 apart from the framing keys) are accepted and have no effect. */
BROTLI_BOOL BrotliEncoderSetParameter(BrotliEncoderState* state, BrotliEncoderParameter p, uint32_t value);
/* :128 */
void BrotliEncoderDestroyInstance(BrotliEncoderState* state);
/* :141 / encode.rs:1273 */
size_t BrotliEncoderMaxCompressedSize(size_t input_size);
/* :194 BrotliEncoderCompress -- one-shot; falls back to an uncompressed stream when the result would not fit
 * (encode.rs:1528-1536) */
BROTLI_BOOL BrotliEncoderCompress(int quality, int lgwin, BrotliEncoderMode mode, size_t input_size, const uint8_t* input_buffer,
                                  size_t* encoded_size, uint8_t* encoded_buffer);
/* :280 BrotliEncoderCompressStream */
BROTLI_BOOL BrotliEncoderCompressStream(BrotliEncoderState* state, BrotliEncoderOperation op, size_t* available_in,
                                        const uint8_t** next_in, size_t* available_out, uint8_t** next_out, size_t* total_out);
/* :260 BrotliEncoderCompressStreaming -- CompressStream with the buffer pointers passed by value and no total_out */
BROTLI_BOOL BrotliEncoderCompressStreaming(BrotliEncoderState* state, BrotliEncoderOperation op, size_t* available_in,
                                           const uint8_t* input_buf, size_t* available_out, uint8_t* output_buf);
/* :162 BrotliEncoderSetCustomDictionary -- the last min(size, 2^lgwin - 16) bytes of dict become window content in front
 * of the stream; the static dictionary is switched off (encode.rs:1205-1260).  Must precede the first input byte. */
void BrotliEncoderSetCustomDictionary(BrotliEncoderState* state, size_t size, const uint8_t* dict);
/* :359-419 host memory through the instance's allocator (malloc / free when none was given) */
uint8_t* BrotliEncoderMallocU8(BrotliEncoderState* state, size_t size);
void BrotliEncoderFreeU8(BrotliEncoderState* state, uint8_t* data, size_t size);
size_t* BrotliEncoderMallocUsize(BrotliEncoderState* state, size_t size);
void BrotliEncoderFreeUsize(BrotliEncoderState* state, size_t* data, size_t size);
/* :150-192 */
BROTLI_BOOL BrotliEncoderIsFinished(BrotliEncoderState* state);
BROTLI_BOOL BrotliEncoderHasMoreOutput(BrotliEncoderState* state);
const uint8_t* BrotliEncoderTakeOutput(BrotliEncoderState* state, size_t* size);
uint32_t BrotliEncoderVersion(void);

/* ---- multi-shard: src/ffi/multicompress/mod.rs ---- */
/* :49 */
size_t BrotliEncoderMaxCompressedSizeMulti(size_t input_size, size_t num_threads);
/* :93  shards = desired_num_threads (<= 16, fixed_queue.rs:1); shard i covers [i*len/n, (i+1)*len/n)
 * (threading/mod.rs:333) and sees the previous 2^lgwin bytes as its window; shards are placed round-robin on the
 * visible GPUs. */
int32_t BrotliEncoderCompressMulti(size_t num_params, const BrotliEncoderParameter* param_keys, const uint32_t* param_values,
                                   size_t input_size, const uint8_t* input, size_t* encoded_size, uint8_t* encoded,
                                   size_t desired_num_threads, brotli_alloc_func alloc_func, brotli_free_func free_func,
                                   void** alloc_opaque_per_thread);
/* :240, :294, :312 */
BrotliEncoderWorkPool* BrotliEncoderCreateWorkPool(size_t num_workers, brotli_alloc_func alloc_func, brotli_free_func free_func,
                                                   void** alloc_opaque_per_thread);
void BrotliEncoderDestroyWorkPool(BrotliEncoderWorkPool* work_pool);
int32_t BrotliEncoderCompressWorkPool(BrotliEncoderWorkPool* work_pool, size_t num_params, const BrotliEncoderParameter* param_keys,
                                      const uint32_t* param_values, size_t input_size, const uint8_t* input, size_t* encoded_size,
                                      uint8_t* encoded, size_t desired_num_threads, brotli_alloc_func alloc_func,
                                      brotli_free_func free_func, void** alloc_opaque_per_thread);

/* ---- device-resident entry points (additions of this library; pointers are CUDA device pointers where noted) ---- */
typedef struct B200Encoder B200Encoder;
int b200_device_count(void);
int b200_effective_quality(int requested_quality);
B200Encoder* b200_encoder_create(int device);
void b200_encoder_destroy(B200Encoder* e);
int b200_encoder_device(const B200Encoder* e); /* CUDA ordinal the encoder lives on */
/* bit d set: device d compressed at least one shard of the last BrotliEncoderCompressMulti / CompressWorkPool call (diagnostic) */
uint32_t b200_last_multi_device_mask(void);
/* encoder options (csrc/bro_encoder.h): context modelling and static dictionary on/off, stage timing, number of lanes, and the
 * switches the tests use to reach single stages (on-demand search, quality 10 / 11 parse unit, levels and splitter); the
 * defaults are the product configuration.  Returns 0 for an unknown option. */
int b200_encoder_set_option(B200Encoder* e, int option, uint32_t value);
size_t b200_max_compressed_size(size_t n);
/* device_io: 0 = in / out are host pointers; 1 = both are device pointers on the encoder's GPU; 2 = host input, device output
 * (e.g. shard outputs that travel on to a peer GPU over NVLink); 3 = device input, host output.
 * These calls return when the output is in place.  They run on the encoder's own streams, which do not wait for any other
 * stream: device input written by a kernel on another stream (a torch stream, the legacy default stream) must be complete
 * before the call, e.g. after torch.cuda.synchronize().  b200_encoder_compress_range_async has no such hazard. */
int b200_encoder_compress(B200Encoder* e, int quality, int lgwin, const uint8_t* in, size_t n, uint8_t* out, size_t out_cap,
                          size_t* out_size, int device_io);
int b200_encoder_compress_range(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, const uint8_t* in, size_t n,
                                size_t range_start, size_t range_len, int first, int last, int byte_align, uint8_t* out,
                                size_t out_cap, size_t* out_size, int device_io);
/* Sizes every device buffer, per-lane workspace and event that a call with these arguments uses. After this call, an async
 * call with the same or smaller (quality, lgwin, size_hint, n, range_len) allocates nothing, as long as the encoder's options
 * (number of lanes, quality 10 / 11 parse unit and splitter) stay the same.  size_hint 0 = n.  Returns 0 if memory runs out. */
int b200_encoder_reserve(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, size_t n, size_t range_len);
/* b200_encoder_compress_range, stream-ordered.  in / out / out_size are device pointers on the encoder's GPU; stream is a
 * cudaStream_t passed as void* (0 = the legacy default stream).  Returns 1 when the work has been enqueued.  out[0, *out_size)
 * is the compressed range once `stream` reaches that point; nothing on the host waits for it.  The bytes equal those of
 * b200_encoder_compress_range with the same arguments.
 *  - Ordering: the input is read only after the work enqueued on `stream` before the call; the output and *out_size are
 *    written before any work enqueued on `stream` after the call.  The call forks from `stream` into the encoder's streams with
 *    one event and joins back with a wait on the last event of each encoder stream it used.
 *  - Calls on one encoder run one at a time on the device: outside a graph capture, each async or blocking call first waits,
 *    on the device, for the encoder's previous call.
 *  - Output: the stream is built directly in `out`, which the call zeroes first; no staging buffer and no copy.  Refused (0,
 *    nothing enqueued): out_cap < b200_max_compressed_size(range_len) + 64, `out` not 4-byte aligned, in / out / out_size not
 *    device memory of the encoder's GPU, n >= 0xFFFFF000, a range outside [0, n).  `in` is not read when range_len == 0.
 *  - Empty input (n == 0 or range_len == 0: the single byte 6 of an empty stream when first && last && n == 0, otherwise
 *    nothing) is enqueued like any other call.
 *  - Allocation: a call whose buffers are too small grows them, and cudaFree may then block the host until the device is
 *    idle.  b200_encoder_reserve beforehand avoids that.
 *  - CUDA graph capture (`stream` capturing): the call never allocates, creates no event and does not wait for work recorded
 *    outside the capture.  If a buffer would have to grow it returns 0 before it enqueues anything, so the capture stays
 *    valid: reserve first.  Once a call has been captured the encoder's workspace is frozen, since the graph points into it:
 *    any later call (async or blocking) that would grow it is refused.  A graph replay does not order itself after other
 *    calls on the encoder, nor they after it: do not use an encoder captured in a graph while a replay may be in flight.
 *  - Stage timing (B200_OPT_TIMING) is not collected for these calls. */
int b200_encoder_compress_range_async(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, const uint8_t* in, size_t n,
                                      size_t range_start, size_t range_len, int first, int last, int byte_align, uint8_t* out,
                                      size_t out_cap, uint64_t* out_size, void* stream);
/* One complete stream of the n device bytes at `in`, with the key / value parameters of BrotliEncoderCompressMulti (the same
 * parameters are refused; the call then enqueues nothing).  For n < 1 GiB (larger n is refused) the bytes equal those of
 * BrotliEncoderCompressStream called once with the whole input and BROTLI_OPERATION_FINISH, with the same parameters: the
 * size hint is SIZE_HINT, or n; every framing mode (CATABLE, APPENDABLE, MAGIC_NUMBER, BYTE_ALIGN, BARE_STREAM) is produced.
 * NO_DICTIONARY, DISABLE_LITERAL_CONTEXT_MODELING and catable's "no static dictionary" apply to this call only: the encoder's
 * options are as they were before.  Ordering, output, refusals (out_cap < b200_max_compressed_size(n) + 64, ...), reservation
 * (b200_encoder_reserve with the same quality, lgwin, size hint and n) and graph capture: as b200_encoder_compress_range_async.
 * The prologue of a framed stream (window bits, magic-number metadata block, the catable stream's first two bytes as an
 * uncompressed metablock; <= 24 bytes) is written by a kernel from host-known bits passed as kernel parameters; a stream of at
 * most two bytes (or empty) is prologue and trailer only and uses no encoder workspace. */
int b200_encoder_compress_params_async(B200Encoder* e, size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values,
                                       const uint8_t* in, size_t n, uint8_t* out, size_t out_cap, uint64_t* out_size, void* stream);
int b200_encoder_last_timings(B200Encoder* e, float* ms, uint32_t* launches);

/* ---- device-resident streams: BrotliEncoderCompressStream with the window, the input and the output on the GPU ---- */
typedef struct B200Stream B200Stream;
/* A stream on e's GPU with the key / value parameters of BrotliEncoderCompressMulti (refused as BrotliEncoderSetParameter
 * refuses them) and, when d_dict is not NULL, the custom dictionary of the dict_len device bytes at d_dict (as
 * BrotliEncoderSetCustomDictionary after those parameters: the last min(dict_len, 2^lgwin - 16) bytes become window content,
 * the static dictionary is off).  The dictionary is copied on `stream`: work enqueued there after this call may overwrite it.
 * dict_len > 0 with a NULL d_dict, or d_dict not device memory of e's GPU, is refused.  e must outlive the stream.  NULL on a
 * refusal or when memory runs out. */
B200Stream* b200_stream_create(B200Encoder* e, size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values,
                               const uint8_t* d_dict, size_t dict_len, void* stream);
/* One BrotliEncoderCompressStream step, stream-ordered on `stream` (a cudaStream_t as void*): the n device bytes at d_in are
 * the new input, op is PROCESS, FLUSH or FINISH.  Returns 1 when the work has been enqueued; nothing on the host waits for it.
 *  - Bytes: the output of all calls on one stream, appended, equals byte for byte what BrotliEncoderCompressStream outputs for
 *    the same parameters, the same dictionary and the same sequence of (op, bytes).  The host and this call share one rule for
 *    when a piece is emitted (PROCESS: a 96 MiB piece whenever two are pending; FLUSH / FINISH: everything pending), its framing
 *    and size hint, and the window kept in front of it (b200_stage_stream_plan).
 *  - Input: d_in is copied into the stream's window buffer on `stream`, so work enqueued after the call may overwrite it.
 *  - Output: each piece is compressed into the stream's scratch buffer; the kernel k_stream_append then reads the piece's size
 *    and the cursor *d_out_size on the device, copies the piece to out + *d_out_size and advances the cursor.  So out[0,
 *    *d_out_size) is one contiguous stream over calls; reset *d_out_size to 0 between calls to get the pieces separately.
 *    *d_status is 0 on success.  A piece that does not fit in out_cap is not written at all and *d_status becomes 2; the stream
 *    is then failed (its host state has advanced): later calls append nothing and report 2.
 *  - Ordering: each call forks from `stream` and joins back into it, like b200_encoder_compress_range_async, and calls on one
 *    encoder run one at a time on the device.  The stream's host state advances when a call is enqueued, so calls on one
 *    B200Stream must be enqueued in the order they are meant to run (each call also waits, on the device, for the previous one).
 *  - Refused (0, nothing enqueued): NULL stream / out / d_out_size / d_status, d_in NULL with n > 0, pointers that are not device
 *    memory of the encoder's GPU, any op after FINISH, EMIT_METADATA, and `stream` capturing a CUDA graph (a replay would not
 *    advance the host state; the capture stays valid).  After a device failure inside a call (out of memory) the call returns 0
 *    and the stream is failed.
 *  - Memory: two window buffers of at most 1.5 x (2^lgwin + 68 KiB + the bytes not yet emitted + n) + 1 MiB each (PROCESS keeps fewer
 *    than 2 x 96 MiB pending), and an output scratch of b200_max_compressed_size(largest piece) + 128 bytes, pieces being at most
 *    1 GiB.  They grow when a call needs more, stream-ordered (cudaMallocAsync / cudaFreeAsync on `stream`): growing never waits
 *    on the host.  The encoder's workspace grows as for b200_encoder_compress_range_async. */
int b200_stream_compress_async(B200Stream* s, BrotliEncoderOperation op, const uint8_t* d_in, size_t n, uint8_t* out, size_t out_cap,
                               uint64_t* d_out_size, int32_t* d_status, void* stream);
/* An upper bound of the bytes b200_stream_compress_async(s, op, ..., n, ...) appends: size `out` by it; 0 for a refused op. */
size_t b200_stream_output_bound(const B200Stream* s, BrotliEncoderOperation op, size_t n);
/* Frees the stream's buffers stream-ordered on the CUDA stream of its last call (which must still exist); does not wait. */
void b200_stream_destroy(B200Stream* s);

/* Counters of one compression stream and the emits of one step (the rule BrotliEncoderCompressStream and b200_stream_* share). */
typedef struct B200StreamCounters {
  uint64_t base;          /* stream offset of the first byte still kept (a multiple of 4096); the dictionary starts at 0 */
  uint64_t flushed;       /* stream offset up to which output has been produced */
  uint64_t end;           /* stream offset of the end of the input so far */
  uint64_t dict_len;      /* custom dictionary bytes in front of the input */
  int32_t header_written; /* the stream header has been emitted */
  int32_t finished;       /* FINISH has been emitted */
} B200StreamCounters;
typedef struct B200StreamEmit {
  uint64_t start, upto;   /* stream bytes [start, upto) become output (empty for an end-of-stream byte) */
  uint64_t base;          /* the window base the emit compresses against (its input buffer begins at stream offset base) */
  uint64_t base_after;    /* the base once the emit is done: bytes in front of it are no longer needed */
  uint64_t size_hint;
  int32_t first, last;    /* the emit writes the stream header / ends the stream */
  int32_t byte;           /* >= 0: the emit's whole output is this byte (6: empty stream; 3: ISLAST + ISLASTEMPTY after a
                             byte-aligned flush); -1: the framed compression of [start, upto) */
} B200StreamEmit;
/* stage hooks of the stream rule (host code, no device needed).  start: the counters of a new stream whose custom dictionary has
 * dict_size bytes (0: none); *dict_from = index of the first dictionary byte kept.  plan: the emits of one step (op, n new bytes)
 * from counters *c, and the counters after it.  Both return 0 for a refused parameter; plan also for EMIT_METADATA, an unknown
 * op, input after FINISH, or more than max_emits emits. */
int b200_stage_stream_start(size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values, uint64_t dict_size,
                            B200StreamCounters* c, uint64_t* dict_from);
int b200_stage_stream_plan(size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values, const B200StreamCounters* c,
                           int op, uint64_t n, B200StreamEmit* emits, size_t max_emits, size_t* num_emits, B200StreamCounters* next);
/* One device call of the framing rule: compress input bytes [start, end), handed over from `rebase` on (the bytes in front of
 * start are its window), with the stream header (first), the end of the stream (last) or a byte-aligned end (byte_align). */
typedef struct B200FramedCall {
  uint64_t rebase, start, end;
  int32_t first, last, byte_align;
} B200FramedCall;
/* stage hook of the framing rule that BrotliEncoderCompress / CompressStream / CompressMulti, b200_encoder_compress_params_async
 * and b200_stream_* share (host code, no device needed): how input bytes [a, b) become output, given whether they begin the
 * stream (first), end it (last) and, when not last, end byte aligned (align_end).  The output is the prologue, the output of each
 * call in order, then the byte *trailer (-1: none).  prologue (32 bytes) receives the prologue's bytes; prologue_info = {length
 * in bytes, or -1 when there is none; offset and count of its placeholder bytes, which are input bytes a, a + 1; 1 when the
 * prologue, its trailing bits included, is the whole output: the one call then compresses nothing}.  Returns 0 for a refused
 * parameter, a framing that cannot end byte aligned, or more than max_calls calls. */
int b200_stage_framed_plan(size_t num_params, const BrotliEncoderParameter* keys, const uint32_t* values, uint64_t a, uint64_t b,
                           int first, int last, int align_end, uint8_t* prologue, int32_t* prologue_info, B200FramedCall* calls,
                           size_t max_calls, size_t* num_calls, int32_t* trailer);

/* ---- device splice of catable streams (the reference's BroCatli, src/concat/mod.rs; host ABI in broccoli.h) ---- */
/* Bytes of device workspace b200_concat_async needs for `count` streams. */
size_t b200_concat_workspace_size(uint32_t count);
/* Splices `count` device-resident streams into one, stream-ordered on `stream` (a cudaStream_t as void*).  d_streams[i] (device
 * array of device pointers) holds d_sizes[i] bytes (device array): the sizes are read on the device, so sizes written by
 * b200_encoder_compress_range_async earlier on `stream` need no host synchronisation.  out, d_out_size, d_result[2] and
 * d_workspace (>= b200_concat_workspace_size(count) bytes) are device memory.
 *  - Result: out[0, *d_out_size) and d_result equal the host sequence window_size ? BroccoliCreateInstanceWithWindowSize(window_size)
 *    : BroccoliCreateInstance(), then per stream BroccoliNewBrotliFile + BroccoliConcatStream over all of its bytes with unbounded
 *    output, then BroccoliConcatFinish.  d_result = {0, -1} on success.
 *  - All or nothing: on the first stream whose ConcatStream fails, d_result = {code (124..127), stream index}; when the output
 *    would pass out_cap, {2, index of the first stream that does not fit, or count for the final bytes}.  Then *d_out_size = 0
 *    and nothing is written to out.
 *  - Size: the output never exceeds the sum of the sizes + 3 bytes (derivation in csrc/bro_concat.cuh); offsets are 64-bit.
 *  - Allocates nothing, never waits on the host and is capturable in a CUDA graph: four launches and one memset on `stream`.
 *    Returns 0 (nothing enqueued) for null pointers, a short workspace, count > 2^31 - 1 or window_size outside 0..255. */
int b200_concat_async(const uint8_t* const* d_streams, const uint64_t* d_sizes, uint32_t count, int window_size, uint8_t* out,
                      size_t out_cap, uint64_t* d_out_size, int32_t* d_result, void* d_workspace, size_t workspace_bytes, void* stream);
/* stage hook of quality 5..9: best[] of the match stage (distance << 8 | capped length, or a static-dictionary candidate) for
 * [range_start, range_start + range_len) of an n-byte buffer, range_len <= one chunk; size_hint 0 = n.  search = 0: the up-front
 * kernels; search = 1: the on-demand search at every position (returns 0 where that path does not run: depth < 64, two batches) */
int b200_stage_match(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, const uint8_t* in, size_t n, size_t range_start,
                     size_t range_len, int search, uint32_t* best_out);
/* stage hook after b200_stage_match with search = 0 at bucket depth 16 / 32 (q5, q6), where best[] is stored through a staging
 * region cut into slabs of 2^21 positions of each sort batch's payload.  For the range's last batch, cursors[s] = records the
 * match kernel claimed in slab s and sizes[s] = records slab s must receive (s < cap).  Returns the number of slabs, 0 when
 * the last call did not stage best[]. */
int b200_stage_match_slabs(B200Encoder* e, uint32_t* cursors, uint32_t* sizes, uint32_t cap);
/* the same for the tiles of 2^13 positions of each batch's payload that the placement fills after the slabs: cursors[t] = records
 * claimed in tile t of the last batch, sizes[t] = records tile t must receive (t < cap).  Returns the number of tiles, 0 when the
 * last call did not stage best[]. */
int b200_stage_match_tiles(B200Encoder* e, uint32_t* cursors, uint32_t* sizes, uint32_t cap);
/* stage hook of quality 10 / 11 (n <= one chunk): matches per position hqn[n], hqm[n][16][2] (distance, length word); per parse
 * unit ncmd, tail, ncopy as units[3][nu]; raw commands raw[nu][unit / 2 + 1][3].  b200_hq_unit gives the unit for size_hint n. */
int b200_stage_hq(B200Encoder* e, int quality, int lgwin, const uint8_t* in, size_t n, uint8_t* hqn, uint32_t* hqm, uint32_t* units,
                  uint32_t* raw);
uint32_t b200_hq_unit(B200Encoder* e, int quality, uint64_t size_hint);
/* stage hook of the sort: the positions 0..n-1 (n <= 2^25) sorted stably by the bucket key of quality / lgwin / size n, or with
 * level 0..2 by the key of that long-prefix level of quality 10 / 11 */
int b200_stage_sort(B200Encoder* e, int quality, int lgwin, const uint8_t* in, size_t n, int level, uint32_t* sorted_out);

#ifdef __cplusplus
}
#endif
#endif /* BROTLI_B200_H_ */

/* bro_encoder.h -- internal C interface of the device encoder (the public C ABI is include/brotli_b200.h). */
#pragma once
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
typedef struct B200Encoder B200Encoder;
enum { B200_OPT_CTX_MODEL = 6, B200_OPT_TIMING = 7, B200_OPT_LANES = 8, B200_OPT_DICT = 9, B200_OPT_HQ_SPLIT = 12, B200_OPT_HQ_UNIT = 13, B200_OPT_ONDEMAND = 15, B200_OPT_HQ_LEVELS = 16,
       B200_OPT_Q9_5 = 17 /* BROTLI_PARAM_Q9_5: quality 10 / 11 run the hash-chain parse under their metablock builder */ };
/* stage timing slots of b200_encoder_last_timings */
enum { B200_ST_SORT = 0, B200_ST_MATCH = 1, B200_ST_PARSE = 2, B200_ST_FINALIZE = 3, B200_ST_SPLIT = 4, B200_ST_HEADER = 5,
       B200_ST_EMIT = 6, B200_NUM_STAGES = 7 };
int b200_device_count(void);
int b200_effective_quality(int requested_quality);
B200Encoder* b200_encoder_create(int device);
void b200_encoder_destroy(B200Encoder* e);
int b200_encoder_set_option(B200Encoder* e, int option, uint32_t value);
size_t b200_max_compressed_size(size_t n);
int b200_encoder_compress(B200Encoder* e, int quality, int lgwin, const uint8_t* in, size_t n, uint8_t* out, size_t out_cap,
                          size_t* out_size, int device_io);
int b200_encoder_compress_range(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, const uint8_t* in, size_t n,
                                size_t range_start, size_t range_len, int first, int last, int byte_align, uint8_t* out,
                                size_t out_cap, size_t* out_size, int device_io);
int b200_encoder_reserve(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, size_t n, size_t range_len);
int b200_encoder_compress_range_async(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, const uint8_t* in, size_t n,
                                      size_t range_start, size_t range_len, int first, int last, int byte_align, uint8_t* out,
                                      size_t out_cap, uint64_t* out_size, void* stream);
/* Framed stream-ordered compression (b200_encoder_compress_params_async builds on it).  The prologue of a framed stream (window
 * bits, magic-number metadata block, catable uncompressed metablock -- bro_capi.cu:write_prologue) as built on the host: `len`
 * bytes, of which [data_off, data_off + n2) are placeholders for the first n2 input bytes.  complete: the prologue is the whole
 * stream (nothing left to compress, trailer included). */
typedef struct B200Prologue {
  uint8_t bytes[32];
  uint32_t len, data_off, n2, complete;
} B200Prologue;
/* b200_encoder_compress_range_async behind a prologue: the range's first metablock starts at byte pro->len (pro may be NULL), and
 * trailer >= 0 appends that byte behind the range's byte-aligned end.  The prologue's n2 data bytes are the input bytes right in
 * front of range_start.  ctx_model / use_dict / q9_5 apply to this call only (-1: the encoder's option). */
int b200_encoder_compress_framed_async(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, int ctx_model, int use_dict,
                                       int q9_5, const uint8_t* in, size_t n, size_t range_start, size_t range_len, int first,
                                       int last, int byte_align, const B200Prologue* pro, int trailer, uint8_t* out, size_t out_cap,
                                       uint64_t* out_size, void* stream);
int b200_encoder_last_timings(B200Encoder* e, float* ms /* [B200_NUM_STAGES] */, uint32_t* launches);
int b200_stage_match(B200Encoder* e, int quality, int lgwin, uint64_t size_hint, const uint8_t* in, size_t n, size_t range_start,
                     size_t range_len, int search, uint32_t* best_out);
int b200_stage_match_slabs(B200Encoder* e, uint32_t* cursors, uint32_t* sizes, uint32_t cap);
int b200_stage_hq(B200Encoder* e, int quality, int lgwin, const uint8_t* in, size_t n, uint8_t* hqn, uint32_t* hqm, uint32_t* units,
                  uint32_t* raw);
uint32_t b200_hq_unit(B200Encoder* e, int quality, uint64_t size_hint);
int b200_stage_sort(B200Encoder* e, int quality, int lgwin, const uint8_t* in, size_t n, int level, uint32_t* sorted_out);
#ifdef __cplusplus
}
#endif

//! `extern "C"` declarations of include/brotli_b200.h -- the same symbols the reference exports from
//! src/ffi/compressor.rs and src/ffi/multicompress/mod.rs, plus the device-resident additions.
#![allow(non_camel_case_types, non_snake_case)]
use std::os::raw::c_void;

#[repr(C)]
pub struct BrotliEncoderState {
    _private: [u8; 0],
}
#[repr(C)]
pub struct BrotliEncoderWorkPool {
    _private: [u8; 0],
}
#[repr(C)]
pub struct B200Encoder {
    _private: [u8; 0],
}
#[repr(C)]
pub struct B200Stream {
    _private: [u8; 0],
}

pub type brotli_alloc_func = Option<unsafe extern "C" fn(opaque: *mut c_void, size: usize) -> *mut c_void>;
pub type brotli_free_func = Option<unsafe extern "C" fn(opaque: *mut c_void, address: *mut c_void)>;

/// src/enc/encode.rs:1380-1385
#[repr(C)]
#[derive(Clone, Copy, PartialEq, Eq, Debug)]
pub enum BrotliEncoderOperation {
    BROTLI_OPERATION_PROCESS = 0,
    BROTLI_OPERATION_FLUSH = 1,
    BROTLI_OPERATION_FINISH = 2,
    BROTLI_OPERATION_EMIT_METADATA = 3,
}

/// Numeric values of src/enc/parameters.rs:1-32 (passed as plain u32 keys).
pub mod param {
    pub const MODE: u32 = 0;
    pub const QUALITY: u32 = 1;
    pub const LGWIN: u32 = 2;
    pub const LGBLOCK: u32 = 3;
    pub const DISABLE_LITERAL_CONTEXT_MODELING: u32 = 4;
    pub const SIZE_HINT: u32 = 5;
    pub const LARGE_WINDOW: u32 = 6;
    pub const Q9_5: u32 = 150;
    pub const CATABLE: u32 = 167;
    pub const APPENDABLE: u32 = 168;
    pub const MAGIC_NUMBER: u32 = 169;
    pub const NO_DICTIONARY: u32 = 170;
    pub const BYTE_ALIGN: u32 = 172;
    pub const BARE_STREAM: u32 = 173;
}

extern "C" {
    // ---- src/ffi/compressor.rs ----
    pub fn BrotliEncoderCreateInstance(alloc: brotli_alloc_func, free: brotli_free_func, opaque: *mut c_void) -> *mut BrotliEncoderState;
    pub fn BrotliEncoderSetParameter(state: *mut BrotliEncoderState, p: u32, value: u32) -> i32;
    pub fn BrotliEncoderDestroyInstance(state: *mut BrotliEncoderState);
    pub fn BrotliEncoderIsFinished(state: *mut BrotliEncoderState) -> i32;
    pub fn BrotliEncoderHasMoreOutput(state: *mut BrotliEncoderState) -> i32;
    pub fn BrotliEncoderSetCustomDictionary(state: *mut BrotliEncoderState, size: usize, dict: *const u8);
    pub fn BrotliEncoderTakeOutput(state: *mut BrotliEncoderState, size: *mut usize) -> *const u8;
    pub fn BrotliEncoderVersion() -> u32;
    pub fn BrotliEncoderMaxCompressedSize(input_size: usize) -> usize;
    pub fn BrotliEncoderCompress(quality: i32, lgwin: i32, mode: i32, input_size: usize, input: *const u8,
                                 encoded_size: *mut usize, encoded: *mut u8) -> i32;
    pub fn BrotliEncoderCompressStreaming(state: *mut BrotliEncoderState, op: BrotliEncoderOperation, available_in: *mut usize,
                                          input: *const u8, available_out: *mut usize, output: *mut u8) -> i32;
    pub fn BrotliEncoderCompressStream(state: *mut BrotliEncoderState, op: BrotliEncoderOperation, available_in: *mut usize,
                                       next_in: *mut *const u8, available_out: *mut usize, next_out: *mut *mut u8,
                                       total_out: *mut usize) -> i32;
    pub fn BrotliEncoderMallocU8(state: *mut BrotliEncoderState, size: usize) -> *mut u8;
    pub fn BrotliEncoderFreeU8(state: *mut BrotliEncoderState, data: *mut u8, size: usize);
    pub fn BrotliEncoderMallocUsize(state: *mut BrotliEncoderState, size: usize) -> *mut usize;
    pub fn BrotliEncoderFreeUsize(state: *mut BrotliEncoderState, data: *mut usize, size: usize);
    // ---- src/ffi/multicompress/mod.rs ----
    pub fn BrotliEncoderMaxCompressedSizeMulti(input_size: usize, num_threads: usize) -> usize;
    pub fn BrotliEncoderCompressMulti(num_params: usize, keys: *const u32, values: *const u32, input_size: usize,
                                      input: *const u8, encoded_size: *mut usize, encoded: *mut u8, desired_num_threads: usize,
                                      alloc: brotli_alloc_func, free: brotli_free_func, opaque_per_thread: *mut *mut c_void) -> i32;
    pub fn BrotliEncoderCreateWorkPool(num_workers: usize, alloc: brotli_alloc_func, free: brotli_free_func,
                                       opaque_per_thread: *mut *mut c_void) -> *mut BrotliEncoderWorkPool;
    pub fn BrotliEncoderDestroyWorkPool(pool: *mut BrotliEncoderWorkPool);
    pub fn BrotliEncoderCompressWorkPool(pool: *mut BrotliEncoderWorkPool, num_params: usize, keys: *const u32, values: *const u32,
                                         input_size: usize, input: *const u8, encoded_size: *mut usize, encoded: *mut u8,
                                         desired_num_threads: usize, alloc: brotli_alloc_func, free: brotli_free_func,
                                         opaque_per_thread: *mut *mut c_void) -> i32;
    // ---- device-resident additions ----
    pub fn b200_device_count() -> i32;
    pub fn b200_effective_quality(requested_quality: i32) -> i32;
    pub fn b200_encoder_create(device: i32) -> *mut B200Encoder;
    pub fn b200_encoder_destroy(e: *mut B200Encoder);
    pub fn b200_max_compressed_size(n: usize) -> usize;
    pub fn b200_encoder_compress_range(e: *mut B200Encoder, quality: i32, lgwin: i32, size_hint: u64, input: *const u8, n: usize,
                                       range_start: usize, range_len: usize, first: i32, last: i32, byte_align: i32, out: *mut u8,
                                       out_cap: usize, out_size: *mut usize, device_io: i32) -> i32;
    pub fn b200_encoder_reserve(e: *mut B200Encoder, quality: i32, lgwin: i32, size_hint: u64, n: usize, range_len: usize) -> i32;
    /// `input`, `out` and `out_size` are device pointers; `stream` is a `cudaStream_t` (null = the legacy default stream).
    pub fn b200_encoder_compress_range_async(e: *mut B200Encoder, quality: i32, lgwin: i32, size_hint: u64, input: *const u8,
                                             n: usize, range_start: usize, range_len: usize, first: i32, last: i32,
                                             byte_align: i32, out: *mut u8, out_cap: usize, out_size: *mut u64,
                                             stream: *mut c_void) -> i32;
    /// `input`, `out` and `out_size` are device pointers; `keys` / `values` are host arrays of `num_params` entries.
    pub fn b200_encoder_compress_params_async(e: *mut B200Encoder, num_params: usize, keys: *const u32, values: *const u32,
                                              input: *const u8, n: usize, out: *mut u8, out_cap: usize, out_size: *mut u64,
                                              stream: *mut c_void) -> i32;
    /// Device-resident stream (include/brotli_b200.h): `d_dict` is a device pointer (null: no custom dictionary); `stream` is a
    /// `cudaStream_t`.  Null on a refused parameter or dictionary.
    pub fn b200_stream_create(e: *mut B200Encoder, num_params: usize, keys: *const u32, values: *const u32, d_dict: *const u8,
                              dict_len: usize, stream: *mut c_void) -> *mut B200Stream;
    /// One PROCESS / FLUSH / FINISH step (`op` as BrotliEncoderOperation); `input`, `out`, `out_size` and `status` are device
    /// pointers.  Returns 1 when enqueued.
    pub fn b200_stream_compress_async(s: *mut B200Stream, op: i32, input: *const u8, n: usize, out: *mut u8, out_cap: usize,
                                      out_size: *mut u64, status: *mut i32, stream: *mut c_void) -> i32;
    pub fn b200_stream_output_bound(s: *const B200Stream, op: i32, n: usize) -> usize;
    pub fn b200_stream_destroy(s: *mut B200Stream);
    pub fn b200_concat_workspace_size(count: u32) -> usize;
    /// Every pointer is a device pointer; `stream` is a `cudaStream_t`.
    pub fn b200_concat_async(streams: *const *const u8, sizes: *const u64, count: u32, window_size: i32, out: *mut u8,
                             out_cap: usize, out_size: *mut u64, result: *mut i32, workspace: *mut c_void, workspace_bytes: usize,
                             stream: *mut c_void) -> i32;
    // ---- src/ffi/broccoli.rs (include/broccoli.h) ----
    pub fn BroccoliCreateInstance() -> BroccoliState;
    pub fn BroccoliCreateInstanceWithWindowSize(window_size: u8) -> BroccoliState;
    pub fn BroccoliDestroyInstance(state: BroccoliState);
    pub fn BroccoliNewBrotliFile(state: *mut BroccoliState);
    pub fn BroccoliConcatStream(state: *mut BroccoliState, available_in: *mut usize, input_buf_ptr: *mut *const u8,
                                available_out: *mut usize, output_buf_ptr: *mut *mut u8) -> BroccoliResult;
    pub fn BroccoliConcatStreaming(state: *mut BroccoliState, available_in: *mut usize, input_buf: *const u8,
                                   available_out: *mut usize, output_buf: *mut u8) -> BroccoliResult;
    pub fn BroccoliConcatFinish(state: *mut BroccoliState, available_out: *mut usize, output_buf_ptr: *mut *mut u8) -> BroccoliResult;
    pub fn BroccoliConcatFinished(state: *mut BroccoliState, available_out: *mut usize, output_buf: *mut u8) -> BroccoliResult;
}

/// include/broccoli.h: the whole splice state as plain data (`unused` is always null).
#[repr(C)]
#[derive(Clone, Copy)]
pub struct BroccoliState {
    pub unused: *mut c_void,
    pub data: [u8; 248],
}

/// BroccoliResult (src/concat/mod.rs:3-13); a C enum, passed as an int.
pub type BroccoliResult = i32;
pub const BROCCOLI_SUCCESS: BroccoliResult = 0;
pub const BROCCOLI_NEEDS_MORE_INPUT: BroccoliResult = 1;
pub const BROCCOLI_NEEDS_MORE_OUTPUT: BroccoliResult = 2;
pub const BROCCOLI_BROTLI_FILE_NOT_CRAFTED_FOR_APPEND: BroccoliResult = 124;
pub const BROCCOLI_INVALID_WINDOW_SIZE: BroccoliResult = 125;
pub const BROCCOLI_WINDOW_SIZE_LARGER_THAN_PREVIOUS_FILE: BroccoliResult = 126;
pub const BROCCOLI_BROTLI_FILE_NOT_CRAFTED_FOR_CONCATENATION: BroccoliResult = 127;

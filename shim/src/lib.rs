//! Drop-in surface of the reference crate's compression path on top of libbrotli_b200 (CUDA, sm_90a).
//!
//! Same names and argument meaning as the reference:
//!   * `BrotliEncoderParams`                 src/enc/backward_references/mod.rs:71, defaults src/enc/encode.rs:318-357
//!   * `CompressorWriter::{new, with_params, write, flush, into_inner}`   src/enc/writer.rs:83-118 (Drop finishes, :253-265)
//!   * `CompressorReader::{new, with_params, read, into_inner}`           src/enc/reader.rs:74-103
//!   * `BrotliCompress(r, w, &params) -> io::Result<usize>`               src/enc/mod.rs:142
//!   * `compress_multi(&params, input, output, num_threads)`              src/enc/mod.rs:95-133 (allocators: device memory is
//!     owned by the library, so the `alloc_per_thread` slice of the reference shrinks to its length = the shard count)
//!   * `BrotliEncoderMaxCompressedSize{,Multi}`                           src/enc/encode.rs:1273-1299
//! Errors: `io::ErrorKind::InvalidData` where the reference's writer reports a failed `compress_stream`
//! (writer.rs:43-44); `BrotliEncoderThreadError` for the multi path (threading/mod.rs:33-40).  There is no CPU fallback:
//! without a CUDA device every constructor fails.
pub mod ffi;

use std::io::{self, ErrorKind, Read, Write};

pub const MAX_THREADS: usize = 16; // src/enc/fixed_queue.rs:1

#[derive(Clone, Debug)]
pub struct BrotliEncoderParams {
    pub mode: u32,
    pub quality: i32,
    pub lgwin: i32,
    pub lgblock: i32,
    pub size_hint: usize,
    pub disable_literal_context_modeling: i32,
    pub catable: bool,
    pub appendable: bool,
    pub magic_number: bool,
    pub byte_align: bool,
    pub bare_stream: bool,
    pub use_dictionary: bool,
    /// "quality 9.5": with quality 10 / 11, the hash-chain parse under the quality 10 / 11 metablock builder
    pub q9_5: bool,
}

impl Default for BrotliEncoderParams {
    fn default() -> Self {
        // encode.rs:318-357
        BrotliEncoderParams { mode: 0, quality: 11, lgwin: 22, lgblock: 0, size_hint: 0, disable_literal_context_modeling: 0,
                              catable: false, appendable: false, magic_number: false, byte_align: false, bare_stream: false,
                              use_dictionary: true, q9_5: false }
    }
}

impl BrotliEncoderParams {
    fn key_values(&self) -> Vec<(u32, u32)> {
        use ffi::param::*;
        let mut kv = vec![(QUALITY, self.quality as u32), (LGWIN, self.lgwin as u32), (MODE, self.mode)];
        if self.lgblock != 0 { kv.push((LGBLOCK, self.lgblock as u32)); }
        if self.size_hint != 0 { kv.push((SIZE_HINT, std::cmp::min(self.size_hint, u32::MAX as usize) as u32)); }
        if self.disable_literal_context_modeling != 0 { kv.push((DISABLE_LITERAL_CONTEXT_MODELING, 1)); }
        if !self.use_dictionary { kv.push((NO_DICTIONARY, 1)); }
        if self.q9_5 { kv.push((Q9_5, 1)); }
        for (k, on) in [(CATABLE, self.catable), (APPENDABLE, self.appendable), (MAGIC_NUMBER, self.magic_number),
                        (BYTE_ALIGN, self.byte_align), (BARE_STREAM, self.bare_stream)].iter() {
            if *on { kv.push((*k, 1)); }
        }
        kv
    }
}

pub fn BrotliEncoderMaxCompressedSize(input_size: usize) -> usize {
    unsafe { ffi::BrotliEncoderMaxCompressedSize(input_size) }
}
pub fn BrotliEncoderMaxCompressedSizeMulti(input_size: usize, num_threads: usize) -> usize {
    unsafe { ffi::BrotliEncoderMaxCompressedSizeMulti(input_size, num_threads) }
}

/// One `BrotliEncoderState` driven through `BrotliEncoderCompressStream`, as writer.rs / reader.rs drive theirs.
struct Stream {
    h: *mut ffi::BrotliEncoderState,
}

impl Stream {
    fn new(params: &BrotliEncoderParams) -> io::Result<Stream> {
        let h = unsafe { ffi::BrotliEncoderCreateInstance(None, None, std::ptr::null_mut()) };
        if h.is_null() {
            return Err(io::Error::new(ErrorKind::Other, "BrotliEncoderCreateInstance failed: no usable CUDA device"));
        }
        let s = Stream { h };
        for (k, v) in params.key_values() {
            if unsafe { ffi::BrotliEncoderSetParameter(s.h, k, v) } == 0 {
                return Err(io::Error::new(ErrorKind::InvalidInput, "parameter not produced by the GPU path"));
            }
        }
        Ok(s)
    }
    /// Feeds `input` with operation `op` and hands every produced byte to `sink`.
    fn step<F: FnMut(&[u8]) -> io::Result<()>>(&mut self, input: &[u8], op: ffi::BrotliEncoderOperation, mut sink: F) -> io::Result<()> {
        let mut avail_in = input.len();
        let mut next_in = input.as_ptr();
        let mut buf = [0u8; 65536];
        loop {
            let mut avail_out = buf.len();
            let mut next_out = buf.as_mut_ptr();
            let mut total = 0usize;
            let ok = unsafe {
                ffi::BrotliEncoderCompressStream(self.h, op, &mut avail_in, &mut next_in, &mut avail_out, &mut next_out, &mut total)
            };
            if ok == 0 {
                return Err(io::Error::new(ErrorKind::InvalidData, "BrotliEncoderCompressStream failed")); // writer.rs:43-44
            }
            let n = buf.len() - avail_out;
            if n != 0 { sink(&buf[..n])?; }
            if avail_in == 0 && unsafe { ffi::BrotliEncoderHasMoreOutput(self.h) } == 0 { return Ok(()); }
        }
    }
}

impl Drop for Stream {
    fn drop(&mut self) {
        unsafe { ffi::BrotliEncoderDestroyInstance(self.h) }
    }
}

pub struct CompressorWriter<W: Write> {
    w: Option<W>,
    s: Stream,
    finished: bool,
}

impl<W: Write> CompressorWriter<W> {
    pub fn new(w: W, _buffer_size: usize, q: u32, lgwin: u32) -> Self {
        let params = BrotliEncoderParams { quality: q as i32, lgwin: lgwin as i32, ..Default::default() };
        Self::with_params(w, _buffer_size, &params)
    }
    pub fn with_params(w: W, _buffer_size: usize, params: &BrotliEncoderParams) -> Self {
        // the reference's constructors are infallible; a missing device surfaces as InvalidData on the first write
        let s = Stream::new(params).unwrap_or(Stream { h: std::ptr::null_mut() });
        CompressorWriter { w: Some(w), s, finished: false }
    }
    pub fn get_ref(&self) -> &W { self.w.as_ref().unwrap() }
    pub fn get_mut(&mut self) -> &mut W { self.w.as_mut().unwrap() }
    fn run(&mut self, buf: &[u8], op: ffi::BrotliEncoderOperation) -> io::Result<()> {
        if self.s.h.is_null() { return Err(io::Error::new(ErrorKind::InvalidData, "no usable CUDA device")); }
        let w = self.w.as_mut().unwrap();
        self.s.step(buf, op, |out| w.write_all(out))
    }
    fn finish(&mut self) -> io::Result<()> {
        if !self.finished {
            self.finished = true;
            self.run(&[], ffi::BrotliEncoderOperation::BROTLI_OPERATION_FINISH)?;
        }
        Ok(())
    }
    pub fn into_inner(mut self) -> W {
        let _ = self.finish();
        self.w.take().unwrap()
    }
}

impl<W: Write> Write for CompressorWriter<W> {
    fn write(&mut self, buf: &[u8]) -> io::Result<usize> {
        self.run(buf, ffi::BrotliEncoderOperation::BROTLI_OPERATION_PROCESS)?;
        Ok(buf.len())
    }
    fn flush(&mut self) -> io::Result<()> {
        self.run(&[], ffi::BrotliEncoderOperation::BROTLI_OPERATION_FLUSH)?;
        self.w.as_mut().unwrap().flush()
    }
}

impl<W: Write> Drop for CompressorWriter<W> {
    fn drop(&mut self) {
        if self.w.is_some() { let _ = self.finish(); } // writer.rs:253-265
    }
}

pub struct CompressorReader<R: Read> {
    r: R,
    s: Stream,
    pending: Vec<u8>,
    pos: usize,
    eof: bool,
    chunk: Vec<u8>,
}

impl<R: Read> CompressorReader<R> {
    pub fn new(r: R, buffer_size: usize, q: u32, lgwin: u32) -> Self {
        let params = BrotliEncoderParams { quality: q as i32, lgwin: lgwin as i32, ..Default::default() };
        Self::with_params(r, buffer_size, &params)
    }
    pub fn with_params(r: R, buffer_size: usize, params: &BrotliEncoderParams) -> Self {
        let s = Stream::new(params).unwrap_or(Stream { h: std::ptr::null_mut() });
        CompressorReader { r, s, pending: Vec::new(), pos: 0, eof: false, chunk: vec![0u8; if buffer_size == 0 { 4096 } else { buffer_size }] }
    }
    pub fn into_inner(self) -> R { self.r }
}

impl<R: Read> Read for CompressorReader<R> {
    fn read(&mut self, out: &mut [u8]) -> io::Result<usize> {
        if self.s.h.is_null() { return Err(io::Error::new(ErrorKind::InvalidData, "no usable CUDA device")); }
        while self.pos == self.pending.len() && !self.eof {
            self.pending.clear();
            self.pos = 0;
            let n = self.r.read(&mut self.chunk)?;
            let pending = &mut self.pending;
            if n == 0 {
                self.eof = true;
                self.s.step(&[], ffi::BrotliEncoderOperation::BROTLI_OPERATION_FINISH, |o| { pending.extend_from_slice(o); Ok(()) })?;
            } else {
                self.s.step(&self.chunk[..n], ffi::BrotliEncoderOperation::BROTLI_OPERATION_PROCESS, |o| { pending.extend_from_slice(o); Ok(()) })?;
            }
        }
        let n = std::cmp::min(out.len(), self.pending.len() - self.pos);
        out[..n].copy_from_slice(&self.pending[self.pos..self.pos + n]);
        self.pos += n;
        Ok(n)
    }
}

/// src/enc/mod.rs:142
pub fn BrotliCompress<R: Read, W: Write>(r: &mut R, w: &mut W, params: &BrotliEncoderParams) -> io::Result<usize> {
    struct Counting<'a, W: Write> { w: &'a mut W, n: usize }
    impl<'a, W: Write> Write for Counting<'a, W> {
        fn write(&mut self, b: &[u8]) -> io::Result<usize> { let k = self.w.write(b)?; self.n += k; Ok(k) }
        fn flush(&mut self) -> io::Result<()> { self.w.flush() }
    }
    let mut cw = CompressorWriter::with_params(Counting { w, n: 0 }, 4096, params);
    io::copy(r, &mut cw)?;
    cw.finish()?;
    Ok(cw.get_ref().n)
}

/// src/enc/threading/mod.rs:33-40
#[derive(Debug)]
pub enum BrotliEncoderThreadError {
    InsufficientOutputSpace,
    ConcatenationDidNotProcessFullFile,
    ConcatenationError(i32),
    ConcatenationFinalizationError(i32),
    OtherThreadPanic,
    ThreadExecError(String),
}

/// `compress_multi` (src/enc/mod.rs:95-133): `num_threads` shards (<= 16, get_range threading/mod.rs:333), placed round-robin
/// on the visible GPUs; shard i > 0 sees the previous 2^lgwin input bytes as its window; the byte-aligned shard outputs are
/// concatenated in order.  The input is only borrowed.
pub fn compress_multi(params: &BrotliEncoderParams, input: &[u8], output: &mut [u8], num_threads: usize) -> Result<usize, BrotliEncoderThreadError> {
    if num_threads == 0 || num_threads > MAX_THREADS {
        return Err(BrotliEncoderThreadError::ThreadExecError("1..=16 shards".to_string()));
    }
    let kv = params.key_values();
    let keys: Vec<u32> = kv.iter().map(|x| x.0).collect();
    let vals: Vec<u32> = kv.iter().map(|x| x.1).collect();
    let mut n = output.len();
    let ok = unsafe {
        ffi::BrotliEncoderCompressMulti(kv.len(), keys.as_ptr(), vals.as_ptr(), input.len(), input.as_ptr(), &mut n, output.as_mut_ptr(),
                                        num_threads, None, None, std::ptr::null_mut())
    };
    if ok != 0 { return Ok(n); }
    if output.len() < BrotliEncoderMaxCompressedSizeMulti(input.len(), num_threads) {
        Err(BrotliEncoderThreadError::InsufficientOutputSpace)
    } else {
        Err(BrotliEncoderThreadError::OtherThreadPanic) // CUDA failure or a parameter this path does not produce
    }
}

/// `BroCatli` (src/concat/mod.rs:125-605) over the Broccoli C ABI: `new`, `new_with_window_size`, `new_brotli_file`,
/// `stream(in, &mut in_offset, out, &mut out_offset)` and `finish(out, &mut out_offset)` with the reference's result codes.
/// Host code: needs no CUDA device.
pub struct BroCatli {
    state: ffi::BroccoliState,
}

impl Default for BroCatli {
    fn default() -> Self {
        Self::new()
    }
}

impl BroCatli {
    pub fn new() -> Self {
        BroCatli { state: unsafe { ffi::BroccoliCreateInstance() } }
    }
    /// A size the reference refuses gives a default instance (broccoli.rs:60-65).
    pub fn new_with_window_size(log_window_size: u8) -> Self {
        BroCatli { state: unsafe { ffi::BroccoliCreateInstanceWithWindowSize(log_window_size) } }
    }
    pub fn new_brotli_file(&mut self) {
        unsafe { ffi::BroccoliNewBrotliFile(&mut self.state) }
    }
    pub fn stream(&mut self, in_bytes: &[u8], in_offset: &mut usize, out_bytes: &mut [u8], out_offset: &mut usize) -> ffi::BroccoliResult {
        let input = &in_bytes[*in_offset..];
        let output = &mut out_bytes[*out_offset..];
        let (mut avail_in, mut avail_out) = (input.len(), output.len());
        let r = unsafe { ffi::BroccoliConcatStreaming(&mut self.state, &mut avail_in, input.as_ptr(), &mut avail_out, output.as_mut_ptr()) };
        *in_offset += input.len() - avail_in;
        *out_offset += output.len() - avail_out;
        r
    }
    pub fn finish(&mut self, out_bytes: &mut [u8], out_offset: &mut usize) -> ffi::BroccoliResult {
        let output = &mut out_bytes[*out_offset..];
        let mut avail_out = output.len();
        let r = unsafe { ffi::BroccoliConcatFinished(&mut self.state, &mut avail_out, output.as_mut_ptr()) };
        *out_offset += output.len() - avail_out;
        r
    }
}

"""rust-brotli_b200 -- host-side mirror of the reference's compression API surface over the C ABI.

The reference (dropbox/rust-brotli) exposes, for the compression path:
  * ``BrotliEncoderParams``                      src/enc/backward_references/mod.rs:71, defaults src/enc/encode.rs:318
  * ``CompressorWriter`` / ``CompressorReader``  src/enc/writer.rs:74, src/enc/reader.rs:65
  * ``BrotliCompress(r, w, params)``             src/enc/mod.rs:142
  * ``compress_multi(params, input, ...)``       src/enc/mod.rs:95
  * ``BrotliEncoderMaxCompressedSize{,Multi}``   src/enc/encode.rs:1273-1299
The host language of the reference is Rust; this image has no Rust toolchain, so the mirror is Python (what the
reference's own c/py wrapper does) calling the same ``BrotliEncoder*`` C ABI a Rust shim would bind -- see
INTEGRATION.md.  Every byte of compressed output comes from the CUDA library; nothing here compresses on the CPU
and importing this package on a machine without the built library raises at first use.
"""
import ctypes
import io
from dataclasses import dataclass

from . import _native
from ._native import DeviceEncoder, lib  # noqa: F401

# BrotliEncoderParameter (src/enc/parameters.rs:1-32)
BROTLI_PARAM_MODE, BROTLI_PARAM_QUALITY, BROTLI_PARAM_LGWIN, BROTLI_PARAM_LGBLOCK = 0, 1, 2, 3
BROTLI_PARAM_DISABLE_LITERAL_CONTEXT_MODELING, BROTLI_PARAM_SIZE_HINT, BROTLI_PARAM_LARGE_WINDOW = 4, 5, 6
BROTLI_PARAM_Q9_5 = 150
BROTLI_PARAM_CATABLE, BROTLI_PARAM_APPENDABLE, BROTLI_PARAM_MAGIC_NUMBER = 167, 168, 169
BROTLI_PARAM_NO_DICTIONARY, BROTLI_PARAM_BYTE_ALIGN, BROTLI_PARAM_BARE_STREAM = 170, 172, 173
BROTLI_OPERATION_PROCESS, BROTLI_OPERATION_FLUSH, BROTLI_OPERATION_FINISH = 0, 1, 2
MAX_THREADS = 16  # src/enc/fixed_queue.rs:1


class BrotliEncoderThreadError(Exception):
    """src/enc/threading/mod.rs:33-40"""


class InsufficientOutputSpace(BrotliEncoderThreadError):
    pass


class OtherThreadPanic(BrotliEncoderThreadError):
    pass


@dataclass
class BrotliEncoderParams:
    """Subset of the reference struct that parameterises this path (defaults: encode.rs:318-357)."""
    quality: int = 11
    lgwin: int = 22
    lgblock: int = 0
    size_hint: int = 0
    mode: int = 0
    disable_literal_context_modeling: int = 0
    catable: bool = False
    appendable: bool = False
    magic_number: bool = False
    byte_align: bool = False
    bare_stream: bool = False
    use_dictionary: bool = True
    q9_5: bool = False  # "quality 9.5": with quality 10 / 11, the hash-chain parse under the quality 10 / 11 metablock builder

    def as_key_values(self):
        kv = [(BROTLI_PARAM_QUALITY, self.quality), (BROTLI_PARAM_LGWIN, self.lgwin), (BROTLI_PARAM_MODE, self.mode)]
        if self.size_hint:
            kv.append((BROTLI_PARAM_SIZE_HINT, min(self.size_hint, 0xFFFFFFFF)))
        if self.disable_literal_context_modeling:
            kv.append((BROTLI_PARAM_DISABLE_LITERAL_CONTEXT_MODELING, 1))
        if self.lgblock:
            kv.append((BROTLI_PARAM_LGBLOCK, self.lgblock))
        if not self.use_dictionary:
            kv.append((BROTLI_PARAM_NO_DICTIONARY, 1))
        if self.q9_5:
            kv.append((BROTLI_PARAM_Q9_5, 1))
        # framing parameters are forwarded, never dropped: the C ABI refuses the ones this path cannot produce
        for key, on in ((BROTLI_PARAM_CATABLE, self.catable), (BROTLI_PARAM_APPENDABLE, self.appendable),
                        (BROTLI_PARAM_MAGIC_NUMBER, self.magic_number), (BROTLI_PARAM_BYTE_ALIGN, self.byte_align),
                        (BROTLI_PARAM_BARE_STREAM, self.bare_stream)):
            if on:
                kv.append((key, 1))
        return kv


def _capi():
    L = lib()
    if not getattr(L, "_capi_ready", False):
        vp, sz = ctypes.c_void_p, ctypes.c_size_t
        L.BrotliEncoderCreateInstance.restype = vp
        L.BrotliEncoderCreateInstance.argtypes = [vp, vp, vp]
        L.BrotliEncoderDestroyInstance.argtypes = [vp]
        L.BrotliEncoderSetParameter.argtypes = [vp, ctypes.c_int, ctypes.c_uint32]
        L.BrotliEncoderSetParameter.restype = ctypes.c_int
        L.BrotliEncoderCompressStream.argtypes = [vp, ctypes.c_int, ctypes.POINTER(sz), ctypes.POINTER(vp), ctypes.POINTER(sz),
                                                  ctypes.POINTER(vp), ctypes.POINTER(sz)]
        L.BrotliEncoderCompressStream.restype = ctypes.c_int
        L.BrotliEncoderIsFinished.argtypes = [vp]
        L.BrotliEncoderHasMoreOutput.argtypes = [vp]
        L.BrotliEncoderTakeOutput.argtypes = [vp, ctypes.POINTER(sz)]
        L.BrotliEncoderTakeOutput.restype = vp
        L.BrotliEncoderMaxCompressedSize.argtypes = [sz]
        L.BrotliEncoderMaxCompressedSize.restype = sz
        L.BrotliEncoderMaxCompressedSizeMulti.argtypes = [sz, sz]
        L.BrotliEncoderMaxCompressedSizeMulti.restype = sz
        L.BrotliEncoderCompress.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, sz, vp, ctypes.POINTER(sz), vp]
        L.BrotliEncoderCompress.restype = ctypes.c_int
        L.BrotliEncoderCompressMulti.argtypes = [sz, vp, vp, sz, vp, ctypes.POINTER(sz), vp, sz, vp, vp, vp]
        L.BrotliEncoderCompressMulti.restype = ctypes.c_int32
        L.BrotliEncoderVersion.restype = ctypes.c_uint32
        L.BrotliEncoderSetCustomDictionary.argtypes = [vp, sz, vp]
        L.BrotliEncoderSetCustomDictionary.restype = None
        L.BrotliEncoderCompressStreaming.argtypes = [vp, ctypes.c_int, ctypes.POINTER(sz), vp, ctypes.POINTER(sz), vp]
        L.BrotliEncoderCompressStreaming.restype = ctypes.c_int
        L.b200_effective_quality.argtypes = [ctypes.c_int]
        L.b200_effective_quality.restype = ctypes.c_int
        L._capi_ready = True
    return L


def BrotliEncoderMaxCompressedSize(input_size: int) -> int:
    return _capi().BrotliEncoderMaxCompressedSize(input_size)


def BrotliEncoderMaxCompressedSizeMulti(input_size: int, num_threads: int) -> int:
    return _capi().BrotliEncoderMaxCompressedSizeMulti(input_size, num_threads)


def encoder_compress(data: bytes, quality: int = 11, lgwin: int = 22) -> bytes:
    """One-shot ``BrotliEncoderCompress`` (src/ffi/compressor.rs:194)."""
    L = _capi()
    cap = L.BrotliEncoderMaxCompressedSize(len(data)) + 16
    out = ctypes.create_string_buffer(cap)
    osz = ctypes.c_size_t(cap)
    ok = L.BrotliEncoderCompress(quality, lgwin, 0, len(data), _native._inptr(data), ctypes.byref(osz), ctypes.cast(out, ctypes.c_void_p))
    if not ok:
        raise IOError("BrotliEncoderCompress failed (no CUDA device or output too small)")
    return out.raw[:osz.value]


_tensor_encoders = {}  # CUDA ordinal -> the DeviceEncoder compress_tensor uses when it is given none


def _tensor_encoder(t, encoder):
    import torch
    dev = t.device.index if t.device.index is not None else torch.cuda.current_device()
    if encoder is None:
        encoder = _tensor_encoders.get(dev)
        if encoder is None:
            encoder = _tensor_encoders[dev] = DeviceEncoder(dev)
    elif encoder.device != dev:
        raise ValueError("the encoder is on cuda:%d, the tensor on cuda:%d" % (encoder.device, dev))
    return encoder


def _check_tensor(t, what):
    import torch
    if not (t.is_cuda and t.dtype == torch.uint8 and t.is_contiguous()):
        raise ValueError("%s needs a contiguous uint8 CUDA tensor" % what)


def compress_tensor(t, quality: int = 5, lgwin: int = 22, encoder: DeviceEncoder = None, params: BrotliEncoderParams = None,
                    dictionary=None):
    """Compresses a contiguous uint8 CUDA tensor on ``torch.cuda.current_stream()`` without waiting for it.

    Returns ``(out, size)``: a uint8 tensor of capacity bytes whose first ``size`` bytes become the brotli stream, and a
    one-element int64 tensor holding that size, both on ``t``'s device and both written in the order of the current stream (read
    them after it, e.g. ``out[:size.item()]``, which synchronises).  Nothing here synchronises.  Inside ``torch.cuda.graph``
    pass an ``encoder`` on which ``reserve(quality, lgwin, t.numel())`` was called before the capture.

    With ``params`` (``quality`` and ``lgwin`` are then taken from it) the stream is the one ``BrotliEncoderCompressStream`` with
    these parameters and one FINISH produces (``b200_encoder_compress_params_async``), framing included: streams made with
    ``catable=True`` can be spliced on the device by ``concat_tensors``.

    With ``dictionary`` (a uint8 CUDA tensor on ``t``'s device) the stream is the one ``BrotliEncoderCompressStream`` makes after
    ``BrotliEncoderSetCustomDictionary`` with those bytes: a ``DeviceStreamEncoder`` with one FINISH.  Not inside a graph capture.
    """
    import torch
    _check_tensor(t, "compress_tensor")
    encoder = _tensor_encoder(t, encoder)
    if dictionary is not None:
        s = DeviceStreamEncoder(params or BrotliEncoderParams(quality=quality, lgwin=lgwin), dictionary=dictionary, encoder=encoder)
        try:
            s.finish(t)
            out, size, _ = s.output()
        finally:
            s.close()
        return out, size
    n = t.numel()
    cap = lib().b200_max_compressed_size(n) + 64
    out = torch.empty(cap, dtype=torch.uint8, device=t.device)
    size = torch.empty(1, dtype=torch.int64, device=t.device)
    stream = torch.cuda.current_stream(t.device)
    if params is not None:
        encoder.compress_params_async(t.data_ptr(), n, out.data_ptr(), cap, size.data_ptr(), params.as_key_values(), stream.cuda_stream)
    else:
        encoder.compress_async(t.data_ptr(), n, out.data_ptr(), cap, size.data_ptr(), quality, lgwin, stream.cuda_stream)
    return out, size


class DeviceStreamEncoder:
    """``CompressorWriter`` with tensors in and tensors out: one brotli stream fed incrementally from CUDA tensors, its window (and
    a custom dictionary) kept on the GPU (``b200_stream_*``).

    ``write(t)`` is a PROCESS step, ``flush()`` a FLUSH (everything written so far becomes decodable output), ``finish()`` ends the
    stream; ``write`` / ``flush`` / ``finish`` also take a tensor to append first.  The output is appended on the device:
    ``output()`` returns ``(out, size, status)`` device tensors, the stream so far being ``out[:size]`` and ``status`` 0.  The bytes
    equal what ``BrotliEncoderCompressStream`` gives for the same parameters, dictionary and sequence of steps.  Everything is
    enqueued on ``torch.cuda.current_stream()`` and nothing synchronises; steps must be called in the order they are meant to run.
    ``out`` grows as needed (a new tensor, stream-ordered copy), so take ``output()`` again after each step.  Not inside a graph
    capture."""

    def __init__(self, params: BrotliEncoderParams = None, dictionary=None, encoder: DeviceEncoder = None, device=None):
        import torch
        self._params = params or BrotliEncoderParams()
        if dictionary is not None:
            _check_tensor(dictionary, "the dictionary")
            device = dictionary.device
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        probe = torch.empty(0, dtype=torch.uint8, device=dev)
        self._enc = _tensor_encoder(probe, encoder)
        self._L = lib()
        self.device = dev
        n, keys, vals = _native.key_value_arrays(self._params.as_key_values())
        stream = torch.cuda.current_stream(dev)
        dptr, dlen = (dictionary.data_ptr(), dictionary.numel()) if dictionary is not None else (0, 0)
        if dictionary is not None and dlen == 0:  # an empty dictionary still switches the static dictionary off: any non-null
            self._empty = torch.zeros(1, dtype=torch.uint8, device=dev)  # pointer says so, nothing is read
            dptr = self._empty.data_ptr()
        self._h = self._L.b200_stream_create(self._enc._h, n, ctypes.cast(keys, ctypes.c_void_p), ctypes.cast(vals, ctypes.c_void_p),
                                             ctypes.c_void_p(dptr), dlen, ctypes.c_void_p(stream.cuda_stream))
        if not self._h:
            raise ValueError("b200_stream_create refused the parameters or the dictionary")
        self._out = torch.empty(4096, dtype=torch.uint8, device=dev)
        self._size = torch.zeros(1, dtype=torch.int64, device=dev)
        self._status = torch.zeros(1, dtype=torch.int32, device=dev)
        self._bound = 0  # what the steps so far can have appended at most

    def _step(self, op, t=None):
        import torch
        if not self._h:
            raise ValueError("the stream is closed")
        if t is None:
            t = torch.empty(0, dtype=torch.uint8, device=self.device)
        _check_tensor(t, "DeviceStreamEncoder")
        if t.device != self.device:
            raise ValueError("the tensor is on %s, the stream on %s" % (t.device, self.device))
        n = t.numel()
        need = self._bound + self._L.b200_stream_output_bound(self._h, op, n)
        if need > self._out.numel():  # grow the output on the stream: the bytes so far move along
            out = torch.empty(max(need, 2 * self._out.numel()), dtype=torch.uint8, device=self.device)
            if self._bound:
                out[:self._bound].copy_(self._out[:self._bound])
            self._out = out
        stream = torch.cuda.current_stream(self.device)
        if not self._L.b200_stream_compress_async(self._h, op, ctypes.c_void_p(t.data_ptr() if n else 0), n,
                                                  ctypes.c_void_p(self._out.data_ptr()), self._out.numel(),
                                                  ctypes.c_void_p(self._size.data_ptr()), ctypes.c_void_p(self._status.data_ptr()),
                                                  ctypes.c_void_p(stream.cuda_stream)):
            raise RuntimeError("b200_stream_compress_async refused the call (after finish, or inside a graph capture)")
        self._bound = need

    def write(self, t):
        self._step(BROTLI_OPERATION_PROCESS, t)
        return t.numel()

    def flush(self, t=None):
        self._step(BROTLI_OPERATION_FLUSH, t)

    def finish(self, t=None):
        self._step(BROTLI_OPERATION_FINISH, t)

    def output(self):
        return self._out, self._size, self._status

    def close(self):
        """Frees the stream's device buffers, stream-ordered behind its last step (no wait)."""
        if getattr(self, "_h", None):
            self._L.b200_stream_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# BroccoliResult / BroCatliResult (src/concat/mod.rs:3-13)
BROCCOLI_SUCCESS, BROCCOLI_NEEDS_MORE_INPUT, BROCCOLI_NEEDS_MORE_OUTPUT = 0, 1, 2
BROCCOLI_NOT_CRAFTED_FOR_APPEND, BROCCOLI_INVALID_WINDOW_SIZE = 124, 125
BROCCOLI_WINDOW_SIZE_LARGER_THAN_PREVIOUS_FILE, BROCCOLI_NOT_CRAFTED_FOR_CONCATENATION = 126, 127


class BroccoliState(ctypes.Structure):
    """include/broccoli.h: the whole splice state, plain data."""
    _fields_ = [("unused", ctypes.c_void_p), ("data", ctypes.c_ubyte * 248)]


def _broccoli():
    L = lib()
    if not getattr(L, "_broccoli_ready", False):
        sz, P = ctypes.c_size_t, ctypes.POINTER
        L.BroccoliCreateInstance.restype = BroccoliState
        L.BroccoliCreateInstance.argtypes = []
        L.BroccoliCreateInstanceWithWindowSize.restype = BroccoliState
        L.BroccoliCreateInstanceWithWindowSize.argtypes = [ctypes.c_uint8]
        L.BroccoliNewBrotliFile.argtypes = [P(BroccoliState)]
        L.BroccoliNewBrotliFile.restype = None
        L.BroccoliConcatStreaming.argtypes = [P(BroccoliState), P(sz), ctypes.c_void_p, P(sz), ctypes.c_void_p]
        L.BroccoliConcatStreaming.restype = ctypes.c_int
        L.BroccoliConcatFinished.argtypes = [P(BroccoliState), P(sz), ctypes.c_void_p]
        L.BroccoliConcatFinished.restype = ctypes.c_int
        L.b200_concat_workspace_size.argtypes = [ctypes.c_uint32]
        L.b200_concat_workspace_size.restype = sz
        L.b200_concat_async.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int, ctypes.c_void_p, sz,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, sz, ctypes.c_void_p]
        L.b200_concat_async.restype = ctypes.c_int
        L._broccoli_ready = True
    return L


class BroCatli:
    """The reference's stream stitcher (src/concat/mod.rs ``BroCatli``) over the Broccoli C ABI (include/broccoli.h).

    ``new_brotli_file()`` starts the next stream; ``stream(data, out_cap)`` feeds it and ``finish(out_cap)`` ends the spliced
    stream.  Both return ``(result, consumed, output)`` / ``(result, output)`` with at most ``out_cap`` output bytes, as one call of
    the reference does over buffers of those sizes.  Host code: no CUDA device is needed."""

    def __init__(self, _state=None):
        self._L = _broccoli()
        self._s = self._L.BroccoliCreateInstance() if _state is None else _state

    @classmethod
    def new_with_window_size(cls, window_size: int):
        """An instance that starts as an empty stream of that window; a size the reference refuses gives a default instance."""
        return cls(_broccoli().BroccoliCreateInstanceWithWindowSize(window_size))

    def new_brotli_file(self):
        self._L.BroccoliNewBrotliFile(ctypes.byref(self._s))

    def stream(self, data: bytes, out_cap: int):
        data = bytes(data)
        avail_in, avail_out = ctypes.c_size_t(len(data)), ctypes.c_size_t(out_cap)
        obuf = ctypes.create_string_buffer(max(1, out_cap))
        r = self._L.BroccoliConcatStreaming(ctypes.byref(self._s), ctypes.byref(avail_in), _native._inptr(data),
                                            ctypes.byref(avail_out), ctypes.cast(obuf, ctypes.c_void_p))
        return r, len(data) - avail_in.value, obuf.raw[:out_cap - avail_out.value]

    def finish(self, out_cap: int):
        avail_out = ctypes.c_size_t(out_cap)
        obuf = ctypes.create_string_buffer(max(1, out_cap))
        r = self._L.BroccoliConcatFinished(ctypes.byref(self._s), ctypes.byref(avail_out), ctypes.cast(obuf, ctypes.c_void_p))
        return r, obuf.raw[:out_cap - avail_out.value]

    def state_bytes(self) -> bytes:
        return bytes(self._s.data)


def concat_tensors(parts, window_size: int = 0, pointers=None, workspace=None):
    """Splices catable streams that live on the GPU into one brotli stream, on ``torch.cuda.current_stream()`` without waiting.

    ``parts`` is a list of ``(out, size)`` pairs as ``compress_tensor`` returns them (``size`` a one-element int64 device tensor,
    read on the device).  Returns ``(out, size, result)`` device tensors: the spliced stream is ``out[:size]`` and ``result`` holds
    (BroccoliResult, stream index), both as the host sequence ``BroCatli`` / new_brotli_file + stream per part / finish gives them
    (``b200_concat_async``).  On failure ``size`` is 0 and ``result`` names the first failing part.

    Inside ``torch.cuda.graph``: the table of stream pointers and the workspace must exist before the capture (building the table
    copies it from host memory).  Pass ``pointers=concat_pointer_table(parts)`` and
    ``workspace=torch.empty(concat_workspace_size(len(parts)), dtype=torch.uint8, device=...)`` made outside the capture."""
    import torch
    if not parts:
        raise ValueError("concat_tensors needs at least one part")
    dev = parts[0][0].device
    for o, s in parts:
        if not (o.is_cuda and o.dtype == torch.uint8 and o.device == dev and s.is_cuda and s.dtype == torch.int64 and s.numel() == 1):
            raise ValueError("parts must be (uint8 CUDA tensor, one-element int64 CUDA tensor) pairs on one device")
    L = _broccoli()
    n = len(parts)
    if pointers is None:
        pointers = concat_pointer_table(parts)
    if workspace is None:
        workspace = torch.empty(L.b200_concat_workspace_size(n), dtype=torch.uint8, device=dev)
    sizes = torch.cat([s.reshape(1) for _, s in parts])
    cap = sum(o.numel() for o, _ in parts) + 3  # a part's size is at most its capacity; the splice adds at most 3 bytes
    out = torch.empty(cap, dtype=torch.uint8, device=dev)
    size = torch.empty(1, dtype=torch.int64, device=dev)
    result = torch.empty(2, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream(dev)
    if not L.b200_concat_async(pointers.data_ptr(), sizes.data_ptr(), n, int(window_size), out.data_ptr(), cap, size.data_ptr(),
                               result.data_ptr(), workspace.data_ptr(), workspace.numel(), stream.cuda_stream):
        raise RuntimeError("b200_concat_async refused the call")
    return out, size, result


def concat_pointer_table(parts):
    """The device table of stream pointers ``concat_tensors`` reads.  It is copied from pinned host memory on the current stream
    without waiting; being a copy from host memory, it must be built outside a graph capture."""
    import torch
    host = torch.tensor([o.data_ptr() for o, _ in parts], dtype=torch.int64).pin_memory()
    return host.to(parts[0][0].device, non_blocking=True)


def concat_workspace_size(count: int) -> int:
    return _broccoli().b200_concat_workspace_size(count)


class _Stream:
    """BrotliEncoderState driven through BrotliEncoderCompressStream, as writer.rs / reader.rs do."""

    def __init__(self, params: BrotliEncoderParams):
        self.L = _capi()
        self.h = self.L.BrotliEncoderCreateInstance(None, None, None)
        if not self.h:
            raise IOError("BrotliEncoderCreateInstance failed: no usable CUDA device")
        for k, v in params.as_key_values():
            if not self.L.BrotliEncoderSetParameter(self.h, k, int(v)):
                self.close()
                raise ValueError("BrotliEncoderSetParameter(%d, %d) refused: not produced by this path" % (k, int(v)))

    def step(self, data: bytes, op: int) -> bytes:
        out = bytearray()
        avail_in = ctypes.c_size_t(len(data))
        inbuf = ctypes.create_string_buffer(data, len(data)) if data else None
        next_in = ctypes.c_void_p(ctypes.addressof(inbuf) if data else 0)
        obuf = ctypes.create_string_buffer(1 << 16)
        while True:
            avail_out = ctypes.c_size_t(len(obuf))
            next_out = ctypes.c_void_p(ctypes.addressof(obuf))
            total = ctypes.c_size_t(0)
            ok = self.L.BrotliEncoderCompressStream(self.h, op, ctypes.byref(avail_in), ctypes.byref(next_in), ctypes.byref(avail_out),
                                                    ctypes.byref(next_out), ctypes.byref(total))
            if not ok:
                raise IOError("BrotliEncoderCompressStream failed")  # io::ErrorKind::InvalidData in writer.rs:43-44
            out += obuf.raw[: len(obuf) - avail_out.value]
            if avail_in.value == 0 and not self.L.BrotliEncoderHasMoreOutput(self.h):
                break
        return bytes(out)

    def close(self):
        if self.h:
            self.L.BrotliEncoderDestroyInstance(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CompressorWriter:
    """``CompressorWriter::new(w, buffer_size, q, lgwin)`` / ``with_params`` (src/enc/writer.rs:83-118)."""

    def __init__(self, w, buffer_size: int = 4096, q: int = 11, lgwin: int = 22, params: BrotliEncoderParams = None):
        self._w = w
        self._params = params or BrotliEncoderParams(quality=q, lgwin=lgwin)
        self._s = _Stream(self._params)
        self._closed = False
        self.buffer_size = buffer_size

    @classmethod
    def with_params(cls, w, buffer_size, params):
        return cls(w, buffer_size, params=params)

    def write(self, buf: bytes) -> int:
        out = self._s.step(bytes(buf), BROTLI_OPERATION_PROCESS)
        if out:
            self._w.write(out)
        return len(buf)

    def flush(self):
        out = self._s.step(b"", BROTLI_OPERATION_FLUSH)
        if out:
            self._w.write(out)
        if hasattr(self._w, "flush"):
            self._w.flush()

    def close(self):
        """Finishes the stream (the reference does this on Drop, writer.rs:253-265)."""
        if not self._closed:
            out = self._s.step(b"", BROTLI_OPERATION_FINISH)
            if out:
                self._w.write(out)
            self._s.close()
            self._closed = True

    def into_inner(self):
        self.close()
        return self._w

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class CompressorReader:
    """``CompressorReader::new(r, buffer_size, q, lgwin)`` (src/enc/reader.rs:74-103): reads raw, yields compressed."""

    def __init__(self, r, buffer_size: int = 4096, q: int = 11, lgwin: int = 22, params: BrotliEncoderParams = None):
        self._r = r
        self._params = params or BrotliEncoderParams(quality=q, lgwin=lgwin)
        self._s = _Stream(self._params)
        self._buf = bytearray()
        self._eof = False
        self.buffer_size = max(1, buffer_size)

    def read(self, n: int = -1) -> bytes:
        while not self._eof and (n < 0 or len(self._buf) < n):
            chunk = self._r.read(self.buffer_size)
            if chunk:
                self._buf += self._s.step(chunk, BROTLI_OPERATION_PROCESS)
            else:
                self._buf += self._s.step(b"", BROTLI_OPERATION_FINISH)
                self._s.close()
                self._eof = True
        if n < 0:
            out, self._buf = bytes(self._buf), bytearray()
        else:
            out, self._buf = bytes(self._buf[:n]), self._buf[n:]
        return out

    def into_inner(self):
        return self._r


def BrotliCompress(r, w, params: BrotliEncoderParams) -> int:
    """``BrotliCompress(r, w, &params) -> io::Result<usize>`` (src/enc/mod.rs:142): returns bytes written."""
    cw = CompressorWriter.with_params(_CountingWriter(w), 4096, params)
    while True:
        chunk = r.read(1 << 20)
        if not chunk:
            break
        cw.write(chunk)
    cw.close()
    return cw._w.count


class _CountingWriter:
    def __init__(self, w):
        self.w = w
        self.count = 0

    def write(self, b):
        self.count += len(b)
        return self.w.write(b)


def compress_multi(params: BrotliEncoderParams, input_bytes: bytes, num_threads: int = 1) -> bytes:
    """``compress_multi`` (src/enc/mod.rs:95-133; CompressMulti src/enc/threading/mod.rs:413).

    The input is split into ``num_threads`` (<= 16) equal ranges (threading/mod.rs:333); range i > 0 sees the previous
    2^lgwin bytes as its LZ77 window.  Ranges are placed round-robin on the visible GPUs and their byte-aligned
    outputs are concatenated.  Raises BrotliEncoderThreadError subclasses on failure.
    """
    L = _capi()
    if num_threads < 1 or num_threads > MAX_THREADS:
        raise BrotliEncoderThreadError("num_threads must be in 1..=%d" % MAX_THREADS)
    kv = params.as_key_values()
    keys = (ctypes.c_int * len(kv))(*[k for k, _ in kv])
    vals = (ctypes.c_uint32 * len(kv))(*[int(v) for _, v in kv])
    cap = L.BrotliEncoderMaxCompressedSizeMulti(len(input_bytes), num_threads) + 64
    out = ctypes.create_string_buffer(cap)
    osz = ctypes.c_size_t(cap)
    ok = L.BrotliEncoderCompressMulti(len(kv), ctypes.cast(keys, ctypes.c_void_p), ctypes.cast(vals, ctypes.c_void_p), len(input_bytes),
                                      _native._inptr(input_bytes), ctypes.byref(osz), ctypes.cast(out, ctypes.c_void_p), num_threads,
                                      None, None, None)
    if not ok:
        raise OtherThreadPanic("BrotliEncoderCompressMulti failed")
    return out.raw[:osz.value]

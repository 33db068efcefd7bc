"""ctypes binding of libbrotli_b200.so (built in-tree by build.py / __graft_entry__.build()).

There is no fallback: if the shared library is missing or CUDA is unavailable, every call raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200_LIB") or os.path.join(_HERE, "libbrotli_b200.so")  # B200_LIB: A/B builds (tools/)

NUM_STAGES = 7
STAGE_NAMES = ("sort", "match", "parse", "finalize", "split", "header", "emit")
OPT_CTX_MODEL, OPT_TIMING, OPT_LANES, OPT_DICT = 6, 7, 8, 9
OPT_HQ_SPLIT, OPT_HQ_UNIT, OPT_ONDEMAND, OPT_HQ_LEVELS = 12, 13, 15, 16
OPT_Q9_5 = 17

_lib = None


class StreamCounters(ctypes.Structure):
    """B200StreamCounters (include/brotli_b200.h): the counters of one compression stream."""
    _fields_ = [("base", ctypes.c_uint64), ("flushed", ctypes.c_uint64), ("end", ctypes.c_uint64), ("dict_len", ctypes.c_uint64),
                ("header_written", ctypes.c_int32), ("finished", ctypes.c_int32)]


class StreamEmit(ctypes.Structure):
    """B200StreamEmit (include/brotli_b200.h): one emit of a stream step."""
    _fields_ = [("start", ctypes.c_uint64), ("upto", ctypes.c_uint64), ("base", ctypes.c_uint64), ("base_after", ctypes.c_uint64),
                ("size_hint", ctypes.c_uint64), ("first", ctypes.c_int32), ("last", ctypes.c_int32), ("byte", ctypes.c_int32)]


class FramedCall(ctypes.Structure):
    """B200FramedCall (include/brotli_b200.h): one device call of the framing rule."""
    _fields_ = [("rebase", ctypes.c_uint64), ("start", ctypes.c_uint64), ("end", ctypes.c_uint64), ("first", ctypes.c_int32),
                ("last", ctypes.c_int32), ("byte_align", ctypes.c_int32)]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libbrotli_b200.so is not built (run `python __graft_entry__.py build`); "
                               "there is no CPU fallback for the compression path")
        L = ctypes.CDLL(LIB_PATH)
        vp, sz = ctypes.c_void_p, ctypes.c_size_t
        L.b200_device_count.restype = ctypes.c_int
        L.b200_encoder_create.restype = vp
        L.b200_encoder_create.argtypes = [ctypes.c_int]
        L.b200_encoder_destroy.argtypes = [vp]
        L.b200_encoder_set_option.argtypes = [vp, ctypes.c_int, ctypes.c_uint32]
        L.b200_encoder_set_option.restype = ctypes.c_int
        L.b200_max_compressed_size.argtypes = [sz]
        L.b200_max_compressed_size.restype = sz
        L.b200_encoder_compress.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, sz, vp, sz, ctypes.POINTER(sz), ctypes.c_int]
        L.b200_encoder_compress.restype = ctypes.c_int
        L.b200_encoder_compress_range.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_uint64, vp, sz, sz, sz, ctypes.c_int,
                                                  ctypes.c_int, ctypes.c_int, vp, sz, ctypes.POINTER(sz), ctypes.c_int]
        L.b200_encoder_compress_range.restype = ctypes.c_int
        L.b200_encoder_reserve.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_uint64, sz, sz]
        L.b200_encoder_reserve.restype = ctypes.c_int
        L.b200_encoder_compress_range_async.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_uint64, vp, sz, sz, sz, ctypes.c_int,
                                                        ctypes.c_int, ctypes.c_int, vp, sz, vp, vp]
        L.b200_encoder_compress_range_async.restype = ctypes.c_int
        L.b200_encoder_compress_params_async.argtypes = [vp, sz, vp, vp, vp, sz, vp, sz, vp, vp]
        L.b200_encoder_compress_params_async.restype = ctypes.c_int
        L.b200_encoder_last_timings.argtypes = [vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32)]
        L.b200_stage_match.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_uint64, vp, sz, sz, sz, ctypes.c_int, vp]
        L.b200_stage_match.restype = ctypes.c_int
        L.b200_stage_match_slabs.argtypes = [vp, vp, vp, ctypes.c_uint32]
        L.b200_stage_match_slabs.restype = ctypes.c_int
        L.b200_stage_match_tiles.argtypes = [vp, vp, vp, ctypes.c_uint32]
        L.b200_stage_match_tiles.restype = ctypes.c_int
        L.b200_stage_hq.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, sz, vp, vp, vp, vp]
        L.b200_stage_hq.restype = ctypes.c_int
        L.b200_hq_unit.argtypes = [vp, ctypes.c_int, ctypes.c_uint64]
        L.b200_hq_unit.restype = ctypes.c_uint32
        L.b200_stage_sort.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, sz, ctypes.c_int, vp]
        L.b200_stage_sort.restype = ctypes.c_int
        L.b200_stream_create.argtypes = [vp, sz, vp, vp, vp, sz, vp]
        L.b200_stream_create.restype = vp
        L.b200_stream_compress_async.argtypes = [vp, ctypes.c_int, vp, sz, vp, sz, vp, vp, vp]
        L.b200_stream_compress_async.restype = ctypes.c_int
        L.b200_stream_output_bound.argtypes = [vp, ctypes.c_int, sz]
        L.b200_stream_output_bound.restype = sz
        L.b200_stream_destroy.argtypes = [vp]
        L.b200_stream_destroy.restype = None
        P = ctypes.POINTER
        L.b200_stage_stream_start.argtypes = [sz, vp, vp, ctypes.c_uint64, P(StreamCounters), P(ctypes.c_uint64)]
        L.b200_stage_stream_start.restype = ctypes.c_int
        L.b200_stage_stream_plan.argtypes = [sz, vp, vp, P(StreamCounters), ctypes.c_int, ctypes.c_uint64, P(StreamEmit), sz, P(sz),
                                             P(StreamCounters)]
        L.b200_stage_stream_plan.restype = ctypes.c_int
        L.b200_stage_framed_plan.argtypes = [sz, vp, vp, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp,
                                             P(ctypes.c_int32), P(FramedCall), sz, P(sz), P(ctypes.c_int32)]
        L.b200_stage_framed_plan.restype = ctypes.c_int
        _lib = L
    return _lib


def _inptr(data):
    return ctypes.cast(ctypes.c_char_p(data), ctypes.c_void_p) if len(data) else ctypes.c_void_p(0)


class DeviceEncoder:
    """One GPU, one stream, one reusable workspace (wraps B200Encoder*)."""

    def __init__(self, device: int = 0):
        self._L = lib()
        self._h = self._L.b200_encoder_create(device)
        if not self._h:
            raise RuntimeError("b200_encoder_create(%d) failed: no usable CUDA device" % device)
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            self._L.b200_encoder_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, opt, value):
        if not self._L.b200_encoder_set_option(self._h, opt, int(value)):
            raise ValueError("bad option")

    def compress(self, data: bytes, quality: int = 5, lgwin: int = 22) -> bytes:
        n = len(data)
        cap = self._L.b200_max_compressed_size(n)
        out = ctypes.create_string_buffer(cap)
        osz = ctypes.c_size_t(0)
        ok = self._L.b200_encoder_compress(self._h, quality, lgwin, _inptr(data), n, ctypes.cast(out, ctypes.c_void_p), cap,
                                           ctypes.byref(osz), 0)
        if not ok:
            raise RuntimeError("b200_encoder_compress failed")
        return out.raw[:osz.value]

    def compress_range(self, data: bytes, start: int, length: int, quality: int, lgwin: int, first: bool, last: bool,
                       byte_align: bool, size_hint: int = 0) -> bytes:
        cap = self._L.b200_max_compressed_size(length)
        out = ctypes.create_string_buffer(cap)
        osz = ctypes.c_size_t(0)
        ok = self._L.b200_encoder_compress_range(self._h, quality, lgwin, size_hint, _inptr(data), len(data), start, length,
                                                 int(first), int(last), int(byte_align), ctypes.cast(out, ctypes.c_void_p), cap,
                                                 ctypes.byref(osz), 0)
        if not ok:
            raise RuntimeError("b200_encoder_compress_range failed")
        return out.raw[:osz.value]

    def compress_device(self, d_in_ptr: int, n: int, d_out_ptr: int, out_cap: int, quality: int = 5, lgwin: int = 22) -> int:
        """Device-resident input/output (raw CUDA pointers, e.g. torch tensor .data_ptr()); returns compressed size."""
        osz = ctypes.c_size_t(0)
        ok = self._L.b200_encoder_compress(self._h, quality, lgwin, ctypes.c_void_p(d_in_ptr), n, ctypes.c_void_p(d_out_ptr),
                                           out_cap, ctypes.byref(osz), 1)
        if not ok:
            raise RuntimeError("b200_encoder_compress (device io) failed")
        return osz.value

    def reserve(self, quality: int, lgwin: int, n: int, range_len=None, size_hint: int = 0):
        """Allocates everything an async call of these or smaller arguments uses (b200_encoder_reserve): such calls then never
        allocate, which a call inside a CUDA graph capture requires."""
        if not self._L.b200_encoder_reserve(self._h, quality, lgwin, size_hint, n, n if range_len is None else range_len):
            raise RuntimeError("b200_encoder_reserve failed")

    def compress_async(self, d_in_ptr: int, n: int, d_out_ptr: int, out_cap: int, d_size_ptr: int, quality: int, lgwin: int,
                       stream_ptr: int, range_start: int = 0, range_len=None, first: bool = True, last: bool = True,
                       byte_align: bool = False, size_hint: int = 0):
        """Enqueues the compression of [range_start, range_start + range_len) of the n device bytes at d_in_ptr on the CUDA stream
        stream_ptr (e.g. torch.cuda.current_stream().cuda_stream) and returns without waiting: out[0, size) and the uint64 size at
        d_size_ptr are written when the stream gets there (b200_encoder_compress_range_async).  Raises if the call is refused;
        nothing is enqueued then."""
        if range_len is None:
            range_len = n - range_start
        ok = self._L.b200_encoder_compress_range_async(self._h, quality, lgwin, size_hint, ctypes.c_void_p(d_in_ptr), n, range_start,
                                                        range_len, int(first), int(last), int(byte_align),
                                                        ctypes.c_void_p(d_out_ptr), out_cap, ctypes.c_void_p(d_size_ptr),
                                                        ctypes.c_void_p(stream_ptr))
        if not ok:
            raise RuntimeError("b200_encoder_compress_range_async refused the call")

    def compress_params_async(self, d_in_ptr: int, n: int, d_out_ptr: int, out_cap: int, d_size_ptr: int, key_values, stream_ptr: int):
        """One complete stream of the n device bytes at d_in_ptr with BrotliEncoderCompressMulti-style (key, value) parameters,
        enqueued on stream_ptr without waiting (b200_encoder_compress_params_async).  Raises if the call is refused."""
        kv = list(key_values)
        keys = (ctypes.c_int * max(1, len(kv)))(*[int(k) for k, _ in kv])
        vals = (ctypes.c_uint32 * max(1, len(kv)))(*[int(v) for _, v in kv])
        ok = self._L.b200_encoder_compress_params_async(self._h, len(kv), ctypes.cast(keys, ctypes.c_void_p), ctypes.cast(vals, ctypes.c_void_p),
                                                         ctypes.c_void_p(d_in_ptr), n, ctypes.c_void_p(d_out_ptr), out_cap,
                                                         ctypes.c_void_p(d_size_ptr), ctypes.c_void_p(stream_ptr))
        if not ok:
            raise RuntimeError("b200_encoder_compress_params_async refused the call")

    def timings(self):
        ms = (ctypes.c_float * NUM_STAGES)()
        launches = ctypes.c_uint32(0)
        self._L.b200_encoder_last_timings(self._h, ms, ctypes.byref(launches))
        return dict(zip(STAGE_NAMES, [float(x) for x in ms])), int(launches.value)

    def stage_match(self, data: bytes, quality: int, lgwin: int, size_hint: int = 0, start: int = 0, length=None,
                    on_demand: bool = False):
        """best[] of the quality 5..9 match stage for data[start:start + length] (length <= 24 MiB; the bytes in front of start
        are its window), as the up-front kernels compute it, or (on_demand) as the on-demand search computes it at every
        position -- which needs bucket depth >= 64 and a range that fits one sort batch.  size_hint 0 = len(data)."""
        import numpy as np
        if length is None:
            length = len(data) - start
        out = np.zeros(length, dtype=np.uint32)
        ok = self._L.b200_stage_match(self._h, quality, lgwin, size_hint, _inptr(data), len(data), start, length, int(on_demand),
                                      out.ctypes.data)
        if not ok:
            raise RuntimeError("b200_stage_match failed")
        return out

    def stage_match_slabs(self):
        """After stage_match (up-front kernels): (cursors, sizes) of the range's last sort batch, uint32 arrays with one entry
        per best[] slab -- the records the match kernel claimed in each slab and the records each slab must receive."""
        import numpy as np
        cursors = np.zeros(64, dtype=np.uint32)
        sizes = np.zeros(64, dtype=np.uint32)
        ns = self._L.b200_stage_match_slabs(self._h, cursors.ctypes.data, sizes.ctypes.data, 64)
        if ns <= 0 or ns > 64:
            raise RuntimeError("b200_stage_match_slabs failed")
        return cursors[:ns], sizes[:ns]

    def stage_match_tiles(self):
        """The same as stage_match_slabs for the tiles of 2^13 positions that the placement fills after the slabs: (cursors,
        sizes) with one entry per tile of the last sort batch."""
        import numpy as np
        nt = self._L.b200_stage_match_tiles(self._h, None, None, 0)
        if nt <= 0:
            raise RuntimeError("b200_stage_match_tiles failed")
        cursors = np.zeros(nt, dtype=np.uint32)
        sizes = np.zeros(nt, dtype=np.uint32)
        if self._L.b200_stage_match_tiles(self._h, cursors.ctypes.data, sizes.ctypes.data, nt) != nt:
            raise RuntimeError("b200_stage_match_tiles failed")
        return cursors, sizes

    def stage_hq(self, data: bytes, quality: int, lgwin: int):
        """Quality 10 / 11 stage results of one chunk: (hqn[n] u8, hqm[n][16][2] u32 (dist, lc), units[3][nu] u32 (ncmd, tail,
        ncopy), raw[nu][unit/2+1][3] u32, unit).  hqm entries past hqn[p] are left over from earlier calls."""
        import numpy as np
        n = len(data)
        unit = int(self._L.b200_hq_unit(self._h, quality, n))
        if n == 0 or unit == 0:
            raise ValueError("stage_hq needs quality >= 10 and a non-empty input")
        nu = (n + unit - 1) // unit
        hqn = np.zeros(n, dtype=np.uint8)
        hqm = np.zeros((n, 16, 2), dtype=np.uint32)
        units = np.zeros((3, nu), dtype=np.uint32)
        raw = np.zeros((nu, unit // 2 + 1, 3), dtype=np.uint32)
        ok = self._L.b200_stage_hq(self._h, quality, lgwin, _inptr(data), n, hqn.ctypes.data, hqm.ctypes.data, units.ctypes.data,
                                   raw.ctypes.data)
        if not ok:
            raise RuntimeError("b200_stage_hq failed")
        return hqn, hqm, units, raw, unit

    def stage_sort(self, data: bytes, quality: int, lgwin: int, level=None):
        """Positions 0..n-1 of one sort batch over `data` (n <= 2^25) in the order of the sort stage: stable by the bucket key
        the configuration (quality, lgwin, size hint n) uses, or by the key of long-prefix level 0..2 of quality 10 / 11."""
        import numpy as np
        out = np.zeros(len(data), dtype=np.uint32)
        ok = self._L.b200_stage_sort(self._h, quality, lgwin, _inptr(data), len(data), -1 if level is None else int(level),
                                     out.ctypes.data)
        if not ok:
            raise RuntimeError("b200_stage_sort failed")
        return out


def key_value_arrays(key_values):
    """(count, keys, values) ctypes arrays of (BrotliEncoderParameter, value) pairs, as the C ABI takes them."""
    kv = list(key_values)
    keys = (ctypes.c_int * max(1, len(kv)))(*[int(k) for k, _ in kv])
    vals = (ctypes.c_uint32 * max(1, len(kv)))(*[int(v) for _, v in kv])
    return len(kv), keys, vals


def stream_start(key_values, dict_size: int):
    """b200_stage_stream_start: (counters, index of the first dictionary byte kept) of a new stream."""
    n, keys, vals = key_value_arrays(key_values)
    c, frm = StreamCounters(), ctypes.c_uint64(0)
    if not lib().b200_stage_stream_start(n, ctypes.cast(keys, ctypes.c_void_p), ctypes.cast(vals, ctypes.c_void_p), dict_size,
                                         ctypes.byref(c), ctypes.byref(frm)):
        raise ValueError("b200_stage_stream_start refused the parameters")
    return c, frm.value


def stream_plan(key_values, counters: StreamCounters, op: int, n: int, max_emits: int = 64):
    """b200_stage_stream_plan: (emits, counters after them) of one stream step, or None when the step is refused."""
    k, keys, vals = key_value_arrays(key_values)
    emits = (StreamEmit * max_emits)()
    count, nxt = ctypes.c_size_t(0), StreamCounters()
    if not lib().b200_stage_stream_plan(k, ctypes.cast(keys, ctypes.c_void_p), ctypes.cast(vals, ctypes.c_void_p), ctypes.byref(counters),
                                        op, n, emits, max_emits, ctypes.byref(count), ctypes.byref(nxt)):
        return None
    return list(emits[:count.value]), nxt


def framed_plan(key_values, a: int, b: int, first: bool, last: bool, align_end: bool, max_calls: int = 16):
    """b200_stage_framed_plan: (prologue, calls, trailer) of input bytes [a, b), or None when the plan is refused.  prologue is
    None or (bytes, data_off, n2, complete); calls are (rebase, start, end, first, last, byte_align) tuples; trailer is -1 or
    the byte behind the last call."""
    k, keys, vals = key_value_arrays(key_values)
    pro, info = (ctypes.c_uint8 * 32)(), (ctypes.c_int32 * 4)()
    calls, count, trailer = (FramedCall * max_calls)(), ctypes.c_size_t(0), ctypes.c_int32(0)
    if not lib().b200_stage_framed_plan(k, ctypes.cast(keys, ctypes.c_void_p), ctypes.cast(vals, ctypes.c_void_p), a, b, int(first),
                                        int(last), int(align_end), pro, info, calls, max_calls, ctypes.byref(count),
                                        ctypes.byref(trailer)):
        return None
    prologue = None if info[0] < 0 else (bytes(pro[:info[0]]), info[1], info[2], bool(info[3]))
    return prologue, [(c.rebase, c.start, c.end, bool(c.first), bool(c.last), bool(c.byte_align)) for c in calls[:count.value]], \
        trailer.value

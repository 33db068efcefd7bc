"""ctypes binding of tools/libgpu_model.so (CPU model of the GPU pipeline; development/test infrastructure)."""
import ctypes, os, subprocess
_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)

class EncParams(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("quality", "lgwin", "hash_type", "key_bits", "hash_len", "depth", "n_last")] + \
               [(n, ctypes.c_uint32) for n in ("lcap", "unit", "mb_units", "max_backward", "n", "abs_base", "size_hint")] + \
               [(n, ctypes.c_int) for n in ("ctx_model", "use_dict", "hq_split", "hq_levels", "zopfli", "hq_meta")]

class ModelStats(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint64) for n in ("num_metablocks", "num_raw_metablocks", "num_commands", "num_literals", "header_bits", "body_bits")] + \
               [(n, ctypes.c_uint32) for n in ("lit_types_total", "cmd_types_total", "dist_types_total")] + [("ctx_ids", ctypes.c_uint32 * 4)]

def build_model(force=False):
    so = os.path.join(_HERE, "libgpu_model.so")
    srcs = [os.path.join(_HERE, "gpu_model.cpp")] + [os.path.join(_ROOT, "rust-brotli_b200", "csrc", f) for f in
            ("bro_common.cuh", "bro_huffman.cuh", "bro_meta.cuh", "bro_parse.cuh", "bro_split.cuh", "bro_dict.cuh", "bro_finalize.cuh", "bro_hq.cuh", "bro_bsplit.cuh")]
    inc = os.path.join(_ROOT, "rust-brotli_b200", "csrc", "bro_dict_data.inc")
    if not os.path.exists(inc):  # generated file (static dictionary from the system libbrotlicommon + our hash table)
        subprocess.check_call([os.sys.executable, os.path.join(_ROOT, "rust-brotli_b200", "gen_dict.py")])
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-fwrapv", "-std=c++17", "-shared", "-fPIC", "-w", "-I",
                               os.path.join(_ROOT, "rust-brotli_b200", "csrc"), srcs[0], "-o", so])
    return so

class Model:
    def __init__(self):
        self.lib = ctypes.CDLL(build_model())
        self.lib.gpu_model_compress.restype = ctypes.c_size_t
        self.lib.gpu_model_compress.argtypes = [ctypes.POINTER(EncParams), ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t,
                                                ctypes.POINTER(ModelStats), ctypes.c_void_p]
        self.lib.gpu_model_default_params.argtypes = [ctypes.POINTER(EncParams), ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32,
                                                      ctypes.c_int]
        self.lib.gpu_model_debug_hq.argtypes = [ctypes.c_void_p] * 4
    def params(self, q, lgwin, n, size_hint=0, q9_5=False, **kw):
        """Default parameters of a configuration (q9_5: BROTLI_PARAM_Q9_5), then the fields of kw."""
        p = EncParams()
        self.lib.gpu_model_default_params(ctypes.byref(p), q, lgwin, n, size_hint, int(bool(q9_5)))
        for k, v in kw.items(): setattr(p, k, v)
        return p
    def compress_range(self, data, start, length, q, lgwin, first, last, byte_align, size_hint=0, best_out=None, **kw):
        p = self.params(q, lgwin, len(data), size_hint or len(data), **kw)
        cap = length + (length >> 2) + 65536
        out = ctypes.create_string_buffer(cap)
        st = ModelStats()
        self.lib.gpu_model_compress_range.restype = ctypes.c_size_t
        self.lib.gpu_model_compress_range.argtypes = [ctypes.POINTER(EncParams), ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32,
                                                      ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_size_t,
                                                      ctypes.POINTER(ModelStats), ctypes.c_void_p]
        n = self.lib.gpu_model_compress_range(ctypes.byref(p), data, start, length, int(first), int(last), int(byte_align), out, cap,
                                              ctypes.byref(st), best_out)
        return out.raw[:n], st

    def compress(self, data, q, lgwin, size_hint=0, best_out=None, **kw):
        p = self.params(q, lgwin, len(data), size_hint, **kw)
        cap = len(data) + (len(data) >> 2) + 65536
        out = ctypes.create_string_buffer(cap)
        st = ModelStats()
        n = self.lib.gpu_model_compress(ctypes.byref(p), data, out, cap, ctypes.byref(st), best_out)
        if n == 0: raise RuntimeError("model failed")
        return out.raw[:n], st

    def stage_hq(self, data, q, lgwin, **kw):
        """Shortest-path parse (quality 10 / 11 without Q9_5) stage results of a one-chunk input, laid out as DeviceEncoder.stage_hq returns them:
        (hqn, hqm, units, raw, unit)."""
        import numpy as np
        n = len(data)
        if not 0 < n <= 24 << 20 or not self.params(q, lgwin, n, 0, **kw).zopfli:
            raise ValueError("stage_hq covers one chunk (1 .. 24 MiB) at quality >= 10")
        unit = self.params(q, lgwin, n, 0, **kw).unit
        nu = (n + unit - 1) // unit
        hqn = np.zeros(n, dtype=np.uint8)
        hqm = np.zeros((n, 16, 2), dtype=np.uint32)
        units = np.zeros((3, nu), dtype=np.uint32)
        raw = np.zeros((nu, unit // 2 + 1, 3), dtype=np.uint32)
        # the taps are static in the library and every later compression writes through them: always detach
        self.lib.gpu_model_debug_hq(hqn.ctypes.data_as(ctypes.c_void_p), hqm.ctypes.data_as(ctypes.c_void_p),
                                    units.ctypes.data_as(ctypes.c_void_p), raw.ctypes.data_as(ctypes.c_void_p))
        try:
            self.compress(data, q, lgwin, **kw)
        finally:
            self.lib.gpu_model_debug_hq(None, None, None, None)
        return hqn, hqm, units, raw, unit

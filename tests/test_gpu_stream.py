"""GPU: device-resident streams (b200_stream_* / rust_brotli_b200.DeviceStreamEncoder) and compress_tensor(dictionary=...).

Everything a device stream appends must equal, byte for byte, what the host BrotliEncoderCompressStream outputs for the same
parameters, custom dictionary and sequence of (op, bytes) -- across write sizes, qualities, windows and framings, and for a
long stream whose pieces are emitted before FINISH.  Every FLUSH must leave a decodable prefix, the call must be stream-ordered
and return before the stream runs, an output that is too small must fail the stream without writing, and refused calls must
enqueue nothing (a capture stays valid)."""
import ctypes

import pytest

from conftest import golden_bytes
from oracle.harness import sys_decompress, sys_decompress_with_dictionary

pytestmark = pytest.mark.gpu

MiB = 1 << 20
PROCESS, FLUSH, FINISH, EMIT_METADATA = 0, 1, 2, 3


def text(n, seed=7):
    from tools import datagen
    return datagen.enwik_like(n, seed=seed)


def host_steps(kv, steps, dictionary=None):
    """The host BrotliEncoderCompressStream's output after each (op, bytes) step."""
    import rust_brotli_b200 as rb
    L = rb._capi()
    h = L.BrotliEncoderCreateInstance(None, None, None)
    assert h
    try:
        for k, v in kv:
            assert L.BrotliEncoderSetParameter(h, k, int(v))
        if dictionary is not None:
            L.BrotliEncoderSetCustomDictionary(h, len(dictionary), dictionary)
        outs = []
        for op, data in steps:
            cap = len(data) + (len(data) >> 3) + (1 << 16)
            buf = ctypes.create_string_buffer(cap)
            got = bytearray()
            avail_in = ctypes.c_size_t(len(data))
            next_in = ctypes.c_void_p(ctypes.cast(ctypes.c_char_p(data), ctypes.c_void_p).value if data else 0)
            while True:
                avail_out, next_out = ctypes.c_size_t(cap), ctypes.c_void_p(ctypes.addressof(buf))
                assert L.BrotliEncoderCompressStream(h, op, ctypes.byref(avail_in), ctypes.byref(next_in), ctypes.byref(avail_out),
                                                     ctypes.byref(next_out), None)
                got += buf.raw[:cap - avail_out.value]
                if not L.BrotliEncoderHasMoreOutput(h):
                    break
            outs.append(bytes(got))
        return outs
    finally:
        L.BrotliEncoderDestroyInstance(h)


def device_steps(kv, steps, dictionary=None):
    """The device stream's output after each step: (the whole output, the size after each step), one synchronisation at the end."""
    import torch
    import rust_brotli_b200 as rb
    p = params_of(kv)
    d = None
    if dictionary is not None:
        d = torch.frombuffer(bytearray(dictionary), dtype=torch.uint8).cuda() if dictionary else torch.empty(0, dtype=torch.uint8,
                                                                                                               device="cuda")
    s = rb.DeviceStreamEncoder(p, dictionary=d)
    blob = b"".join(data for _, data in steps)
    dev = torch.frombuffer(bytearray(blob) + b"\0", dtype=torch.uint8).cuda()
    sizes, o = [], 0
    for op, data in steps:
        t = dev[o:o + len(data)]
        o += len(data)
        {PROCESS: s.write, FLUSH: s.flush, FINISH: s.finish}[op](t)
        sizes.append(s.output()[1].clone())
    out, size, status = s.output()
    torch.cuda.synchronize()
    s.close()
    assert int(status.item()) == 0
    return bytes(out[:int(size.item())].cpu().numpy()), [int(x.item()) for x in sizes]


def params_of(kv):
    import rust_brotli_b200 as rb
    p = rb.BrotliEncoderParams()
    names = {rb.BROTLI_PARAM_QUALITY: "quality", rb.BROTLI_PARAM_LGWIN: "lgwin", rb.BROTLI_PARAM_SIZE_HINT: "size_hint",
             rb.BROTLI_PARAM_DISABLE_LITERAL_CONTEXT_MODELING: "disable_literal_context_modeling", rb.BROTLI_PARAM_CATABLE: "catable",
             rb.BROTLI_PARAM_APPENDABLE: "appendable", rb.BROTLI_PARAM_MAGIC_NUMBER: "magic_number",
             rb.BROTLI_PARAM_BYTE_ALIGN: "byte_align", rb.BROTLI_PARAM_BARE_STREAM: "bare_stream"}
    for k, v in kv:
        if k == rb.BROTLI_PARAM_NO_DICTIONARY:
            p.use_dictionary = not v
        else:
            setattr(p, names[k], type(getattr(p, names[k]))(v))
    return p


def check(kv, steps, dictionary=None):
    """Device bytes == host bytes after every step; returns the whole stream."""
    want = host_steps(params_of(kv).as_key_values(), steps, dictionary)
    got, sizes = device_steps(kv, steps, dictionary)
    cum, acc = [], 0
    for w in want:
        acc += len(w)
        cum.append(acc)
    assert sizes == cum
    assert got == b"".join(want)
    return got, sizes


def q(quality, lgwin=22, *extra):
    import rust_brotli_b200 as rb
    return [(rb.BROTLI_PARAM_QUALITY, quality), (rb.BROTLI_PARAM_LGWIN, lgwin)] + list(extra)


WRITE_SIZES = [0, 1, 2, 3, 4095, 4096, 65537, MiB, 24 * MiB + 1]


@pytest.mark.parametrize("flush", [False, True])
def test_write_sizes(flush):
    src = text(sum(WRITE_SIZES))
    steps, o = [], 0
    for n in WRITE_SIZES:
        steps.append((PROCESS, src[o:o + n]))
        o += n
        if flush:
            steps.append((FLUSH, b""))
    steps.append((FINISH, b""))
    c, _ = check(q(5), steps)
    assert sys_decompress(c, len(src)) == src


@pytest.mark.parametrize("quality,lgwin,n", [(5, 16, 700_000), (7, 18, 700_000), (9, 22, 700_000), (5, 24, 700_000),
                                             (10, 22, 90_000), (11, 16, 90_000), (11, 24, 60_000)])
def test_qualities_and_windows(quality, lgwin, n):
    d = text(n, seed=quality)
    a, b = n // 3, n // 3 + 5
    c, _ = check(q(quality, lgwin), [(PROCESS, d[:a]), (FLUSH, b""), (PROCESS, d[a:b]), (FLUSH, d[b:b + 7]), (FINISH, d[b + 7:])])
    assert sys_decompress(c, n) == d


def test_large_window_two_sort_batches():
    """lgwin 24: a 24 MiB FLUSH behind a full 16 MiB window takes two sort batches and rebases the window."""
    d = text(17 * MiB + 24 * MiB + 3, seed=11)
    c, _ = check(q(5, 24), [(FLUSH, d[:17 * MiB]), (FLUSH, d[17 * MiB:]), (FINISH, b"")])
    assert sys_decompress(c, len(d)) == d


def _flags():
    import rust_brotli_b200 as rb
    return {"catable": [(rb.BROTLI_PARAM_CATABLE, 1)], "appendable": [(rb.BROTLI_PARAM_APPENDABLE, 1)],
            "magic": [(rb.BROTLI_PARAM_MAGIC_NUMBER, 1)], "byte_align": [(rb.BROTLI_PARAM_BYTE_ALIGN, 1)],
            "appendable_byte_align": [(rb.BROTLI_PARAM_APPENDABLE, 1), (rb.BROTLI_PARAM_BYTE_ALIGN, 1)],
            "bare": [(rb.BROTLI_PARAM_BARE_STREAM, 1)], "catable_bare": [(rb.BROTLI_PARAM_CATABLE, 1), (rb.BROTLI_PARAM_BARE_STREAM, 1)],
            "catable_magic_byte_align": [(rb.BROTLI_PARAM_CATABLE, 1), (rb.BROTLI_PARAM_MAGIC_NUMBER, 1), (rb.BROTLI_PARAM_BYTE_ALIGN, 1)],
            "no_dictionary": [(rb.BROTLI_PARAM_NO_DICTIONARY, 1)], "no_context": [(rb.BROTLI_PARAM_DISABLE_LITERAL_CONTEXT_MODELING, 1)],
            "size_hint": [(rb.BROTLI_PARAM_SIZE_HINT, 5000)]}


FLAG_NAMES = ["catable", "appendable", "magic", "byte_align", "appendable_byte_align", "bare", "catable_bare",
              "catable_magic_byte_align", "no_dictionary", "no_context", "size_hint"]


@pytest.mark.parametrize("flag", FLAG_NAMES)
def test_framing_and_options(flag):
    import rust_brotli_b200 as rb
    extra = _flags()[flag]
    d = golden_bytes("alice29.txt")
    sequences = [[(FINISH, b"")], [(FLUSH, d[:1]), (FINISH, b"")], [(FINISH, d[:2])], [(FLUSH, b""), (FINISH, d[:3])],
                 [(PROCESS, d[:1]), (FLUSH, b""), (PROCESS, d[1:100_001]), (FLUSH, b""), (PROCESS, d[100_001:100_003]), (FINISH, b"")]]
    for seq in sequences:
        check(q(5, 22, *extra), seq)
    check(q(9, 20, *extra), [(FLUSH, d[:40_000]), (FINISH, d[40_000:])], dictionary=d[100_000:130_000])
    bare = any(k == rb.BROTLI_PARAM_BARE_STREAM for k, _ in extra)
    if not bare:  # a bare stream has no final metablock: it does not decode on its own
        c, _ = check(q(5, 22, *extra), [(FLUSH, d[:50_000]), (FINISH, d[50_000:])])
        assert sys_decompress(c, len(d)) == d


@pytest.mark.parametrize("dict_size", [0, 1, 2, 1000, 70_000])
def test_custom_dictionary(dict_size):
    """Dictionaries of 0, 1, 2, a few and more than 2^lgwin - 16 bytes (lgwin 16): host identity; the stream decodes with the
    dictionary and does not reproduce the input with another one."""
    alice = golden_bytes("alice29.txt")
    dictionary, payload = alice[:dict_size], alice[dict_size // 2:dict_size // 2 + 90_000]
    c, _ = check(q(5, 16), [(FLUSH, payload[:30_000]), (PROCESS, payload[30_000:]), (FINISH, b"")], dictionary=dictionary)
    if dict_size > 1:
        assert sys_decompress_with_dictionary(c, len(payload), dictionary) == payload
    else:  # nothing of it is window content
        assert sys_decompress(c, len(payload)) == payload
    if dict_size >= 1000:
        other = bytes(reversed(dictionary))
        try:
            assert sys_decompress_with_dictionary(c, len(payload), other) != payload
        except ValueError:
            pass  # rejected outright


def _decode_prefix(comp, max_out, dictionary=None):
    """(result, output) of one BrotliDecoderDecompressStream call over comp: 1 = finished, 2 = needs more input."""
    from oracle.harness import _libs
    _, dec = _libs()
    dec.BrotliDecoderCreateInstance.restype = ctypes.c_void_p
    dec.BrotliDecoderCreateInstance.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    dec.BrotliDecoderAttachDictionary.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_char_p]
    dec.BrotliDecoderAttachDictionary.restype = ctypes.c_int
    dec.BrotliDecoderDecompressStream.argtypes = [ctypes.c_void_p] + [ctypes.c_void_p] * 5
    dec.BrotliDecoderDecompressStream.restype = ctypes.c_int
    dec.BrotliDecoderDestroyInstance.argtypes = [ctypes.c_void_p]
    st = dec.BrotliDecoderCreateInstance(None, None, None)
    try:
        if dictionary:
            assert dec.BrotliDecoderAttachDictionary(st, 0, len(dictionary), dictionary)
        out = ctypes.create_string_buffer(max_out + 16)
        avail_in, avail_out = ctypes.c_size_t(len(comp)), ctypes.c_size_t(len(out))
        next_in = ctypes.c_void_p(ctypes.cast(ctypes.c_char_p(comp), ctypes.c_void_p).value)
        next_out = ctypes.c_void_p(ctypes.addressof(out))
        res = dec.BrotliDecoderDecompressStream(st, ctypes.addressof(avail_in), ctypes.addressof(next_in), ctypes.addressof(avail_out),
                                                ctypes.addressof(next_out), None)
        return res, out.raw[:len(out) - avail_out.value]
    finally:
        dec.BrotliDecoderDestroyInstance(st)


@pytest.mark.parametrize("with_dict", [False, True])
def test_every_flush_decodes(with_dict):
    """After each FLUSH, out[:size] decodes to exactly the input so far and the decoder asks for more; after FINISH it is done."""
    alice = golden_bytes("alice29.txt") + golden_bytes("asyoulik.txt")
    dictionary = alice[-40_000:] if with_dict else None
    d = text(3 * MiB, seed=2) + alice
    cuts = [0, 1, 5, 4096, 70_000, 1_000_000, 3 * MiB, len(d)]
    steps = [(FLUSH, d[a:b]) for a, b in zip(cuts, cuts[1:])] + [(FINISH, b"")]
    whole, sizes = device_steps(q(5, 20), steps, dictionary)
    for (a, b), size in zip(zip(cuts, cuts[1:]), sizes):
        res, got = _decode_prefix(whole[:size], len(d), dictionary)
        assert res == 2 and got == d[:b], b
    res, got = _decode_prefix(whole, len(d), dictionary)
    assert res == 1 and got == d
    if with_dict:
        assert sys_decompress_with_dictionary(whole, len(d), dictionary) == d
    else:
        assert sys_decompress(whole, len(d)) == d


def test_long_stream_is_emitted_in_pieces():
    """230 MB in 8 MiB PROCESS writes: 96 MiB pieces leave before FINISH, the window stays bounded, the bytes equal the host's."""
    base = text(23_000_000, seed=5)
    d = base * 10
    steps = [(PROCESS, d[o:o + 8 * MiB]) for o in range(0, len(d), 8 * MiB)] + [(FINISH, b"")]
    c, sizes = check(q(5), steps)
    assert sizes[-2] > 0, "no output before FINISH"
    assert sys_decompress(c, len(d)) == d


def test_compress_tensor_dictionary_gain():
    """compress_tensor(dictionary=...) equals the host stream with BrotliEncoderSetCustomDictionary and one FINISH, and gains
    from a dictionary that holds the payload's prefix (as test_custom_dictionary_and_abi_details)."""
    import torch
    import rust_brotli_b200 as rb
    d = golden_bytes("alice29.txt")
    dictionary, payload = d[:60000], d[50000:120000]
    p = rb.BrotliEncoderParams(quality=5)
    t = torch.frombuffer(bytearray(payload), dtype=torch.uint8).cuda()
    dd = torch.frombuffer(bytearray(dictionary), dtype=torch.uint8).cuda()
    out, size = rb.compress_tensor(t, params=p, dictionary=dd)
    plain, psize = rb.compress_tensor(t, params=p)
    with_dict = bytes(out[:int(size.item())].cpu().numpy())
    assert with_dict == b"".join(host_steps(p.as_key_values(), [(FINISH, payload)], dictionary))
    assert sys_decompress_with_dictionary(with_dict, len(payload), dictionary) == payload
    assert len(with_dict) < 0.9 * int(psize.item())


def test_stream_order():
    """The call returns before the stream runs; the input is read after the work in front of it (a sleep, then the kernel that
    writes it) and copied before the work behind it (which overwrites it)."""
    import time
    import torch
    import rust_brotli_b200 as rb
    d = golden_bytes("alice29.txt")
    src = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
    t = torch.zeros_like(src)
    for timed in (False, True):  # the first round sizes the shared encoder's workspace, which grows with a blocking cudaFree
        s = rb.DeviceStreamEncoder(rb.BrotliEncoderParams(quality=5))
        s.write(torch.zeros(1, dtype=torch.uint8, device="cuda"))
        s.flush()
        torch.cuda.synchronize()
        head = bytes(s.output()[0][:int(s.output()[1].item())].cpu().numpy())
        done = torch.cuda.Event()
        if timed:
            torch.cuda._sleep(200_000_000)
        t.copy_(src)
        t0 = time.perf_counter()
        s.finish(t)
        host_ms = (time.perf_counter() - t0) * 1e3
        done.record()
        t.fill_(0x55)
        if timed:
            assert not done.query(), "the call waited for the stream"
        torch.cuda.synchronize()
    out, size, status = s.output()
    got = bytes(out[:int(size.item())].cpu().numpy())
    want = host_steps(rb.BrotliEncoderParams(quality=5).as_key_values(), [(PROCESS, b"\0"), (FLUSH, b""), (FINISH, d)])
    assert got == b"".join(want) and got[:len(head)] == head and int(status.item()) == 0
    assert host_ms < 1000


def _raw_stream(kv, dictionary=None):
    import torch
    import rust_brotli_b200 as rb
    from rust_brotli_b200 import _native
    L = rb.lib()
    enc = rb.DeviceEncoder(0)
    n, keys, vals = _native.key_value_arrays(kv)
    h = L.b200_stream_create(enc._h, n, ctypes.cast(keys, ctypes.c_void_p), ctypes.cast(vals, ctypes.c_void_p),
                             ctypes.c_void_p(dictionary.data_ptr() if dictionary is not None else 0),
                             dictionary.numel() if dictionary is not None else 0, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return L, enc, h


def _call(L, h, op, t, out, size, status, cap=None, stream=None):
    import torch
    st = torch.cuda.current_stream() if stream is None else stream
    n = t.numel() if t is not None else 0
    return L.b200_stream_compress_async(h, op, ctypes.c_void_p(t.data_ptr() if n else 0), n, ctypes.c_void_p(out.data_ptr()),
                                        out.numel() if cap is None else cap, ctypes.c_void_p(size.data_ptr()),
                                        ctypes.c_void_p(status.data_ptr()), ctypes.c_void_p(st.cuda_stream))


def test_output_too_small_fails_the_stream():
    import torch
    d = golden_bytes("alice29.txt")
    t = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
    L, enc, h = _raw_stream(q(5))
    try:
        out = torch.full((1 << 20,), 0xA5, dtype=torch.uint8, device="cuda")
        size = torch.zeros(1, dtype=torch.int64, device="cuda")
        status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        assert _call(L, h, FLUSH, t[:20_000], out, size, status)
        torch.cuda.synchronize()
        first = int(size.item())
        assert int(status.item()) == 0 and 0 < first
        assert _call(L, h, FLUSH, t[20_000:], out, size, status, cap=first + 100)  # the piece needs far more than 100 bytes
        torch.cuda.synchronize()
        assert int(status.item()) == 2 and int(size.item()) == first
        assert bool((out[first:] == 0xA5).all())
        status.fill_(-1)
        assert _call(L, h, FINISH, None, out, size, status)  # failed: nothing more is appended
        torch.cuda.synchronize()
        assert int(status.item()) == 2 and int(size.item()) == first and bool((out[first:] == 0xA5).all())
        # the cursor was reset on purpose: the pieces come separately
    finally:
        L.b200_stream_destroy(h)
        enc.close()


def test_cursor_reset_gives_separate_pieces():
    import torch
    d = golden_bytes("alice29.txt")
    t = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
    L, enc, h = _raw_stream(q(5))
    try:
        out = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
        size = torch.zeros(1, dtype=torch.int64, device="cuda")
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        pieces = []
        for op, a, b in ((FLUSH, 0, 50_000), (PROCESS, 50_000, 60_000), (FINISH, 60_000, len(d))):
            size.zero_()
            assert _call(L, h, op, t[a:b], out, size, status)
            torch.cuda.synchronize()
            pieces.append(bytes(out[:int(size.item())].cpu().numpy()))
        assert int(status.item()) == 0
        assert pieces == host_steps(q(5), [(FLUSH, d[:50_000]), (PROCESS, d[50_000:60_000]), (FINISH, d[60_000:])])
    finally:
        L.b200_stream_destroy(h)
        enc.close()


def test_refusals_enqueue_nothing():
    import torch
    import rust_brotli_b200 as rb
    d = golden_bytes("alice29.txt")[:10_000]
    t = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
    L, enc, h = _raw_stream(q(5))
    try:
        assert L.b200_stream_create(enc._h, 1, ctypes.cast((ctypes.c_int * 1)(rb.BROTLI_PARAM_LARGE_WINDOW), ctypes.c_void_p),
                                    ctypes.cast((ctypes.c_uint32 * 1)(1), ctypes.c_void_p), None, 0, None) is None
        out = torch.full((1 << 16,), 0xA5, dtype=torch.uint8, device="cuda")
        size = torch.full((1,), 7, dtype=torch.int64, device="cuda")
        status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        host = ctypes.create_string_buffer(1 << 16)
        vp = ctypes.c_void_p
        st = vp(torch.cuda.current_stream().cuda_stream)
        assert not L.b200_stream_compress_async(None, FLUSH, vp(t.data_ptr()), 10, vp(out.data_ptr()), 1 << 16, vp(size.data_ptr()),
                                                vp(status.data_ptr()), st)
        assert not L.b200_stream_compress_async(h, FLUSH, None, 10, vp(out.data_ptr()), 1 << 16, vp(size.data_ptr()),
                                                vp(status.data_ptr()), st)
        assert not L.b200_stream_compress_async(h, FLUSH, vp(t.data_ptr()), 10, ctypes.cast(host, vp), 1 << 16, vp(size.data_ptr()),
                                                vp(status.data_ptr()), st)
        assert not L.b200_stream_compress_async(h, FLUSH, ctypes.cast(host, vp), 10, vp(out.data_ptr()), 1 << 16,
                                                vp(size.data_ptr()), vp(status.data_ptr()), st)
        assert not L.b200_stream_compress_async(h, FLUSH, vp(t.data_ptr()), 10, vp(out.data_ptr()), 1 << 16, None,
                                                vp(status.data_ptr()), st)
        assert not _call(L, h, EMIT_METADATA, t, out, size, status)
        assert not _call(L, h, 9, t, out, size, status)
        # under capture: refused, and the capture stays valid
        side = torch.cuda.Stream()
        x = torch.zeros(4, device="cuda")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(side):
            with torch.cuda.graph(g, stream=side):
                x.add_(1)
                assert not _call(L, h, FLUSH, t, out, size, status, stream=side)
                x.add_(1)
        g.replay()
        torch.cuda.synchronize()
        assert x.tolist() == [2.0] * 4
        assert int(size.item()) == 7 and int(status.item()) == -1 and bool((out == 0xA5).all())
        # after FINISH every op is refused
        size.zero_()
        assert _call(L, h, FINISH, t, out, size, status)
        torch.cuda.synchronize()
        n = int(size.item())
        assert sys_decompress(bytes(out[:n].cpu().numpy()), len(d)) == d
        for op in (PROCESS, FLUSH, FINISH):
            assert not _call(L, h, op, None, out, size, status)
            assert not _call(L, h, op, t, out, size, status)
        assert L.b200_stream_output_bound(h, FINISH, 0) == 0
        torch.cuda.synchronize()
        assert int(size.item()) == n
    finally:
        L.b200_stream_destroy(h)
        enc.close()

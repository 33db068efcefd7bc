"""Stream-ordered device compression: b200_encoder_compress_range_async, DeviceEncoder.compress_async / reserve and
rust_brotli_b200.compress_tensor.

The async call must give the bytes of the blocking device path (b200_encoder_compress_range, device_io 1), return before the
caller's stream has run, read its input only after the work enqueued before it, replay correctly from a CUDA graph, refuse what
it cannot do without enqueuing anything, and keep the calls of one encoder in order across streams."""
import ctypes

import pytest

from conftest import golden_bytes
from oracle.harness import sys_decompress

SLEEP_CYCLES = 400_000_000  # torch.cuda._sleep: about 0.2 s of one spinning thread at the H100's clocks


def test_refused_without_encoder():
    """No device or a null encoder: the async call and the reservation return 0 and touch nothing."""
    import rust_brotli_b200 as rb
    L = rb.lib()
    size = ctypes.c_uint64(7)
    assert L.b200_encoder_compress_range_async(None, 5, 22, 0, None, 0, 0, 0, 1, 1, 0, None, 0, ctypes.addressof(size), None) == 0
    assert L.b200_encoder_reserve(None, 5, 22, 0, 1000, 1000) == 0
    assert size.value == 7


# ---- helpers (GPU) ----

def _dev(data: bytes):
    import torch
    if not data:
        return torch.empty(0, dtype=torch.uint8, device="cuda")
    return torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()


def _cap(enc, range_len):
    return enc._L.b200_max_compressed_size(range_len) + 64


def _blocking(enc, d_in, n, q, w, rs=0, rl=None, first=True, last=True, align=False):
    """b200_encoder_compress_range with device input and output (device_io 1), read back to bytes."""
    import torch
    rl = n - rs if rl is None else rl
    cap = _cap(enc, rl)
    out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    osz = ctypes.c_size_t(0)
    torch.cuda.synchronize()
    assert enc._L.b200_encoder_compress_range(enc._h, q, w, 0, ctypes.c_void_p(d_in.data_ptr()), n, rs, rl, int(first), int(last),
                                              int(align), ctypes.c_void_p(out.data_ptr()), cap, ctypes.byref(osz), 1)
    return bytes(out[:osz.value].cpu().numpy())


def _async(enc, d_in, n, q, w, rs=0, rl=None, first=True, last=True, align=False, stream=None):
    """compress_async on `stream` (default: the current stream); returns the (out, size) tensors without waiting."""
    import torch
    rl = n - rs if rl is None else rl
    cap = _cap(enc, rl)
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    size = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream() if stream is None else stream
    enc.compress_async(d_in.data_ptr(), n, out.data_ptr(), cap, size.data_ptr(), q, w, st.cuda_stream, rs, rl, first, last, align)
    return out, size


def _read(out, size):
    import torch
    torch.cuda.synchronize()
    k = int(size.item())
    assert 0 <= k <= out.numel()
    return bytes(out[:k].cpu().numpy())


def _inputs():
    from tools import datagen
    return {"empty": b"", "1B": b"x", "alice29": golden_bytes("alice29.txt"), "enwik300k": datagen.enwik_like(300_000),
            "json5m": datagen.json_logs(5_000_000), "random1m": datagen.pcg_random(1_000_000)}


_CACHE = {}


def _cached_inputs():
    if not _CACHE:
        _CACHE.update(_inputs())
    return _CACHE


# ---- byte parity with the blocking path ----

@pytest.mark.gpu
@pytest.mark.parametrize("q", [5, 6, 9, 10, 11])
@pytest.mark.parametrize("lgwin", [16, 22, 24])
def test_async_equals_blocking(encoder, q, lgwin):
    for name, d in _cached_inputs().items():
        if q == 11 and len(d) > 200_000:  # quality 11 on small inputs only
            continue
        t = _dev(d)
        ref = _blocking(encoder, t, len(d), q, lgwin)
        got = _read(*_async(encoder, t, len(d), q, lgwin))
        assert got == ref, (name, q, lgwin, len(got), len(ref))
        assert sys_decompress(got, max(len(d), 1)) == d, name


@pytest.mark.gpu
def test_async_three_chunks_over_the_lanes(encoder):
    """60 MB: three 24 MiB chunks on three lanes, bit positions chained through k_layout, one size launch at the end."""
    from tools import datagen
    d = datagen.enwik_like(60_000_000, seed=11)
    t = _dev(d)
    ref = _blocking(encoder, t, len(d), 5, 22)
    got = _read(*_async(encoder, t, len(d), 5, 22))
    assert got == ref
    assert sys_decompress(got, len(d)) == d


@pytest.mark.gpu
def test_async_lgwin24_two_sort_batches(encoder):
    """lgwin 24: a 24 MiB chunk with its 16 MiB window takes two sort batches."""
    from tools import datagen
    d = datagen.enwik_like(28_000_000, seed=3)
    t = _dev(d)
    ref = _blocking(encoder, t, len(d), 5, 24)
    got = _read(*_async(encoder, t, len(d), 5, 24))
    assert got == ref
    assert sys_decompress(got, len(d)) == d


@pytest.mark.gpu
@pytest.mark.parametrize("q", [5, 10])
def test_async_ranges(encoder, q):
    """Ranges with every first / last / byte_align combination, including ranges whose window starts inside the input (the staged
    span begins at a 4 KiB boundary in front of the range); the byte-aligned pieces concatenate into one stream."""
    from tools import datagen
    d = datagen.json_logs(6_000_000, seed=9)
    t = _dev(d)
    cuts = [(0, 1, True, False, True), (1, 2_999_999, False, False, True), (3_000_000, 2_000_000, False, False, True),
            (5_000_000, 1_000_000, False, True, False)]
    pieces = []
    for rs, rl, first, last, align in cuts:
        ref = _blocking(encoder, t, len(d), q, 22, rs, rl, first, last, align)
        got = _read(*_async(encoder, t, len(d), q, 22, rs, rl, first, last, align))
        assert got == ref, (rs, rl, first, last, align)
        pieces.append(got)
    assert sys_decompress(b"".join(pieces), len(d)) == d
    for rs, rl, first, last, align in [(4_500_000, 70_001, False, False, False), (4_500_000, 70_001, True, True, False),
                                       (4_500_000, 70_001, False, True, True), (4_500_000, 0, True, True, True),
                                       (0, 0, True, True, False)]:
        ref = _blocking(encoder, t, len(d), q, 22, rs, rl, first, last, align)
        got = _read(*_async(encoder, t, len(d), q, 22, rs, rl, first, last, align))
        assert got == ref, (rs, rl, first, last, align)


# ---- no host wait, ordering after the caller's stream ----

@pytest.mark.gpu
def test_call_returns_before_the_stream_runs():
    import torch
    import rust_brotli_b200 as rb
    from tools import datagen
    d = datagen.enwik_like(3_000_000, seed=2)
    enc = rb.DeviceEncoder(0)
    try:
        t = _dev(d)
        ref = _blocking(enc, t, len(d), 5, 22)
        enc.reserve(5, 22, len(d))
        s = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
            out, size = _async(enc, t, len(d), 5, 22, stream=s)
            assert not s.query(), "the call waited for the stream"
        s.synchronize()
        assert _read(out, size) == ref
    finally:
        enc.close()


@pytest.mark.gpu
def test_input_is_read_after_the_callers_work(encoder):
    """A torch copy writes the input on the stream behind a spin kernel; the call follows with no synchronisation and must see
    the new contents.  The same through compress_tensor on the current stream."""
    import torch
    import rust_brotli_b200 as rb
    d = golden_bytes("alice29.txt")
    src = _dev(d)
    ref = _blocking(encoder, src, len(d), 5, 22)
    s = torch.cuda.Stream()
    for via_tensor in (False, True):
        dst = torch.zeros_like(src)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
            dst.copy_(src)
            if via_tensor:
                out, size = rb.compress_tensor(dst, 5, 22, encoder=encoder)
            else:
                out, size = _async(encoder, dst, len(d), 5, 22, stream=s)
        s.synchronize()
        assert out.dtype == torch.uint8 and size.dtype == torch.int64 and size.numel() == 1 and size.is_cuda
        assert _read(out, size) == ref, via_tensor


@pytest.mark.gpu
def test_compress_tensor_default_encoder_and_empty():
    import torch
    import rust_brotli_b200 as rb
    d = golden_bytes("asyoulik.txt")
    out, size = rb.compress_tensor(_dev(d), quality=9, lgwin=20)
    assert sys_decompress(_read(out, size), len(d)) == d
    out, size = rb.compress_tensor(torch.empty(0, dtype=torch.uint8, device="cuda"))
    assert _read(out, size) == b"\x06"
    with pytest.raises(ValueError):
        rb.compress_tensor(torch.zeros(16, dtype=torch.int32, device="cuda"))


# ---- CUDA graph capture ----

def _capture_one(enc, static_in, n, q, w, static_out, static_size):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        enc.compress_async(static_in.data_ptr(), n, static_out.data_ptr(), static_out.numel(), static_size.data_ptr(), q, w,
                           torch.cuda.current_stream().cuda_stream)
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("q", [5, 10])
def test_graph_capture_and_replay(encoder, q):
    """One call captured with static input / output / size tensors; three different inputs of the same length copied into the
    static input, each replay equals the blocking compression of that input."""
    import torch
    import rust_brotli_b200 as rb
    from tools import datagen
    n = 1_000_000
    inputs = [datagen.enwik_like(n, seed=21), datagen.json_logs(n, seed=22), (golden_bytes("alice29.txt") * 7)[:n]]
    refs = [_blocking(encoder, _dev(d), n, q, 22) for d in inputs]
    enc = rb.DeviceEncoder(0)
    try:
        enc.reserve(q, 22, n)
        static_in = torch.zeros(n, dtype=torch.uint8, device="cuda")
        static_out = torch.empty(_cap(enc, n), dtype=torch.uint8, device="cuda")
        static_size = torch.zeros(1, dtype=torch.int64, device="cuda")
        _read(*_async(enc, static_in, n, q, 22))  # warm-up outside the capture (module loading)
        g = _capture_one(enc, static_in, n, q, 22, static_out, static_size)
        for d, ref in zip(inputs, refs):
            static_in.copy_(torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda())
            g.replay()
            assert _read(static_out, static_size) == ref
        # the captured encoder still serves calls of its reserved size outside the graph
        assert _read(*_async(enc, _dev(inputs[0]), n, q, 22)) == refs[0]
    finally:
        enc.close()


@pytest.mark.gpu
def test_capture_refusals():
    """Without a reservation the call inside a capture is refused and the capture still ends cleanly; after a capture a larger
    call on the same encoder (async or blocking) is refused, and the graph still replays correctly."""
    import torch
    import rust_brotli_b200 as rb
    from tools import datagen
    n = 300_000
    d = datagen.enwik_like(2 * n, seed=31)
    enc = rb.DeviceEncoder(0)
    try:
        static_in = _dev(d[:n])
        static_out = torch.empty(_cap(enc, n), dtype=torch.uint8, device="cuda")
        static_size = torch.zeros(1, dtype=torch.int64, device="cuda")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            static_size.fill_(-5)
            with pytest.raises(RuntimeError):
                enc.compress_async(static_in.data_ptr(), n, static_out.data_ptr(), static_out.numel(), static_size.data_ptr(), 5,
                                   22, torch.cuda.current_stream().cuda_stream)
        g.replay()
        torch.cuda.synchronize()
        assert int(static_size.item()) == -5
        ref = _blocking(enc, static_in, n, 5, 22)
        enc.reserve(5, 22, n)
        _read(*_async(enc, static_in, n, 5, 22))  # warm-up outside the capture (module loading)
        g2 = _capture_one(enc, static_in, n, 5, 22, static_out, static_size)
        big = _dev(d)
        with pytest.raises(RuntimeError):
            _async(enc, big, 2 * n, 5, 22)
        big_out = torch.empty(_cap(enc, 2 * n), dtype=torch.uint8, device="cuda")
        osz = ctypes.c_size_t(0)
        torch.cuda.synchronize()
        assert not enc._L.b200_encoder_compress_range(enc._h, 5, 22, 0, ctypes.c_void_p(big.data_ptr()), 2 * n, 0, 2 * n, 1, 1, 0,
                                                      ctypes.c_void_p(big_out.data_ptr()), big_out.numel(), ctypes.byref(osz), 1)
        g2.replay()
        assert _read(static_out, static_size) == ref
    finally:
        enc.close()


@pytest.mark.gpu
def test_reserve_covers_smaller_calls(encoder):
    """A reservation for (q11, lgwin 24, 1 MB) covers a captured q10 call with a smaller size hint (smaller parse units) and a
    q5 call of fewer bytes with a smaller window."""
    import torch
    import rust_brotli_b200 as rb
    from tools import datagen
    d = datagen.enwik_like(200_000, seed=41)
    enc = rb.DeviceEncoder(0)
    try:
        enc.reserve(11, 24, 1_000_000)
        t = _dev(d)
        for q, w in ((10, 22), (5, 18)):
            out = torch.empty(_cap(enc, len(d)), dtype=torch.uint8, device="cuda")
            size = torch.zeros(1, dtype=torch.int64, device="cuda")
            _read(*_async(encoder, t, len(d), q, w))  # module loading outside the capture, on another encoder
            g = _capture_one(enc, t, len(d), q, w, out, size)
            g.replay()
            assert _read(out, size) == _blocking(encoder, t, len(d), q, w), (q, w)
    finally:
        enc.close()


# ---- one encoder, several streams ----

@pytest.mark.gpu
def test_two_streams_and_a_blocking_call():
    """Back-to-back async calls on one encoder from two streams (the first one held back by a spin kernel), then a blocking call,
    all without user synchronisation: the calls run one after the other on the device and every output is correct."""
    import torch
    import rust_brotli_b200 as rb
    from tools import datagen
    a, b, c = golden_bytes("alice29.txt"), datagen.enwik_like(3_000_000, seed=51), datagen.json_logs(2_000_000, seed=52)
    ta, tb, tc = _dev(a), _dev(b), _dev(c)
    enc = rb.DeviceEncoder(0)
    try:
        refs = [_blocking(enc, t, len(x), 5, 22) for t, x in ((ta, a), (tb, b), (tc, c))]
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(s1):
            torch.cuda._sleep(SLEEP_CYCLES)
            o1 = _async(enc, ta, len(a), 5, 22, stream=s1)
        with torch.cuda.stream(s2):
            o2 = _async(enc, tb, len(b), 5, 22, stream=s2)
        got3 = _blocking_no_sync(enc, tc, len(c), 5, 22)
        assert [_read(*o1), _read(*o2), got3] == refs
    finally:
        enc.close()


def _blocking_no_sync(enc, d_in, n, q, w):
    """As _blocking, without the torch.cuda.synchronize() in front of the call (the input is already complete)."""
    import torch
    cap = _cap(enc, n)
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")  # (no fill kernel: it would race with the copy into it)
    osz = ctypes.c_size_t(0)
    assert enc._L.b200_encoder_compress_range(enc._h, q, w, 0, ctypes.c_void_p(d_in.data_ptr()), n, 0, n, 1, 1, 0,
                                              ctypes.c_void_p(out.data_ptr()), cap, ctypes.byref(osz), 1)
    return bytes(out[:osz.value].cpu().numpy())


# ---- validation: refused with nothing enqueued ----

@pytest.mark.gpu
def test_validation_refuses_and_enqueues_nothing(encoder):
    import torch
    d = golden_bytes("alice29.txt")
    t = _dev(d)
    n = len(d)
    cap = _cap(encoder, n)
    out = torch.full((cap + 8,), 0x55, dtype=torch.uint8, device="cuda")
    size = torch.full((1,), -3, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    bad = [
        (t.data_ptr(), out.data_ptr(), cap - 1, size.data_ptr()),      # out_cap below b200_max_compressed_size + 64
        (t.data_ptr(), out.data_ptr() + 1, cap, size.data_ptr()),      # out not 4-byte aligned
        (t.data_ptr(), out.data_ptr(), cap, 0),                        # no size word
        (0, out.data_ptr(), cap, size.data_ptr()),                     # no input
    ]
    host = ctypes.create_string_buffer(cap)
    bad.append((t.data_ptr(), ctypes.addressof(host), cap, size.data_ptr()))  # host memory
    for i, (pin, pout, c, psize) in enumerate(bad):
        with pytest.raises(RuntimeError):
            encoder.compress_async(pin, n, pout, c, psize, 5, 22, st)
    with pytest.raises(RuntimeError):  # range past the end
        encoder.compress_async(t.data_ptr(), n, out.data_ptr(), cap, size.data_ptr(), 5, 22, st, range_start=10, range_len=n)
    torch.cuda.synchronize()
    assert int(size.item()) == -3
    assert bool((out == 0x55).all())
    if torch.cuda.device_count() < 2:
        pytest.skip("a pointer on another device needs a second GPU")
    other = torch.empty(cap, dtype=torch.uint8, device="cuda:1")
    with pytest.raises(RuntimeError):
        encoder.compress_async(t.data_ptr(), n, other.data_ptr(), cap, size.data_ptr(), 5, 22, st)
    torch.cuda.synchronize()
    assert int(size.item()) == -3

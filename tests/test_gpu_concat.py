"""GPU: b200_concat_async / rust_brotli_b200.concat_tensors, the BroCatli splice of device-resident streams.

Output and result must equal the host Broccoli ABI's sequence (create, new file + stream per part, finish) for every input,
successful outputs must decode to the concatenated inputs, failures must leave `out` untouched with size 0, totals above 4 GiB
must work, and the call must replay from a CUDA graph."""
import ctypes
import random

import pytest

from conftest import golden_bytes
from oracle.harness import sys_decompress
from test_broccoli import _pack, _window_bits, catable_from_model, splice

pytestmark = pytest.mark.gpu


def synthetic(data: bytes, lgwin: int, block: int = 65536) -> bytes:
    """A catable stream of uncompressed metablocks (MNIBBLES 4, <= 64 KiB each) ending in the empty last metablock."""
    bits = []

    def put(n, v):
        bits.extend((v >> i) & 1 for i in range(n))
    _window_bits(put, lgwin)
    parts = []
    for a in range(0, len(data), block):
        chunk = data[a:a + block]
        put(1, 0); put(2, 0); put(16, len(chunk) - 1); put(1, 1)
        parts.append(_pack(bits) + chunk)
        bits = []
    put(2, 3)
    return b"".join(parts) + _pack(bits)


def _lib():
    import rust_brotli_b200 as rb
    return rb._broccoli()


def device_splice(streams, window_size=0, out_cap=None):
    """All streams in one device buffer at odd offsets; returns (bytes, (code, index), out untouched past the size)."""
    import torch
    L = _lib()
    rnd = random.Random(len(streams))
    blob, offs = bytearray(), []
    for s in streams:
        blob += bytes(rnd.randrange(0, 20))
        offs.append(len(blob))
        blob += s
    blob += bytes(32)
    d = torch.frombuffer(blob, dtype=torch.uint8).cuda()
    n = len(streams)
    ptrs = torch.tensor([d.data_ptr() + o for o in offs] or [0], dtype=torch.int64, device="cuda")
    sizes = torch.tensor([len(s) for s in streams] or [0], dtype=torch.int64, device="cuda")
    ws = torch.empty(L.b200_concat_workspace_size(n), dtype=torch.uint8, device="cuda")
    cap = sum(len(s) for s in streams) + 3 if out_cap is None else out_cap
    out = torch.full((cap + 16,), 0xA5, dtype=torch.uint8, device="cuda")
    size = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    res = torch.full((2,), 99, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream()
    assert L.b200_concat_async(ptrs.data_ptr(), sizes.data_ptr(), n, window_size, out.data_ptr() + 1, cap, size.data_ptr(),
                               res.data_ptr(), ws.data_ptr(), ws.numel(), st.cuda_stream)
    torch.cuda.synchronize()
    sz = int(size.item())
    host = bytes(out.cpu().numpy())
    untouched = host[0] == 0xA5 and all(b == 0xA5 for b in host[1 + sz:])
    return host[1:1 + sz], tuple(int(x) for x in res.cpu()), untouched


def host_reference(streams, window_size=0):
    """The host sequence the device call must equal: (bytes, (code, index))."""
    import rust_brotli_b200 as rb
    bc = rb.BroCatli.new_with_window_size(window_size) if window_size else rb.BroCatli()
    out = bytearray()
    for k, s in enumerate(streams):
        bc.new_brotli_file()
        r, used, o = bc.stream(s, len(s) + 16)
        out += o
        if r >= 124:
            return b"", (r, k)
        assert r == rb.BROCCOLI_NEEDS_MORE_INPUT and used == len(s)
    r, o = bc.finish(16)
    assert r == 0
    return bytes(out + o), (0, -1)


def check(streams, window_size=0, datas=None):
    want, code = host_reference(streams, window_size)
    got, res, untouched = device_splice(streams, window_size)
    assert res == code
    assert got == want
    assert untouched
    assert len(got) <= sum(len(s) for s in streams) + 3
    if datas is not None and code[0] == 0:
        whole = b"".join(datas)
        assert sys_decompress(got, max(1, len(whole))) == whole
    return got


@pytest.fixture(scope="module")
def model_streams(model):
    alice, you = golden_bytes("alice29.txt"), golden_bytes("asyoulik.txt")
    return [(catable_from_model(model, alice[:30000], 5, 22), alice[:30000]),
            (catable_from_model(model, you[:20000], 10, 22, byte_align=True), you[:20000]),
            (catable_from_model(model, alice[500:9000], 9, 20, magic=True), alice[500:9000])]


def test_three_streams(model_streams):
    check([s for s, _ in model_streams], datas=[d for _, d in model_streams])


def test_two_thousand_streams_mixed_windows(model):
    rnd = random.Random(5)
    alice = golden_bytes("alice29.txt") * 2
    streams, datas = [], []
    windows = sorted([rnd.choice([10, 12, 15, 16, 17, 18, 20, 22, 24]) for _ in range(2000)], reverse=True)
    for i, w in enumerate(windows):
        n = rnd.choice([0, 1, 2, 3, rnd.randrange(0, 70000), rnd.randrange(0, 3000)])
        a = rnd.randrange(0, len(alice) - n)
        d = alice[a:a + n]
        if i % 20 == 0 and 3 <= n <= 3000:  # streams that end at any bit: the model's compressed metablocks
            s = catable_from_model(model, d, 5, w)
        else:
            s = synthetic(d, w)
        streams.append(s)
        datas.append(d)
    check(streams, datas=datas)


def test_edge_streams(model_streams):
    a, ad = model_streams[0]
    b, bd = model_streams[1]
    edges = [b"", b";", b"\x3b", b"\x3b\x00", b"\x11\x02\x03\x04", b"\x3b\x00\x00\x00"]
    for e in edges:
        check([e, a, b])
        check([a, e, b])
        check([a, b, e])
        check([e])
        check([e, e])
    check([])
    check([b"", a], datas=[ad])
    check([a, b"", b"\x3b", b], datas=[ad, bd])


@pytest.mark.parametrize("ws", [0, 5, 10, 15, 16, 17, 22, 24, 25, 30])
def test_window_size_instances(model_streams, ws):
    a = model_streams[0][0]
    small = synthetic(b"tiny window stream" * 10, 10)
    check([], window_size=ws)
    check([b""], window_size=ws)
    check([small, small], window_size=ws)
    check([a, small], window_size=ws)


def test_errors_leave_out_untouched(model, model_streams):
    a = model_streams[0][0]
    plain = model.compress(golden_bytes("asyoulik.txt")[:5000], 5, 22)[0]
    big = synthetic(b"x" * 1000, 24)
    for streams, code in (([a, plain], 127), ([a, b"\x71\x1b\x00\x00"], 127), ([synthetic(b"y" * 100, 18), big], 126),
                          ([a, a[:-1] + b"\x02", a], 124), ([a + b"\x00\x00", b""], 124), ([a, b"\x91\x00\x00\x00\x00"], 125)):
        got = check(streams)
        assert got == b""
        assert host_reference(streams)[1][0] == code
    # too small an output buffer: code 2, the first stream that does not fit, nothing written
    s3 = [synthetic(bytes(range(256)) * 40, 22)] * 3
    full, _, _ = device_splice(s3)
    for cap, idx in ((len(full) - 1, 3), (len(s3[0]) + 10, 1), (0, 0)):
        got, res, untouched = device_splice(s3, out_cap=cap)
        assert got == b"" and res == (2, idx) and untouched


def test_total_above_4gib():
    """Five 0.9 GiB catable streams of uncompressed metablocks spliced into one 4.5 GB stream: sizes and offsets past 2^32."""
    import torch
    L = _lib()
    n_streams, block = 5, 1 << 24
    payload = 56 * block  # 0.875 GiB per stream, 16 MiB metablocks (MNIBBLES 6)
    hdr = []
    for m in range(payload // block):  # byte-aligned headers: [window 22] ISLAST 0, MNIBBLES 6, MLEN - 1, ISUNCOMPRESSED
        bits = []

        def put(n, v):
            bits.extend((v >> i) & 1 for i in range(n))
        if m == 0:
            _window_bits(put, 22)
        put(1, 0); put(2, 2); put(24, block - 1); put(1, 1)
        hdr.append(_pack(bits))
    assert all(len(h) == 4 for h in hdr)
    slen = payload + 4 * len(hdr) + 1
    gen = torch.Generator(device="cuda").manual_seed(3)
    bufs = []
    for k in range(n_streams):
        t = torch.randint(0, 256, (slen,), dtype=torch.uint8, device="cuda", generator=gen)
        v = t[:slen - 1].view(len(hdr), block + 4)
        v[:, :4] = torch.tensor(list(b"".join(hdr)), dtype=torch.uint8, device="cuda").view(len(hdr), 4)
        t[-1] = 3
        bufs.append(t)
    ptrs = torch.tensor([t.data_ptr() for t in bufs], dtype=torch.int64, device="cuda")
    sizes = torch.full((n_streams,), slen, dtype=torch.int64, device="cuda")
    ws = torch.empty(L.b200_concat_workspace_size(n_streams), dtype=torch.uint8, device="cuda")
    cap = n_streams * slen + 3
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    size = torch.zeros(1, dtype=torch.int64, device="cuda")
    res = torch.zeros(2, dtype=torch.int32, device="cuda")
    assert L.b200_concat_async(ptrs.data_ptr(), sizes.data_ptr(), n_streams, 0, out.data_ptr(), cap, size.data_ptr(), res.data_ptr(),
                               ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert tuple(res.tolist()) == (0, -1)
    # stream 0 is copied but for its final 0x03; each later stream loses its window bits to the realigned header and its own
    # 0x03 byte, except the last: every stream adds exactly slen - 1 bytes, plus the final 0x03
    total = int(size.item())
    assert total == n_streams * (slen - 1) + 1 > (1 << 32)
    for k, t in enumerate(bufs):
        o = k * (slen - 1)
        assert torch.equal(out[o + 4:o + slen - 1], t[4:slen - 1]), k
        if k:  # the header bits behind the window bits, moved down by its 4 bits
            h = t[:4].cpu().tolist()
            v = int.from_bytes(bytes(h), "little") >> 4
            assert out[o:o + 4].cpu().tolist() == list(v.to_bytes(4, "little")), k
    assert out[:4].tolist() == bufs[0][:4].tolist() and int(out[total - 1]) == 3


def test_concat_tensors_stream_ordered_and_graph(model_streams):
    """concat_tensors on (out, size) device pairs: no host synchronisation in between, and a graph replay with new contents."""
    import torch
    import rust_brotli_b200 as rb
    streams = [s for s, _ in model_streams]
    datas = [d for _, d in model_streams]

    def as_parts(ss, caps):
        parts = []
        for s, c in zip(ss, caps):
            o = torch.zeros(c, dtype=torch.uint8, device="cuda")
            o[:len(s)] = torch.frombuffer(bytearray(s), dtype=torch.uint8).cuda()
            parts.append((o, torch.tensor([len(s)], dtype=torch.int64, device="cuda")))
        return parts
    caps = [len(s) + 100 for s in streams]
    parts = as_parts(streams, caps)
    out, size, result = rb.concat_tensors(parts)
    assert result.tolist() == [0, -1]
    got = bytes(out[:int(size.item())].cpu().numpy())
    assert got == host_reference(streams)[0]
    assert sys_decompress(got, sum(map(len, datas))) == b"".join(datas)

    # graph: pointer table and workspace are built before the capture; new contents are written into the same tensors
    ptrs = rb.concat_pointer_table(parts)
    ws = torch.empty(rb.concat_workspace_size(len(parts)), dtype=torch.uint8, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        rb.concat_tensors(parts, pointers=ptrs, workspace=ws)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gout, gsize, gres = rb.concat_tensors(parts, pointers=ptrs, workspace=ws)
    alice = golden_bytes("alice29.txt")
    new_datas = [alice[40000:40000 + caps[0] - 40], alice[:caps[1] // 2], b"q"]
    new_streams = [synthetic(new_datas[0], 22), synthetic(new_datas[1], 20), synthetic(b"q", 18)]
    for (o, s), ns in zip(parts, new_streams):
        assert len(ns) <= o.numel()
        o[:len(ns)] = torch.frombuffer(bytearray(ns), dtype=torch.uint8).cuda()
        s.fill_(len(ns))
    g.replay()
    torch.cuda.synchronize()
    assert gres.tolist() == [0, -1]
    got = bytes(gout[:int(gsize.item())].cpu().numpy())
    assert got == host_reference(new_streams)[0]
    assert sys_decompress(got, sum(map(len, new_datas))) == b"".join(new_datas)


def test_refused_calls():
    L = _lib()
    assert L.b200_concat_async(None, None, 1, 0, None, 0, None, None, None, 0, None) == 0
    buf = ctypes.create_string_buffer(64)
    p = ctypes.addressof(buf)
    assert L.b200_concat_async(p, p, 1, 0, p, 8, p, p, p, 0, None) == 0  # workspace too small
    assert L.b200_concat_async(p, p, 1, 300, p, 8, p, p, p, 1 << 20, None) == 0  # window size not a uint8


# ---- b200_encoder_compress_params_async / compress_tensor(params=...) ----

FRAMINGS = {"catable": dict(catable=True), "catable+magic": dict(catable=True, magic_number=True),
            "catable+byte_align": dict(catable=True, byte_align=True), "catable+bare": dict(catable=True, bare_stream=True),
            "appendable+byte_align": dict(appendable=True, byte_align=True), "magic": dict(magic_number=True),
            "bare": dict(bare_stream=True)}


def one_call_stream(data: bytes, params) -> bytes:
    """BrotliEncoderCompressStream called once with the whole input and BROTLI_OPERATION_FINISH."""
    import rust_brotli_b200 as rb
    s = rb._Stream(params)
    try:
        return s.step(data, rb.BROTLI_OPERATION_FINISH)
    finally:
        s.close()


def tensor_stream(enc, data: bytes, params) -> bytes:
    import torch
    import rust_brotli_b200 as rb
    t = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda() if data else torch.empty(0, dtype=torch.uint8, device="cuda")
    out, size = rb.compress_tensor(t, encoder=enc, params=params)
    return bytes(out[:int(size.item())].cpu().numpy())


@pytest.fixture(scope="module")
def framed_encoder():
    import rust_brotli_b200 as rb
    enc = rb.DeviceEncoder(0)
    yield enc
    enc.close()


@pytest.mark.parametrize("framing", sorted(FRAMINGS))
def test_params_async_equals_one_call_stream(framed_encoder, framing):
    import rust_brotli_b200 as rb
    alice = golden_bytes("alice29.txt")
    for data in (b"", b"A", b"Al", b"Ali", alice):
        p = rb.BrotliEncoderParams(quality=5, lgwin=22, **FRAMINGS[framing])
        want = one_call_stream(data, p)
        assert tensor_stream(framed_encoder, data, p) == want, (framing, len(data))
        if want and "bare" not in framing:  # a bare stream has no final metablock: it decodes only inside another stream
            assert sys_decompress(want, max(1, len(data))) == data


@pytest.mark.parametrize("q", [5, 9, 10, 11])
def test_params_async_qualities_and_windows(framed_encoder, q):
    import rust_brotli_b200 as rb
    alice = golden_bytes("alice29.txt")
    for w in (10, 16, 22, 24):
        for kw in (FRAMINGS["catable"], FRAMINGS["catable+magic"], {}):
            p = rb.BrotliEncoderParams(quality=q, lgwin=w, **kw)
            assert tensor_stream(framed_encoder, alice, p) == one_call_stream(alice, p), (q, w, kw)
    # options of this call only: the encoder's own stay as they were (context modelling and dictionary on)
    p = rb.BrotliEncoderParams(quality=q, lgwin=22, disable_literal_context_modeling=1, use_dictionary=False)
    assert tensor_stream(framed_encoder, alice, p) == one_call_stream(alice, p)
    assert tensor_stream(framed_encoder, alice, rb.BrotliEncoderParams(quality=q, lgwin=22)) == \
        one_call_stream(alice, rb.BrotliEncoderParams(quality=q, lgwin=22))


def test_params_async_multi_chunk(framed_encoder):
    import rust_brotli_b200 as rb
    from tools import datagen
    data = datagen.enwik_like(30_000_000, seed=4)
    for kw in (FRAMINGS["catable+byte_align"], FRAMINGS["magic"]):
        p = rb.BrotliEncoderParams(quality=5, lgwin=22, **kw)
        got = tensor_stream(framed_encoder, data, p)
        assert got == one_call_stream(data, p)
    assert sys_decompress(got, len(data)) == data


def test_params_async_refusals(framed_encoder):
    import torch
    L = framed_encoder._L
    t = torch.zeros(100, dtype=torch.uint8, device="cuda")
    out = torch.zeros(L.b200_max_compressed_size(100) + 64, dtype=torch.uint8, device="cuda")
    size = torch.full((1,), 7, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for kv in ([(6, 1)], [(3, 5)]):  # LARGE_WINDOW, LGBLOCK out of range: refused as by BrotliEncoderCompressMulti
        with pytest.raises(RuntimeError):
            framed_encoder.compress_params_async(t.data_ptr(), 100, out.data_ptr(), out.numel(), size.data_ptr(), kv, st)
    with pytest.raises(RuntimeError):  # out_cap below b200_max_compressed_size(n) + 64
        framed_encoder.compress_params_async(t.data_ptr(), 100, out.data_ptr(), out.numel() - 1, size.data_ptr(), [(167, 1)], st)
    assert int(size.item()) == 7


def test_params_async_graph_replay(framed_encoder):
    import torch
    import rust_brotli_b200 as rb
    alice = golden_bytes("alice29.txt")
    n = 100_000
    p = rb.BrotliEncoderParams(quality=5, lgwin=22, catable=True, magic_number=True, size_hint=n)
    framed_encoder.reserve(5, 22, n, size_hint=n)
    t = torch.frombuffer(bytearray(alice[:n]), dtype=torch.uint8).cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        rb.compress_tensor(t, encoder=framed_encoder, params=p)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gout, gsize = rb.compress_tensor(t, encoder=framed_encoder, params=p)
    new = (alice[60000:] + alice)[:n]
    t.copy_(torch.frombuffer(bytearray(new), dtype=torch.uint8).cuda())
    g.replay()
    torch.cuda.synchronize()
    assert bytes(gout[:int(gsize.item())].cpu().numpy()) == one_call_stream(new, p)


def test_compress_tensor_then_concat_without_host_sync():
    """Catable streams compressed on the GPU and spliced there: everything is enqueued behind a long kernel before any of it
    runs, so nothing in between waits on the host; the result decodes to the concatenated tensors."""
    import torch
    import rust_brotli_b200 as rb
    alice, you = golden_bytes("alice29.txt"), golden_bytes("asyoulik.txt")
    datas = [alice[:50000], b"", b"x", you[:40000], alice[100:30000]]
    ts = [torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda() if d else torch.empty(0, dtype=torch.uint8, device="cuda")
          for d in datas]
    enc = rb.DeviceEncoder(0)
    try:
        p = rb.BrotliEncoderParams(quality=5, lgwin=22, catable=True)
        for d, t in zip(datas, ts):  # allocate everything once, outside the timed part
            rb.compress_tensor(t, encoder=enc, params=p)
        torch.cuda.synchronize()
        torch.cuda._sleep(400_000_000)
        parts = [rb.compress_tensor(t, encoder=enc, params=p) for t in ts]
        out, size, result = rb.concat_tensors(parts)
        assert not torch.cuda.current_stream().query()  # still behind the sleep: no host wait happened
        torch.cuda.synchronize()
        assert result.tolist() == [0, -1]
        got = bytes(out[:int(size.item())].cpu().numpy())
        assert got == host_reference([one_call_stream(d, p) for d in datas])[0]
        assert sys_decompress(got, sum(map(len, datas))) == b"".join(datas)
    finally:
        enc.close()

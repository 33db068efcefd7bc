"""GPU (H100): quality 9.5 (BROTLI_PARAM_Q9_5) -- the hash-chain parse under the quality 10 / 11 metablock builder.

  * the reference's own size pin (random_then_unicode, quality 11 + Q9_5, lgwin 22, size hint 2 MiB, 4096-byte writes);
  * device == the CPU model's sha256 goldens (tests/q95_cases.py, checked on the CPU by tests/test_model_q95.py), every stream
    decoded by libbrotlidec;
  * the match stage: Q9_5 at quality 5..8 switches H5 to H6 above a 1 MiB size hint; the 512-deep buckets of quality 11 + Q9_5
    against the brute force of tests/match_ref.py, up front and on demand, including a chunk of two sort batches;
  * the entropy stage read back by tests/stream_audit.py;
  * every entry point gives the same bytes, including a CUDA graph capture after reserve();
  * the parameter key: accepted, and the research knobs 151..173 unchanged."""
import io

import numpy as np
import pytest

import match_ref
import q95_cases as C
import stream_audit
from conftest import golden_bytes
from oracle.harness import sys_decompress

pytestmark = pytest.mark.gpu

MIB = 1 << 20


def _rb():
    import rust_brotli_b200 as rb
    return rb


class _options:
    """Encoder options for the duration of a block (the session encoder is shared by every test)."""

    def __init__(self, encoder, **opts):
        rb = _rb()
        self.encoder = encoder
        names = {"q9_5": rb._native.OPT_Q9_5, "use_dict": rb._native.OPT_DICT, "ctx_model": rb._native.OPT_CTX_MODEL}
        self.opts = [(names[k], v) for k, v in opts.items()]

    def __enter__(self):
        for o, v in self.opts:
            self.encoder.set_option(o, v)

    def __exit__(self, *a):
        for o, _ in self.opts:
            self.encoder.set_option(o, 0 if o == _rb()._native.OPT_Q9_5 else 1)


def test_reference_pin_random_then_unicode():
    """src/bin/integration_tests.rs:399,432-434: 129 715 B; here within +0.5 %."""
    rb = _rb()
    d = golden_bytes("random_then_unicode")
    sink = io.BytesIO()
    w = rb.CompressorWriter(sink, 4096, params=rb.BrotliEncoderParams(quality=11, lgwin=22, size_hint=2 * MIB, q9_5=True))
    for i in range(0, len(d), 4096):
        w.write(d[i:i + 4096])
    w.close()
    c = sink.getvalue()
    assert sys_decompress(c, len(d)) == d
    assert len(c) <= 130_364, len(c)
    print("random_then_unicode q11 + Q9_5: %d B (reference 129 715 B, %+.3f %%)" % (len(c), (len(c) - 129715) / 1297.15))


@pytest.fixture(scope="module")
def case_inputs():
    return {}


@pytest.mark.parametrize("name", list(C.CASES))
def test_device_equals_model_golden(encoder, case_inputs, name):
    inp, q, w, hint, kw = C.CASES[name]
    if inp not in case_inputs:
        case_inputs.clear()  # one input at a time
        case_inputs[inp] = C.inputs(inp)
    d = case_inputs[inp]
    with _options(encoder, q9_5=1, **kw):
        c = encoder.compress_range(d, 0, len(d), q, w, True, True, False, size_hint=hint)
    assert sys_decompress(c, len(d)) == d, name
    assert C.sha(c) == C.GOLDEN[name], "%s: device stream differs from the CPU model (%d B)" % (name, len(c))


@pytest.fixture(scope="module")
def inputs():
    from tools import datagen
    return {"text": datagen.enwik_like(400_000), "json": datagen.json_logs(400_000), "random": datagen.pcg_random(400_000),
            "alice": golden_bytes("alice29.txt")}


def _sample(n, k, seed=5):
    return np.random.default_rng(seed).integers(0, n, k)


def _match_ref(cfg, d, q, w, hint, start, length, query):
    """match_ref.match_ref with the hasher rule cfg (match_ref.config, or C.hasher_q95)."""
    orig = match_ref.config
    match_ref.config = cfg
    try:
        return match_ref.match_ref(d, q, w, hint, start, length, query=query)
    finally:
        match_ref.config = orig


def _check_match(encoder, cfg, d, q, w, hint, query=None, on_demand=True, start=0):
    length = len(d) - start
    got = encoder.stage_match(d, q, w, hint, start, length)
    qi = np.arange(start, len(d)) if query is None else np.unique(np.clip(query, start, len(d) - 1))
    diff = match_ref.first_difference(_match_ref(cfg, d, q, w, hint, start, length, qi), got[qi - start], qi)
    assert diff is None, "q%d lgwin %d hint %d n=%d: device vs brute force: %s" % (q, w, hint, len(d), diff)
    if on_demand:
        od = encoder.stage_match(d, q, w, hint, start, length, on_demand=True)
        diff = match_ref.first_difference(got, od, np.arange(start, len(d)))
        assert diff is None, "q%d lgwin %d: on-demand search vs up-front kernels: %s" % (q, w, diff)
    return got


@pytest.mark.parametrize("q", [5, 7, 8])
def test_q95_selects_h6_above_1MiB_at_quality_5_to_8(encoder, inputs, q):
    """1 MiB < size hint <= 4 MiB, lgwin >= 19: H6 with Q9_5, H5 without."""
    d = inputs["text"]
    hint = 2 * MIB
    assert C.hasher_q95(q, 22, hint)[0] == 6 and match_ref.config(q, 22, hint)[0] == 5
    query = np.concatenate([np.arange(3000), _sample(len(d), 30_000)])
    plain = _check_match(encoder, match_ref.config, d, q, 22, hint, query=query, on_demand=False)
    with _options(encoder, q9_5=1):
        h6 = _check_match(encoder, C.hasher_q95, d, q, 22, hint, query=query, on_demand=q >= 7)
    assert not np.array_equal(plain, h6)


@pytest.mark.parametrize("hint", [MIB, 2 * MIB])
def test_depth512_match_stage(encoder, inputs, hint):
    """Quality 11 + Q9_5 at lgwin 22: H5 (hint <= 1 MiB) or H6 with 512-deep buckets, k_match_deep<512> and the on-demand
    search against the brute force, on planted edges, text, JSON logs and random bytes."""
    assert C.hasher_q95(11, 22, hint)[2] == 512
    with _options(encoder, q9_5=1):
        d, marks = match_ref.planted_input(22, with_positions=True)
        maxb = (1 << 22) - 16
        query = np.concatenate([marks, np.arange(maxb - 64, maxb + 4096), np.arange(len(d) - 300, len(d)), _sample(len(d), 20_000)])
        _check_match(encoder, C.hasher_q95, d, 11, 22, hint, query=query)
        for name in ("alice", "text", "json", "random"):
            x = inputs[name]
            query = None if name == "random" else np.concatenate([np.arange(2000), np.arange(len(x) - 2000, len(x)), _sample(len(x), 12_000)])
            _check_match(encoder, C.hasher_q95, x, 11, 22, hint, query=query)


def test_depth512_two_sort_batches(encoder):
    """A 24 MiB chunk at lgwin 24 takes two sort batches (the second starts at 16 773 120): up-front kernels only."""
    from tools import datagen
    big = datagen.enwik_like(24 * MIB, seed=6)
    seam = (1 << 25) - (1 << 24) - 4096
    pl, marks = match_ref.planted_input(16, with_positions=True)
    at = seam - 150_000
    d = big[:at] + pl + big[at + len(pl):]
    query = np.concatenate([np.arange(seam - 10_000, seam + 10_000), np.arange(len(d) - 5_000, len(d)), marks + at,
                            _sample(len(d), 15_000)])
    with _options(encoder, q9_5=1):
        _check_match(encoder, C.hasher_q95, d, 11, 24, 0, query=query, on_demand=False)
        with pytest.raises(RuntimeError):  # the on-demand path needs the chunk in one batch
            encoder.stage_match(d, 11, 24, on_demand=True)


@pytest.mark.parametrize("q", [10, 11])
def test_entropy_stage_audit(encoder, q):
    """Every metablock of a 9.5 stream read back (the audit decodes every command and distance code against the input): the
    quality 10 / 11 metablock structure -- ChooseContextMode's UTF8 / SIGNED modes, clustered context maps, block switches --
    on the hash-chain commands."""
    from tools import datagen
    d = datagen.json_logs(3_000_000) + golden_bytes("alice29.txt") * 8
    with _options(encoder, q9_5=1):
        c = encoder.compress_range(d, 0, len(d), q, 22, True, True, False)
    c10 = encoder.compress_range(d, 0, len(d), q, 22, True, True, False)
    assert c != c10
    _, mbs = stream_audit.audit(c, d)
    comp = [m for m in mbs if not m.raw]
    assert len(comp) >= 2
    for mb in comp:
        assert set(mb.cmodes) <= {2, 3}, mb.cmodes  # CONTEXT_UTF8 / CONTEXT_SIGNED
        assert len(mb.lit_cmap) == 64 * mb.ntypes[0] and len(mb.dist_cmap) == 4 * mb.ntypes[2]
        assert mb.cmds and all(cm[5] < mb.dist_alphabet for cm in mb.cmds)
    assert any(max(mb.ntypes) > 1 for mb in comp), "no block switch in any metablock"
    assert any(mb.nlit_trees > 1 for mb in comp), "no clustered literal context map"
    assert sys_decompress(c10, len(d)) == d


def test_every_entry_point_same_bytes(encoder):
    import torch
    rb = _rb()
    from tools import datagen
    d = datagen.json_logs(2_500_000) + datagen.enwik_like(1_500_000)
    for q in (10, 11):
        p = rb.BrotliEncoderParams(quality=q, lgwin=22, q9_5=True)
        s = rb._Stream(p)
        try:
            ref = s.step(d, rb.BROTLI_OPERATION_FINISH)
        finally:
            s.close()
        assert sys_decompress(ref, len(d)) == d
        with _options(encoder, q9_5=1):
            assert ref == encoder.compress_range(d, 0, len(d), q, 22, True, True, False)
        t = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
        out, size = rb.compress_tensor(t, params=p, encoder=encoder)
        assert bytes(out[:size.item()].cpu().numpy()) == ref, "compress_tensor(params=)"
        sink = io.BytesIO()
        w = rb.CompressorWriter(sink, 4096, params=p)
        w.write(d)
        w.close()
        assert sink.getvalue() == ref, "CompressorWriter"
        # a FLUSH sequence: the host stream and the device stream
        pieces = [(0, 700_000), (700_000, 1_900_000)]
        s = rb._Stream(p)
        try:
            host = b"".join(s.step(d[a:b], rb.BROTLI_OPERATION_FLUSH) for a, b in pieces)
            host += s.step(d[1_900_000:], rb.BROTLI_OPERATION_FINISH)
        finally:
            s.close()
        ds = rb.DeviceStreamEncoder(p, encoder=encoder)
        try:
            for a, b in pieces:
                ds.flush(t[a:b])
            ds.finish(t[1_900_000:])
            o, sz, _ = ds.output()
            dev = bytes(o[:sz.item()].cpu().numpy())
        finally:
            ds.close()
        assert dev == host, "DeviceStreamEncoder vs BrotliEncoderCompressStream over FLUSH"
        assert sys_decompress(host, len(d)) == d
        multi = rb.compress_multi(p, d, 3)
        assert sys_decompress(multi, len(d)) == d


def test_graph_capture_after_reserve():
    import torch
    rb = _rb()
    from tools import datagen
    d = datagen.enwik_like(1_200_000)
    enc = rb.DeviceEncoder(0)
    try:
        t = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
        p = rb.BrotliEncoderParams(quality=11, lgwin=22, q9_5=True)
        enc.reserve(11, 22, len(d))
        ref_out, ref_size = rb.compress_tensor(t, params=p, encoder=enc)
        ref = bytes(ref_out[:ref_size.item()].cpu().numpy())
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                out, size = rb.compress_tensor(t, params=p, encoder=enc)
        g.replay()
        torch.cuda.synchronize()
        assert bytes(out[:size.item()].cpu().numpy()) == ref
        assert sys_decompress(ref, len(d)) == d
    finally:
        enc.close()


def test_parameter_keys():
    """Q9_5 is accepted and acts; the research knobs 151..173 (other than the framing keys) are accepted and change nothing."""
    rb = _rb()
    d = golden_bytes("alice29.txt")

    def stream(kv):
        s = rb._Stream(rb.BrotliEncoderParams(quality=11, lgwin=22))
        try:
            for k, v in kv:
                assert s.L.BrotliEncoderSetParameter(s.h, k, v), (k, v)
            return s.step(d, rb.BROTLI_OPERATION_FINISH)
        finally:
            s.close()

    plain = stream([])
    q95 = stream([(rb.BROTLI_PARAM_Q9_5, 1)])
    assert q95 != plain and sys_decompress(q95, len(d)) == d
    assert C.sha(q95) == C.GOLDEN["alice-q11-w22"]
    assert stream([(rb.BROTLI_PARAM_Q9_5, 1), (rb.BROTLI_PARAM_Q9_5, 0)]) == plain
    framing = {167, 168, 169, 170, 172, 173}
    for k in range(151, 174):
        if k not in framing:
            assert stream([(k, 1)]) == plain, k

"""CPU: the framing rule every entry point runs (BrotliEncoderCompress / CompressStream / CompressMulti on the host,
b200_encoder_compress_params_async and the device stream), b200_stage_framed_plan, against a Python restatement: the prologue's
bits (window bits, magic-number metadata block, catable's uncompressed metablock, the empty trailer), the first / last /
byte_align flags of each device call, the trailer byte, and how a body is cut into pieces of at most 1 GiB, each handed over
from a base at most one window in front of it.  The hook does no arithmetic on data, so multi-GiB ranges cost nothing."""
import pytest

import rust_brotli_b200 as rb
from rust_brotli_b200 import _native

GiB = 1 << 30
PIECE = GiB  # positions inside the device encoder are 32-bit: a call compresses at most this many bytes


class Params:
    """EncoderParams after apply_param, and SanitizeParams (encode.rs:559-568)."""

    def __init__(self, lgwin, size_hint, flags):
        self.lgwin, self.size_hint = lgwin, size_hint
        self.catable = rb.BROTLI_PARAM_CATABLE in flags
        self.appendable = self.catable or rb.BROTLI_PARAM_APPENDABLE in flags
        self.magic = rb.BROTLI_PARAM_MAGIC_NUMBER in flags
        self.bare = rb.BROTLI_PARAM_BARE_STREAM in flags
        self.byte_align = self.bare or (self.appendable and rb.BROTLI_PARAM_BYTE_ALIGN in flags)
        self.lw = min(max(lgwin, 10), 24)

    def framed(self):
        return self.catable or self.appendable or self.magic or self.byte_align or self.bare


class Bits:
    """LSB-first bit writer."""

    def __init__(self):
        self.v, self.pos = 0, 0

    def put(self, n, v):
        self.v |= (v & ((1 << n) - 1)) << self.pos
        self.pos += n

    def align(self):
        self.pos = (self.pos + 7) & ~7

    def bytes(self, data):
        for x in data:
            self.put(8, x)

    def out(self):
        return self.v.to_bytes(self.pos >> 3, "little")


def write_prologue(w, p, length):
    """[window bits unless catable && bare] [magic-number metadata metablock] [catable: the first min(2, length) bytes as an
    uncompressed metablock, zeros in their place]; returns (data_off, n2)."""
    if not (p.catable and p.bare):  # EncodeWindowBits, no large window
        if p.lw == 16:
            w.put(1, 0)
        elif p.lw == 17:
            w.put(7, 1)
        elif p.lw > 17:
            w.put(4, ((p.lw - 17) << 1) | 1)
        else:
            w.put(7, ((p.lw - 8) << 4) | 1)
    if p.magic:
        sh, v = [], p.size_hint  # base 128, least significant group first
        while True:
            sh.append(v & 0x7F)
            v >>= 7
            if not v:
                break
            sh[-1] |= 0x80
        w.put(1, 0), w.put(2, 3), w.put(1, 0), w.put(2, 1), w.put(8, 3 + len(sh))  # ISLAST 0, MNIBBLES 0, reserved, MSKIPBYTES 1
        w.align()
        w.bytes([0xE1, 0x97, 0x81 if p.catable else (0x82 if p.appendable else 0x80), 1])
        w.bytes(sh)
    if p.catable and length:
        n2 = min(2, length)
        w.put(1, 0), w.put(2, 0), w.put(16, n2 - 1), w.put(1, 1)  # ISLAST 0, MNIBBLES 4, MLEN - 1, ISUNCOMPRESSED
        w.align()
        data_off = w.pos >> 3
        w.bytes([0] * n2)
        return data_off, n2
    return 0, 0


def write_empty_trailer(w, p, last, align_end):
    if last:
        if p.byte_align and w.pos & 7:
            w.put(6, 6), w.align()  # padding metablock
        if not p.bare:
            w.put(2, 3), w.align()  # ISLAST + ISLASTEMPTY
    elif align_end and w.pos & 7:
        w.put(6, 6), w.align()


def span_calls(p, a, b, first, last, align_end):
    """The pieces of [a, b): at most PIECE bytes each, the first with the header, the last with the stream's end, every other one
    ending byte aligned.  An empty range still makes one call."""
    window = (1 << p.lw) + 65536
    calls, s = [], a
    while True:
        e = min(b, s + PIECE)
        rebase = (s - window) & ~4095 if s > window else 0  # a full window in front: min(pos, 2^lgwin - 16) is unchanged
        l = e == b
        calls.append((rebase, s, e, first and s == a, last and l, (align_end and not last) if l else True))
        if l:
            return calls
        s = e


def restated_plan(p, a, b, first, last, align_end):
    """(prologue, calls, trailer) as the shared rule lays out input [a, b), or None for a framing that cannot end byte aligned."""
    if not p.framed():
        return None, span_calls(p, a, b, first, last, align_end), -1
    w = Bits()
    prologue = (first and (p.magic or p.catable)) or a == b
    data_off = n2 = 0
    if first and prologue:
        data_off, n2 = write_prologue(w, p, b - a)
    body_a = a + n2
    dev_last = last and not p.byte_align and not p.bare  # the device writes the plain 2-bit trailer itself
    dev_align = p.byte_align if last else align_end
    calls = span_calls(p, body_a, b, first and not prologue, dev_last, dev_align)
    if body_a == b:  # nothing (left) to compress: the trailer follows the prologue, which is the whole output
        write_empty_trailer(w, p, last, align_end)
        return None if w.pos & 7 else ((w.out(), data_off, n2, True), calls, -1)
    if w.pos & 7:
        return None
    return ((w.out(), data_off, n2, False) if prologue else None), calls, 3 if last and p.byte_align and not p.bare else -1


def kv(lgwin, size_hint, flags):
    return [(rb.BROTLI_PARAM_QUALITY, 5), (rb.BROTLI_PARAM_LGWIN, lgwin)] + \
        ([(rb.BROTLI_PARAM_SIZE_HINT, size_hint)] if size_hint else []) + [(f, 1) for f in flags]


FLAGS = [(), (rb.BROTLI_PARAM_CATABLE,), (rb.BROTLI_PARAM_APPENDABLE,), (rb.BROTLI_PARAM_MAGIC_NUMBER,),
         (rb.BROTLI_PARAM_APPENDABLE, rb.BROTLI_PARAM_BYTE_ALIGN), (rb.BROTLI_PARAM_BYTE_ALIGN,), (rb.BROTLI_PARAM_BARE_STREAM,),
         (rb.BROTLI_PARAM_CATABLE, rb.BROTLI_PARAM_BARE_STREAM),
         (rb.BROTLI_PARAM_MAGIC_NUMBER, rb.BROTLI_PARAM_CATABLE), (rb.BROTLI_PARAM_CATABLE, rb.BROTLI_PARAM_BYTE_ALIGN)]
LENGTHS = [0, 1, 2, 3, 4096, GiB - 1, GiB, GiB + 1, GiB + 3, 3 * GiB + 17]
SIZE_HINTS = [0, 127, 128, (1 << 32) - 1]  # base-128 size hint of 1, 2 and 5 groups (SIZE_HINT is a 32-bit value)


def check(params, p, a, b, first, last, align_end):
    got = _native.framed_plan(params, a, b, first, last, align_end)
    want = restated_plan(p, a, b, first, last, align_end)
    assert got == want, (a, b, first, last, align_end)
    if got is None:
        return
    prologue, calls, _ = got
    window = (1 << p.lw) + 65536
    body_a = a + (prologue[2] if prologue else 0)
    assert calls[0][1] == body_a and calls[-1][2] == b
    for (rebase, s, e, *_), nxt in zip(calls, calls[1:] + [None]):
        assert 0 <= e - s <= PIECE
        assert rebase % 4096 == 0 and rebase <= s <= rebase + window + 4095
        assert nxt is None or nxt[1] == e  # no gap, no overlap


@pytest.mark.parametrize("flags", FLAGS, ids=lambda f: "+".join(str(x) for x in f) or "plain")
def test_plan_matches_restated_rule(flags):
    for lgwin in (10, 16, 22, 24):
        window = (1 << lgwin) + 65536
        for size_hint in SIZE_HINTS:
            params, p = kv(lgwin, size_hint, flags), Params(lgwin, size_hint, flags)
            for a in (0, 5, window + 1, 3 * GiB):
                for n in LENGTHS:
                    for bits in range(8):
                        check(params, p, a, a + n, bool(bits & 1), bool(bits & 2), bool(bits & 4))


def test_lgwin_is_clamped():
    """LGWIN outside 10..24 is accepted and runs as the nearest bound: window bits and rebase window both."""
    for lgwin in (0, 9, 25, 30):
        for flags in FLAGS:
            p = Params(lgwin, 0, flags)
            for a, n in ((0, 0), (0, 3), (5 << 20, GiB + 1)):
                check(kv(lgwin, 0, flags), p, a, a + n, True, True, False)


def test_streams_use_the_whole_plan():
    """A framed stream's prologue is at most 24 bytes; a stream of at most two bytes is prologue and trailer alone."""
    flags = (rb.BROTLI_PARAM_MAGIC_NUMBER, rb.BROTLI_PARAM_CATABLE)
    pro, calls, trailer = _native.framed_plan(kv(24, (1 << 32) - 1, flags), 0, 2, True, True, True)
    assert pro[3] and len(pro[0]) <= 24 and calls == [(0, 2, 2, False, True, False)] and trailer == -1
    pro, calls, trailer = _native.framed_plan(kv(22, 0, (rb.BROTLI_PARAM_CATABLE, rb.BROTLI_PARAM_BYTE_ALIGN)), 0, 3, True, True, True)
    assert not pro[3] and pro[1:3] == (3, 2) and calls == [(0, 2, 3, False, False, True)] and trailer == 3


def test_refusals():
    assert _native.framed_plan([(rb.BROTLI_PARAM_LARGE_WINDOW, 1)], 0, 10, True, True, False) is None
    assert _native.framed_plan([(rb.BROTLI_PARAM_LGBLOCK, 3)], 0, 10, True, True, False) is None
    assert len(_native.framed_plan(kv(22, 0, ()), 0, 3 * GiB + 17, True, True, False)[1]) == 4
    assert _native.framed_plan(kv(22, 0, ()), 0, 3 * GiB + 17, True, True, False, max_calls=3) is None
    # an empty appendable stream that neither ends nor ends byte aligned would stop inside a byte
    assert _native.framed_plan(kv(22, 0, (rb.BROTLI_PARAM_APPENDABLE,)), 0, 0, True, False, False) is None

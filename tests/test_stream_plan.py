"""CPU: the stream rule BrotliEncoderCompressStream and the device stream (b200_stream_*) share, b200_stage_stream_start /
b200_stage_stream_plan, against a Python restatement of the host state machine: which byte ranges become output at each
PROCESS / FLUSH / FINISH, their framing, size hint and window base, the end-of-stream bytes, and the custom dictionary rule."""
import itertools

import pytest

import rust_brotli_b200 as rb
from rust_brotli_b200 import _native

MiB = 1 << 20
PIECE = 96 * MiB  # four 24 MiB chunks
PROCESS, FLUSH, FINISH, EMIT_METADATA = 0, 1, 2, 3


class HostStream:
    """BrotliEncoderCompressStream's bookkeeping (csrc/bro_capi.cu), restated: input is buffered, PROCESS emits a 96 MiB piece
    whenever two are pending, FLUSH / FINISH emit everything pending, and the bytes kept in front of the unflushed part are
    trimmed to 2^lgwin + 64 KiB, aligned down to 4096."""

    def __init__(self, lgwin=22, size_hint=0, framed=False, bare=False, dict_size=0):
        self.lw = min(max(lgwin, 10), 24)
        self.size_hint, self.framed, self.bare = size_hint, framed, bare
        self.base = self.flushed = self.end = self.dict_len = 0
        self.header = self.finished = False
        self.dict_from = dict_size
        if dict_size > 1:  # the last min(size, 2^lgwin - 16) dictionary bytes sit in front of the stream
            keep = min(dict_size, (1 << self.lw) - 16)
            self.dict_len = self.flushed = self.end = keep
            self.dict_from = dict_size - keep

    def counters(self):
        return (self.base, self.flushed, self.end, self.dict_len, int(self.header), int(self.finished))

    def step(self, op, n):
        """The emits of one step: (start, upto, base, base_after, size_hint, first, last, byte)."""
        out = []
        self.end += n
        hint = self.size_hint or self.end - self.dict_len

        def emit(last, upto):
            start, base, first = self.flushed, self.base, not self.header
            if upto == start and not (self.framed and first):  # nothing to compress
                if last:
                    if first:
                        out.append((start, upto, base, base, hint, first, last, 6))  # the empty stream
                    elif not self.bare:
                        out.append((start, upto, base, base, hint, first, last, 3))  # ISLAST + ISLASTEMPTY
                    self.header = True
                return
            self.flushed, self.header = upto, True
            window = (1 << self.lw) + 65536
            if self.flushed > self.base + window:
                self.base = max(self.base, (self.flushed - window) & ~4095)
            out.append((start, upto, base, self.base, hint, first, last, -1))

        if op == PROCESS:
            while self.end - self.flushed >= 2 * PIECE:
                emit(False, self.flushed + PIECE)
        elif op == FLUSH:
            if self.flushed < self.end:
                emit(False, self.end)
        elif op == FINISH and not self.finished:
            emit(True, self.end)
            self.finished = True
        return out


def kv(lgwin=22, size_hint=0, flags=()):
    return [(rb.BROTLI_PARAM_QUALITY, 5), (rb.BROTLI_PARAM_LGWIN, lgwin)] + ([(rb.BROTLI_PARAM_SIZE_HINT, size_hint)] if size_hint else []) + \
        [(f, 1) for f in flags]


def as_tuple(m):
    return (m.start, m.upto, m.base, m.base_after, m.size_hint, bool(m.first), bool(m.last), m.byte)


def run_sequence(seq, lgwin=22, size_hint=0, flags=(), dict_size=0):
    framed = bool(set(flags) & {rb.BROTLI_PARAM_CATABLE, rb.BROTLI_PARAM_APPENDABLE, rb.BROTLI_PARAM_MAGIC_NUMBER,
                                rb.BROTLI_PARAM_BARE_STREAM})
    host = HostStream(lgwin, size_hint, framed, rb.BROTLI_PARAM_BARE_STREAM in flags, dict_size)
    params = kv(lgwin, size_hint, flags)
    c, dict_from = _native.stream_start(params, dict_size)
    assert dict_from == host.dict_from
    assert (c.base, c.flushed, c.end, c.dict_len, c.header_written, c.finished) == host.counters()
    emitted = 0
    for op, n in seq:
        want = host.step(op, n)
        got = _native.stream_plan(params, c, op, n)
        assert got is not None, (op, n)
        emits, c = got
        assert [as_tuple(m) for m in emits] == want, (op, n)
        assert (c.base, c.flushed, c.end, c.dict_len, c.header_written, c.finished) == host.counters(), (op, n)
        emitted += len(emits)
    return emitted, c


SEQUENCES = {
    "empty": [(FINISH, 0)],
    "process_8mib_runs": [(PROCESS, 8 * MiB)] * 30 + [(FINISH, 0)],
    "one_large_write": [(PROCESS, 250 * MiB + 3), (PROCESS, 1), (FINISH, 0)],
    "write_then_finish": [(FINISH, 300 * MiB)],
    "flush_nothing_pending": [(FLUSH, 0), (PROCESS, 5), (FLUSH, 0), (FLUSH, 0), (FINISH, 0)],
    "finish_after_flush": [(PROCESS, 65537), (FLUSH, 0), (FINISH, 0)],
    "flush_each_write": [(FLUSH, n) for n in (1, 2, 3, 4095, 4096, 65537, MiB, 24 * MiB + 1)] + [(FINISH, 0)],
    "process_exact_threshold": [(PROCESS, 2 * PIECE - 1), (PROCESS, 1), (PROCESS, PIECE), (FLUSH, 7), (FINISH, 0)],
    "finish_twice": [(PROCESS, 100), (FINISH, 0), (FINISH, 0), (FLUSH, 0), (PROCESS, 0)],
}
FLAGS = [(), (rb.BROTLI_PARAM_CATABLE,), (rb.BROTLI_PARAM_APPENDABLE,), (rb.BROTLI_PARAM_MAGIC_NUMBER,),
         (rb.BROTLI_PARAM_APPENDABLE, rb.BROTLI_PARAM_BYTE_ALIGN), (rb.BROTLI_PARAM_BYTE_ALIGN,), (rb.BROTLI_PARAM_BARE_STREAM,),
         (rb.BROTLI_PARAM_CATABLE, rb.BROTLI_PARAM_BARE_STREAM)]


@pytest.mark.parametrize("name", sorted(SEQUENCES))
@pytest.mark.parametrize("flags", FLAGS, ids=lambda f: "+".join(str(x) for x in f) or "plain")
def test_plan_matches_host_state_machine(name, flags):
    for lgwin, dict_size in ((22, 0), (16, 2), (10, 60000)):
        run_sequence(SEQUENCES[name], lgwin=lgwin, flags=flags, dict_size=dict_size)


@pytest.mark.parametrize("dict_size", [0, 1, 2, 3, 1000, (1 << 16) - 16, (1 << 16) - 15, 1 << 20])
@pytest.mark.parametrize("lgwin", [10, 16, 22, 24])
def test_dictionary_rule(dict_size, lgwin):
    for name in ("empty", "flush_each_write", "process_8mib_runs"):
        run_sequence(SEQUENCES[name], lgwin=lgwin, dict_size=dict_size)


def test_size_hint_and_window_trim():
    """SIZE_HINT replaces the running input size; the window base stays a multiple of 4096 at most 2^lgwin + 64 KiB + 4095 bytes
    in front of the unflushed part."""
    _, c = run_sequence([(FLUSH, 3 * MiB + 17)] * 5 + [(FINISH, 0)], lgwin=18, size_hint=12345)
    assert c.base % 4096 == 0 and c.flushed - c.base <= (1 << 18) + 65536 + 4095
    emits, _ = _native.stream_plan(kv(18, 12345), _native.stream_start(kv(18, 12345), 0)[0], FLUSH, 100)
    assert [m.size_hint for m in emits] == [12345]


def test_pieces_are_emitted_before_finish():
    """230 MB in 8 MiB writes: PROCESS emits 96 MiB pieces while input keeps arriving, FINISH the rest."""
    params = kv()
    c, _ = _native.stream_start(params, 0)
    early = []
    for _ in range(230_000_000 // (8 * MiB)):
        emits, c = _native.stream_plan(params, c, PROCESS, 8 * MiB)
        early += emits
    assert [m.upto - m.start for m in early] == [PIECE]
    assert c.end - c.base <= 2 * PIECE + (1 << 22) + 65536 + 4096


def test_refusals():
    params = kv()
    c, _ = _native.stream_start(params, 0)
    assert _native.stream_plan(params, c, EMIT_METADATA, 0) is None
    assert _native.stream_plan(params, c, 7, 0) is None
    _, done = _native.stream_plan(params, c, FINISH, 10)
    assert done.finished
    assert _native.stream_plan(params, done, PROCESS, 1) is None  # input after FINISH
    assert _native.stream_plan(params, done, FINISH, 0)[0] == []  # the host ignores a second FINISH
    with pytest.raises(ValueError):
        _native.stream_start([(rb.BROTLI_PARAM_LARGE_WINDOW, 1)], 0)
    assert _native.stream_plan([(rb.BROTLI_PARAM_LGBLOCK, 3)], c, FLUSH, 0) is None
    # more emits than the caller has room for
    assert _native.stream_plan(params, c, PROCESS, 10 * PIECE, max_emits=2) is None
    emits, _ = _native.stream_plan(params, c, PROCESS, 10 * PIECE, max_emits=16)
    assert len(emits) == 9

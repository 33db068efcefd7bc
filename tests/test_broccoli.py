"""CPU: the Broccoli C ABI (include/broccoli.h, csrc/bro_broccoli.cu over the splice rules of csrc/bro_concat.cuh).

Spliced output must equal the whole-buffer restatement tests/brocatli_ref.py where that applies and decode to the concatenated
inputs; it must not depend on how input and output are cut into buffers; the edge cases follow the reference's lines
(src/concat/mod.rs, src/ffi/broccoli.rs) by hand."""
import ctypes
import os
import subprocess

import pytest

from conftest import golden_bytes
from oracle.harness import sys_decompress

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "rust-brotli_b200")

SYMBOLS = ["BroccoliCreateInstance", "BroccoliCreateInstanceWithWindowSize", "BroccoliDestroyInstance", "BroccoliNewBrotliFile",
           "BroccoliConcatStream", "BroccoliConcatStreaming", "BroccoliConcatFinish", "BroccoliConcatFinished"]


def _window_bits(put, lgwin):  # EncodeWindowBits (encode.rs:600-627)
    if lgwin == 16:
        put(1, 0)
    elif lgwin == 17:
        put(7, 1)
    elif lgwin > 17:
        put(4, ((lgwin - 17) << 1) | 1)
    else:
        put(7, ((lgwin - 8) << 4) | 1)


def _pack(bits):
    bits = bits + [0] * (-len(bits) % 8)
    return bytes(sum(bits[i + j] << j for j in range(8)) for i in range(0, len(bits), 8))


def catable_from_model(model, d, q, lgwin=22, byte_align=False, magic=False):
    """The framing csrc/bro_capi.cu:compress_framed builds around a catable stream, from the CPU model's ranges: window bits,
    [magic-number metadata block], the first two bytes as an uncompressed metablock, the rest without static dictionary, the
    empty last metablock ([padding metablock + 0x03 when byte aligned])."""
    bits = []

    def put(n, v):
        bits.extend((v >> i) & 1 for i in range(n))
    _window_bits(put, lgwin)
    if magic:  # brotli_bit_stream.rs:2855-2896, size hint len(d)
        sh, v = [], len(d)
        while True:
            sh.append(v & 0x7f)
            v >>= 7
            if not v:
                break
            sh[-1] |= 0x80
        put(1, 0); put(2, 3); put(1, 0); put(2, 1); put(8, 3 + len(sh))
        bits.extend([0] * (-len(bits) % 8))
        for byte in bytes([0xe1, 0x97, 0x81, 1]) + bytes(sh):
            put(8, byte)
    n2 = min(2, len(d))
    if n2:
        put(1, 0); put(2, 0); put(16, n2 - 1); put(1, 1)
        bits.extend([0] * (-len(bits) % 8))
        for byte in d[:n2]:
            put(8, byte)
    if len(d) <= 2:
        if byte_align and len(bits) % 8:
            put(6, 6)
            bits.extend([0] * (-len(bits) % 8))
        put(2, 3)
        return _pack(bits)
    head = _pack(bits)
    if byte_align:
        body, _ = model.compress_range(d, 2, len(d) - 2, q, lgwin, False, False, True, use_dict=0)
        return head + body + b"\x03"
    body, _ = model.compress_range(d, 2, len(d) - 2, q, lgwin, False, True, False, use_dict=0)
    return head + body


def splice(streams, in_piece=None, out_piece=1 << 20, window_size=None):
    """Host Broccoli over `streams`: input fed in pieces of `in_piece` bytes, output taken in buffers of `out_piece`.  Returns
    (bytes, code): code is the first result >= 124 (the output so far is then returned) or the final Finish result."""
    import rust_brotli_b200 as rb
    bc = rb.BroCatli() if window_size is None else rb.BroCatli.new_with_window_size(window_size)
    out = bytearray()
    for s in streams:
        bc.new_brotli_file()
        pieces = [s[i:i + in_piece] for i in range(0, len(s), in_piece)] if in_piece else [s]
        for p in pieces or [b""]:
            while True:
                r, used, o = bc.stream(p, out_piece)
                out += o
                p = p[used:]
                if r >= 124:
                    return bytes(out), r
                if r == rb.BROCCOLI_NEEDS_MORE_INPUT and not p:
                    break
                assert r in (rb.BROCCOLI_NEEDS_MORE_INPUT, rb.BROCCOLI_NEEDS_MORE_OUTPUT), r
    while True:
        r, o = bc.finish(out_piece)
        out += o
        if r != rb.BROCCOLI_NEEDS_MORE_OUTPUT:
            return bytes(out), r


@pytest.fixture(scope="module")
def corpus(model):
    """Catable streams of several shapes with their inputs, windows non-increasing in list order."""
    alice, you = golden_bytes("alice29.txt"), golden_bytes("asyoulik.txt")
    cases = [(alice[:40000], 5, 24, {}), (you[:30000], 5, 22, {"byte_align": True}), (alice[1000:9000], 10, 22, {"magic": True}),
             (b"", 5, 20, {}), (b"z", 5, 20, {}), (b"xy", 5, 18, {"byte_align": True}), (you[5000:20000], 9, 18, {}),
             (alice[:3], 5, 16, {}), (alice[7:5007], 5, 16, {"byte_align": True})]
    return [(catable_from_model(model, d, q, w, **kw), d) for d, q, w, kw in cases]


def test_symbols_and_state_layout():
    import rust_brotli_b200 as rb
    assert ctypes.sizeof(rb.BroccoliState) == 256
    L = ctypes.CDLL(os.path.join(LIBDIR, "libbrotli_b200.so"))
    for name in SYMBOLS:
        assert hasattr(L, name), name
    nm = subprocess.run(["nm", "-D", "--defined-only", os.path.join(LIBDIR, "libbrotli_b200.so")], capture_output=True, text=True).stdout
    for name in SYMBOLS:
        assert (" T " + name) in nm, name


def test_whole_buffer_equals_restatement_and_decodes(model, corpus):
    import brocatli_ref as bc
    streams = [s for s, _ in corpus]
    for s, d in corpus:
        assert sys_decompress(s, max(1, len(d))) == d
    out, code = splice(streams)
    assert code == 0
    assert out == bc.concat(streams)
    want = b"".join(d for _, d in corpus)
    assert sys_decompress(out, len(want)) == want
    # a plain (not catable) stream may go first: it is copied as it is
    plain = model.compress(golden_bytes("alice29.txt")[:20000], 5, 24)[0]
    out, code = splice([plain] + streams[1:])
    assert code == 0 and out == bc.concat([plain] + streams[1:])
    want = golden_bytes("alice29.txt")[:20000] + b"".join(d for _, d in corpus[1:])
    assert sys_decompress(out, len(want)) == want
    # magic number first
    out, code = splice([corpus[2][0], corpus[1][0]])
    assert code == 0 and out == bc.concat([corpus[2][0], corpus[1][0]])
    assert sys_decompress(out, len(corpus[2][1]) + len(corpus[1][1])) == corpus[2][1] + corpus[1][1]


@pytest.mark.parametrize("in_piece", [1, 2, 3, 7, 4096])
@pytest.mark.parametrize("out_piece", [1, 2, 5])
def test_streaming_invariance(corpus, in_piece, out_piece):
    """Same bytes and codes for every cut of input and output buffers (the reference's stream() resumes at any byte)."""
    streams = [s for s, _ in corpus[1:6]] + [corpus[7][0]]
    whole = splice(streams)
    assert splice(streams, in_piece=in_piece, out_piece=out_piece) == whole
    bad = [corpus[0][0], golden_bytes("compressed_file")[:50]]  # an error code is reached the same way
    assert splice(bad, in_piece=in_piece, out_piece=out_piece)[1] == splice(bad)[1]


def test_finish_of_empty_instance_is_semicolon():
    """mod.rs:595-602: an instance that never emitted writes ';'; dropped streams emit nothing (mod.rs:750-777)."""
    assert splice([]) == (b";", 0)
    assert splice([b";", b";"]) == (b";", 0)
    assert splice([b""]) == (b";", 0)


def test_short_streams_are_dropped(corpus):
    """mod.rs:31-36, :474-476: a stream shorter than 4 bytes (5 after a first byte 0x11) never gets spliced; the next
    new_brotli_file discards its pending bytes (:274-276), so a dropped first stream lets the next one be first (:345-352)."""
    a = corpus[0][0]
    for short in (b"", b"\x3b", b"\x3b\x00", b"\x01\x02\x03", b"\x11\x02\x03\x04"):
        assert splice([short, a]) == (a, 0)  # the first spliced stream is copied unchanged, finish puts its 1 1 back
        assert splice([a, short]) == (a, 0)
    # 4 bytes after any other first byte are enough to parse; 5 after 0x11
    assert splice([a, b"\x3b\x00\x00\x00"])[1] == 0


def test_tiny_streams_one_to_five_bytes(model):
    """Catable streams of 1..3 input bytes are 5..7 bytes long; spliced, they decode."""
    parts = [catable_from_model(model, d, 5, 22) for d in (b"a", b"bc", b"def", b"ghij")]
    assert [len(p) for p in parts[:2]] == [5, 6]
    out, code = splice(parts)
    assert code == 0
    assert sys_decompress(out, 10) == b"abcdefghij"
    # a 1-byte stream of an empty stream with window 22 (0x3b) and a 5-byte one of an empty uncompressed block
    out, code = splice([parts[0], b"\x3b", parts[1]])
    assert code == 0 and sys_decompress(out, 3) == b"abc"


def test_window_size_instances():
    """broccoli.rs:60-65 / mod.rs:231-272: sizes 0..9 give a default instance; a valid size seeds the bytes of an empty stream of
    that window, which finish writes unchanged; a larger window in a later stream is refused (126, mod.rs:354-356)."""
    import rust_brotli_b200 as rb
    for ws in range(10):
        assert splice([], window_size=ws) == (b";", 0)
        assert rb.BroCatli.new_with_window_size(ws).state_bytes() == rb.BroCatli().state_bytes()
    assert splice([], window_size=22) == (b"\x3b", 0)       # (3 + 4 * 2) | 48
    assert splice([], window_size=16) == (b"\x07", 0)       # 1 | 2 | 4
    assert splice([], window_size=10) == (b"\xa1\x01", 0)   # 0x21 | 0x80, 1
    assert splice([], window_size=25) == (b"\x11\xd9", 0)   # 17, 25 | 64 | 128
    for ws in (10, 16, 22, 25):
        assert rb.BroCatli.new_with_window_size(ws).state_bytes()[11] == ws


def test_window_instance_with_only_dropped_streams_keeps_reference_bytes():
    """mod.rs:567-580 on a two-byte tail: a window-10 instance whose 1 1 sits at bits 7 / 8 is stripped to 7 bits with the
    zero byte behind it kept (:303-324), and append_eof then sets bit 15 of the u16 (bit 16 is lost) and counts 3 bytes, which
    :585-594 writes as lb[0], lb[1], lb[1].  The reference's output is kept, including its shape."""
    assert splice([b""], window_size=10) == (b"\x21\x80\x80", 0)
    assert splice([b""], window_size=22) == (b"\x3b", 0)


def test_error_codes(model, corpus):
    a, a_d = corpus[0]
    b18 = catable_from_model(model, b"window eighteen " * 40, 5, 18)
    b22 = catable_from_model(model, b"window twenty-two " * 40, 5, 22)
    # 127: the second stream's first metablock is compressed (mod.rs:114-116 via :359-366)
    plain = model.compress(golden_bytes("asyoulik.txt")[:5000], 5, 22)[0]
    assert splice([a, plain])[1] == 127
    # 127: the metadata header reaches past the 4 bytes read (mod.rs:387-389; the reference's own case, :779-807)
    assert splice([a, b"\x71\x1b\x00\x00"])[1] == 127
    # 126: a later stream with a larger window (mod.rs:354-356)
    assert splice([b18, b22])[1] == 126
    assert splice([b22, b18])[1] == 0
    # 125: not a window header (mod.rs:63-70 via :338-344)
    assert splice([a, b"\x91\x00\x00\x00\x00"])[1] == 125
    # 124: the previous stream does not end in 1 1 (mod.rs:299-306); reported by the next new stream, even a dropped one
    assert splice([a + b"\x00\x00", b18])[1] == 124
    assert splice([a[:-1] + b"\x02", b""])[1] == 124
    # the last stream's end is not checked: finish writes its bytes as they are (mod.rs:585-594)
    assert splice([a + b"\x00"])[1] == 0


def test_c_client_splices_with_three_byte_buffers(tmp_path, model, corpus):
    exe = str(tmp_path / "broccoli_client")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c_client", "broccoli_client.c"), "-o", exe, "-L", LIBDIR, "-lbrotli_b200",
                           "-Wl,-rpath," + LIBDIR])
    files = []
    for i in (0, 1, 2):
        p = tmp_path / ("in%d.br" % i)
        p.write_bytes(corpus[i][0])
        files.append(str(p))
    out = tmp_path / "out.br"
    r = subprocess.run([exe, str(out)] + files, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = out.read_bytes()
    assert got == splice([s for s, _ in corpus[:3]])[0]
    want = b"".join(d for _, d in corpus[:3])
    assert sys_decompress(got, len(want)) == want

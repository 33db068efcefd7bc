"""CPU: the sequential model of the GPU pipeline (tools/gpu_model.cpp, built from the same host/device headers as the
kernels).  It must produce valid brotli, stay within +0.5 % of the reference restatement, and match its goldens --
the GPU tests then assert that the kernels reproduce these streams bit for bit."""
import hashlib
import os

import pytest

from conftest import assert_size_parity, golden_bytes
from oracle.harness import sys_decompress

FILES = ["alice29.txt", "asyoulik.txt", "random_then_unicode", "quickfox_repeated", "random_org_10k.bin", "backward65536",
         "64x", "ukkonooa", "monkey", "x", "xyzzy", "10x10y", "aaabaaaa", "empty", "quickfox", "compressed_file"]


@pytest.mark.parametrize("name", FILES)
@pytest.mark.parametrize("q,w", [(5, 20), (5, 22), (7, 22), (9, 22), (9, 16), (5, 18), (10, 22), (11, 22), (11, 24), (10, 16)])
def test_model_golden_roundtrip_and_size(model, golden_table, name, q, w):
    d = golden_bytes(name)
    c, _ = model.compress(d, q, w)
    assert sys_decompress(c, len(d)) == d
    g = golden_table["%s|q%d|w%d" % (name, q, w)]
    assert hashlib.sha256(c).hexdigest() == g["model_sha256"]
    assert_size_parity(len(c), g["oracle_size"], "%s q%d w%d" % (name, q, w))


def test_model_against_reference_kats_q10_q11(model):
    """The reference's own exact size vectors for the binary-tree / Zopfli qualities (src/bin/integration_tests.rs:408-449):
    alice29.txt, lgwin 22: quality 10 -> 47 488 B, quality 11 -> 46 493 B.  The pipeline must land within +-0.5 %."""
    d = golden_bytes("alice29.txt")
    for q, pin in ((10, 47488), (11, 46493)):
        c, _ = model.compress(d, q, 22)
        assert sys_decompress(c, len(d)) == d
        assert abs(len(c) - pin) <= pin * 0.005, (q, len(c), pin)


def test_model_hq_options(model):
    """quality 10 / 11 knobs: every variant is a valid stream; the histogram stage (BrotliSplitBlock + context maps) and the
    static dictionary each pay for themselves on English text."""
    d = golden_bytes("asyoulik.txt")
    base = len(model.compress(d, 10, 22)[0])
    for kw in ({"hq_split": 0}, {"use_dict": 0}, {"ctx_model": 0}, {"unit": 65536, "mb_units": 64}, {"depth": 1024}):
        c, _ = model.compress(d, 10, 22, **kw)
        assert sys_decompress(c, len(d)) == d
        if "unit" not in kw and "depth" not in kw:
            assert len(c) > base, kw


@pytest.mark.parametrize("shards", [1, 2, 3, 5])
def test_model_sharded_seams(model, shards):
    """compress_multi split rule (threading/mod.rs:333) with byte-aligned seams: concatenation must decode."""
    d = golden_bytes("random_then_unicode")
    n = len(d)
    parts = []
    for i in range(shards):
        a, b = i * n // shards, (i + 1) * n // shards
        c, _ = model.compress_range(d, a, b - a, 5, 22, i == 0, i + 1 == shards, i + 1 != shards)
        parts.append(c)
    out = b"".join(parts)
    assert sys_decompress(out, n) == d
    if shards == 3:
        assert len(out) <= 144325  # src/bin/test_threading.rs:101 bound for 3 threads q5


@pytest.mark.parametrize("n", [0, 1, 2, 3, 7, 8, 9, 63, 64, 65, 4095, 4096, 4097, 8191, 8192, 12289])
def test_model_edge_sizes(model, n):
    d = (golden_bytes("alice29.txt") * 2)[:n]
    c, _ = model.compress(d, 5, 22)
    assert sys_decompress(c, max(n, 1)) == d


def test_model_options(model):
    d = golden_bytes("asyoulik.txt")
    base, _ = model.compress(d, 5, 22)
    for kw in ({"ctx_model": 0}, {"unit": 2048}, {"unit": 16384}, {"lcap": 32}, {"mb_units": 8}):
        c, _ = model.compress(d, 5, 22, **kw)
        assert sys_decompress(c, len(d)) == d
        assert len(c) < len(base) * 1.03


def test_shipped_parse_windows_equal_sequential_spec(model):
    """The parse kernels resolve a window of G positions with the distance cache of the window start and then walk it with
    straight-line predicated code (G = 8: one unit per warp, q7..q9; G = 2: four units per warp, q5 / q6).  tools/window_emul.cpp
    is that formulation on the CPU; it must reproduce parse_range() command for command, for both window sizes.  G = 2 needs
    more windows than G = 8; measured on these inputs: 1.10x (compressed_file, q5..q7) to 1.71x (random_then_unicode, q9),
    1.33x on alice29."""
    import ctypes
    import subprocess
    import numpy as np
    from conftest import assert_size_parity, golden_bytes
    from tools.model_harness import EncParams
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = os.path.join(root, "tools", "libwindow_emul.so")
    src = os.path.join(root, "tools", "window_emul.cpp")
    if not os.path.exists(so) or os.path.getmtime(src) > os.path.getmtime(so):
        subprocess.check_call(["g++", "-O2", "-fwrapv", "-std=c++17", "-shared", "-fPIC", "-w", "-I",
                               os.path.join(root, "rust-brotli_b200", "csrc"), src, "-o", so])
    L = ctypes.CDLL(so)
    L.window_emul_check.argtypes = [ctypes.POINTER(EncParams), ctypes.c_char_p, ctypes.c_void_p, ctypes.c_uint32,
                                    ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64)]
    for name in ("alice29.txt", "random_then_unicode", "compressed_file", "quickfox_repeated"):
        d = golden_bytes(name)
        for q in (5, 6, 7, 9):  # q7 / q9: 10 / 16 cache candidates, the H9 scores, the 512-byte literal-spree window
            p = model.params(q, 22, len(d), len(d))
            best = np.zeros(len(d) + 1, dtype=np.uint32)
            model.compress(d, q, 22, best_out=best.ctypes.data)
            w2, w8 = ctypes.c_uint64(0), ctypes.c_uint64(0)
            bad = L.window_emul_check(ctypes.byref(p), d + bytes(512), best.ctypes.data, len(d), ctypes.byref(w2), ctypes.byref(w8))
            assert bad == 0, (name, q)
            assert w2.value <= w8.value * 1.75  # G = 2 costs at most 3/4 more windows


def test_model_two_chunks_roundtrip(model):
    """Streams longer than one 24 MiB chunk: the chunk loop (shared with the device encoder) appends independent chunks to one
    bit stream; matches may reach back across the seam (left halo), nothing may read across it to the right."""
    from tools import datagen
    d = datagen.enwik_like(26_000_000, seed=11)
    c, st = model.compress(d, 5, 22)
    assert st.num_metablocks == 7  # 6 in the first chunk, 1 in the second
    assert sys_decompress(c, len(d)) == d
    assert len(c) < 0.36 * len(d)


def test_model_structured_logs_within_half_percent_of_reference_restatement(model, oracle):
    """The 256-byte warm-up in front of every parse unit keeps record-structured input at reference size
    (+1.4 % without it, DESIGN.md section 2)."""
    from tools import datagen
    d = datagen.json_logs(4_000_000)
    for q in (5, 9):
        c = model.compress(d, q, 22)[0]
        assert sys_decompress(c, len(d)) == d
        assert len(c) <= len(oracle.compress(d, q, 22)[0]) * 1.005


def test_model_static_dictionary_reaches_libbrotlienc_on_english(model):
    """Config 1 (alice29, q5, lgwin 20): with static-dictionary matches the size is within 0.5 % of Google's encoder, whose
    code the reference is a port of (52 809 B); without them it is 0.7 % larger."""
    from oracle.harness import sys_compress
    d = golden_bytes("alice29.txt")
    on = model.compress(d, 5, 20)[0]
    off = model.compress(d, 5, 20, use_dict=0)[0]
    ref = len(sys_compress(d, 5, 20))
    assert sys_decompress(on, len(d)) == d and sys_decompress(off, len(d)) == d
    assert len(on) <= ref * 1.005 < len(off)


def _catable_from_model(model, d, q, lgwin=22, byte_align=False):
    """The framing csrc/bro_capi.cu:compress_framed builds around a catable stream, assembled here from the CPU model's ranges:
    window bits, the first two bytes as an uncompressed metablock, the rest without static dictionary, empty last metablock."""
    bits = []
    def put(n, v):
        bits.extend((v >> i) & 1 for i in range(n))
    put(4, ((lgwin - 17) << 1) | 1)
    n2 = min(2, len(d))
    if n2:
        put(1, 0); put(2, 0); put(16, n2 - 1); put(1, 1)
        bits.extend([0] * (-len(bits) % 8))
        for byte in d[:n2]:
            put(8, byte)
    head = bytes(sum(bits[i + j] << j for j in range(8)) for i in range(0, len(bits) - len(bits) % 8, 8))
    if len(d) <= 2:
        tail_bits = bits[len(head) * 8:] + [1, 1]
        tail_bits += [0] * (-len(tail_bits) % 8)
        return head + bytes(sum(tail_bits[i + j] << j for j in range(8)) for i in range(0, len(tail_bits), 8))
    if byte_align:
        body, _ = model.compress_range(d, 2, len(d) - 2, q, lgwin, False, False, True, use_dict=0)
        return head + body + b"\x03"
    body, _ = model.compress_range(d, 2, len(d) - 2, q, lgwin, False, True, False, use_dict=0)
    return head + body


@pytest.mark.parametrize("q", [5, 10])
def test_catable_framing_stitches_like_brocatli(model, q):
    """Streams framed as BROTLI_PARAM_CATABLE asks (encode.rs:2285-2333) go through the restated BroCatli splice
    (tests/brocatli_ref.py, src/concat/mod.rs) and decode to the concatenated inputs; a plain stream is refused by it."""
    import brocatli_ref as bc
    a, b = golden_bytes("alice29.txt")[:40000], golden_bytes("asyoulik.txt")[:30000]
    sa, sb, se, s1 = (_catable_from_model(model, a, q), _catable_from_model(model, b, q, byte_align=True),
                      _catable_from_model(model, b"", q), _catable_from_model(model, b"z", q))
    for s, d in ((sa, a), (sb, b), (se, b""), (s1, b"z")):
        assert sys_decompress(s, max(1, len(d))) == d
    whole = bc.concat([sa, sb, se, s1, sa])
    assert sys_decompress(whole, 2 * len(a) + len(b) + 1) == a + b + b"z" + a
    with pytest.raises(bc.NotCraftedForConcatenation):
        bc.concat([sa, model.compress(b, q, 22)[0]])
    assert bc.window_bits(sa) == (22, 4)


@pytest.mark.parametrize("q", [10, 11])
def test_model_hq_matches_equal_brute_force(model, q):
    """The all-matches stage of quality 10 / 11 against tests/hq_ref.py, a numpy restatement of its contract (short distances,
    256-deep 4-byte buckets, 1024-deep 8 / 16 / 32-byte levels, Pareto fronts of the 8 longest): every window entry of every
    position must agree.  Inputs: planted copies at the distance / length edges, text and JSON logs, and a two-byte period that
    fills every bucket to its depth."""
    import hq_ref
    from tools import datagen
    alice = golden_bytes("alice29.txt")
    cases = [(hq_ref.planted_input(10), 10), (hq_ref.planted_input(16), 16), (alice[:60000], 16), (alice[:30000], 12),
             (datagen.json_logs(40000), 12 if q == 10 else 16), (b"ab" * 6000, 10), (b"ab" * 6000 + alice[:3000], 16)]
    for d, w in cases:
        cnt, ent = hq_ref.hq_ref(d, q, w)
        hqn, hqm, _, _, _ = model.stage_hq(d, q, w)
        got = hq_ref.window_part(hqn, hqm)
        diff = hq_ref.first_difference(cnt, ent, *got)
        assert diff is None, "n=%d lgwin=%d: %s" % (len(d), w, diff)
        assert cnt.sum() > 10000  # the inputs are full of matches: the comparison is not vacuous


@pytest.mark.parametrize("q", [10, 11])
@pytest.mark.parametrize("n", [0, 1, 2, 3, 7, 8, 9, 39, 40, 41, 63, 64, 65, 511, 512, 513, 8191, 8192, 8193, 16383, 16385, 70001])
def test_model_hq_edge_sizes(model, q, n):
    """quality 10 / 11 around every size that switches something on: 8 bytes (first bucket match), 8 + 8 / 16 / 32 bytes (the
    long-prefix levels), the 512-byte warm-up, one and more 2 KiB parse units (the default up to 256 KiB), the 64 KiB
    statistics window."""
    d = (golden_bytes("alice29.txt") * 2)[:n]
    c, _ = model.compress(d, q, 22)
    assert sys_decompress(c, max(n, 1)) == d


def test_model_entropy_stage_equals_float64_reference(model):
    """The entropy stage of the model's streams against tests/entropy_ref.py, read back symbol by symbol through
    tests/stream_audit.py: literal context decision and greedy block split (float64, guided replay), every prefix code
    (recount -> smoothing -> length-limited Huffman exactly, Kraft, optimality gap), every command and distance code.
    Measured on these inputs (same on the device): of 3 124 splitter decisions 19 fall inside the bound on their Q16 error
    -- 12 of 394 in the 8 MiB case, whose histograms reach millions of counts, 5 of 160 in fibonacci-30, one each in
    type-cap-complex13 and hint-1MiB-q7, none elsewhere -- and none of them went against float64.  The largest
    Q16-vs-float64 margin error is 8.6 bits (8 MiB case; 3.1 bits in fibonacci-30, under 1.7 bits elsewhere), always within
    its bound.  No context decision was ambiguous.  The Kraft repair was reached by 7 codes (unlimited depth up to 20) and
    cost at most 0.09 % over the package-merge optimum (1 571 bits on a 4 MiB metablock; 0, 2, 59, 325 and 995 bits for
    the others)."""
    import entropy_ref as er
    from tools import datagen
    cases = er.planted_cases(golden_bytes, datagen, big=True) + er.hq_cases(golden_bytes, datagen)
    total = er.new_report()
    for name, d, q, w, hint in cases:
        c, _ = model.compress(d, q, w, size_hint=hint)
        r = er.audit_stream(c, d, q, hint)
        for k in ("decisions", "ambiguous", "repaired", "new", "second", "merge"):
            total[k] += r[k]
        total["max_margin_error"] = max(total["max_margin_error"], r["max_margin_error"])
        total["gaps"] += r["gaps"]
        if name == "type-cap":
            assert r["new"] >= 255, r
        if name == "type-cap-complex13":
            assert r["maps"] == {"complex-13": 1} and r["new"] >= 19, r
    assert total["repaired"] >= 5 and total["second"] > 100 and total["ambiguous"] < total["decisions"] // 20, total
    print({k: v for k, v in total.items() if k != "gaps"}, "repair gaps", total["gaps"])


def _model_best(model, d, q, w, hint=0, start=0, length=None):
    import numpy as np
    length = len(d) - start if length is None else length
    best = np.zeros(length + 1, dtype=np.uint32)
    model.compress_range(d, start, length, q, w, True, True, False, size_hint=hint, best_out=best.ctypes.data)
    return best[:length]


def test_model_match_stage_equals_brute_force(model):
    """best[] of quality 5..9 (the model's sequential bucket rings) against tests/match_ref.py, a numpy restatement of the
    stage's contract that shares no code with the kernels' headers: every hasher / key width / depth of ChooseHasher, planted
    edges at lgwin 10, 12, 16 and 22, English text (dictionary words) and ranges whose window lies in front of them."""
    import numpy as np
    import match_ref
    alice = golden_bytes("alice29.txt")[:40000]
    mib = 1 << 20
    cases = [(alice, q, w, h) for q, w, h in ((5, 22, mib), (5, 22, 2 * mib), (5, 22, 8 * mib), (6, 22, mib), (6, 22, 8 * mib),
                                              (7, 22, 2 * mib), (7, 22, 8 * mib), (8, 22, mib), (9, 22, mib), (5, 16, 0), (8, 16, 0),
                                              (6, 10, 0), (6, 12, 0))]
    cases += [(match_ref.planted_input(10), 6, 10, 0), (match_ref.planted_input(12), 6, 12, 0), (match_ref.planted_input(16), 5, 16, 0),
              (match_ref.planted_input(16), 9, 16, 0)]
    seen = set()
    for d, q, w, h in cases:
        ref = match_ref.match_ref(d, q, w, h)
        diff = match_ref.first_difference(ref, _model_best(model, d, q, w, h))
        assert diff is None, "q%d lgwin %d hint %d n=%d: %s" % (q, w, h, len(d), diff)
        seen.add(match_ref.config(q, w, h or len(d)))
        assert (ref & 0x80).any() and ((ref != 0) & (ref & 0x80 == 0)).sum() > 1000  # dictionary and bucket matches
    assert len(seen) == 10  # H5/14/16, H5/15/16, H6/15/16, H5/14/32, H6/15/32, H5/15/64, H6/15/64, H5/15/128, H9/15/256, H6/15/256
    # lgwin 22 (H6, 16 deep: the size is above 4 MiB): the planted positions, the window edge and a sample
    d, marks = match_ref.planted_input(22, with_positions=True)
    maxb = (1 << 22) - 16
    rng = np.random.default_rng(1)
    query = np.unique(np.concatenate([marks, np.arange(maxb, maxb + 4096), rng.integers(0, len(d), 50000), np.arange(len(d) - 64, len(d))]))
    ref = match_ref.match_ref(d, 5, 22, query=query)
    diff = match_ref.first_difference(ref, _model_best(model, d, 5, 22)[query], query)
    assert diff is None, "planted lgwin 22: %s" % diff
    # ranges with a window in front of them
    pl = match_ref.planted_input(16) + golden_bytes("alice29.txt")
    for q, w, start, length in ((5, 18, 4113, 70001), (9, 16, 65536 + 12345, 30001)):
        ref = match_ref.match_ref(pl, q, w, 0, start, length)
        diff = match_ref.first_difference(ref, _model_best(model, pl, q, w, 0, start, length), np.arange(start, start + length))
        assert diff is None, "q%d lgwin %d range %d+%d: %s" % (q, w, start, length, diff)

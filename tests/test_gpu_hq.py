"""GPU (H100): the quality 10 / 11 path at the shapes its whole-stream tests do not reach.

The match stage is compared position by position with a brute-force restatement of its contract (tests/hq_ref.py) and with
the CPU model; the rest with the model's stream: every parse-unit size, the default unit bands, a size hint smaller than the
data, small windows, ranges that start past 0, and two sort batches in one chunk."""
import contextlib
import io

import numpy as np
import pytest

import hq_ref
from conftest import golden_bytes
from oracle.harness import sys_compress, sys_decompress

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def _option(encoder, opt, value, default):
    encoder.set_option(opt, value)
    try:
        yield
    finally:
        encoder.set_option(opt, default)


def _live(hqn, width):
    return np.arange(width)[None, :] < hqn[:, None].astype(np.int64)


def _stage_cases():
    from tools import datagen
    alice, logs = golden_bytes("alice29.txt"), datagen.json_logs(60000)
    cases = [(hq_ref.planted_input(w), w) for w in (10, 12, 16, 18)]
    cases += [(b"ab" * 20000, 10), (b"ab" * 20000 + alice[:5000], 16)]
    cases += [(alice[:60000], w) for w in (10, 12, 16, 18)] + [(logs, w) for w in (10, 12, 16, 18)]
    return cases


@pytest.mark.parametrize("q", [10, 11])
def test_hq_match_stage_equals_brute_force_and_model(encoder, model, q):
    """k_match_all + k_match_level: the window entries of every position equal the brute-force front; the whole lists
    (dictionary entries too), the per-unit results and the raw commands of the shortest-path parse equal the model."""
    for d, w in _stage_cases():
        what = "n=%d lgwin=%d" % (len(d), w)
        hqn, hqm, units, raw, unit = encoder.stage_hq(d, q, w)
        cnt, ent = hq_ref.hq_ref(d, q, w)
        diff = hq_ref.first_difference(cnt, ent, *hq_ref.window_part(hqn, hqm))
        assert diff is None, "%s, device vs brute force: %s" % (what, diff)
        mhqn, mhqm, munits, mraw, munit = model.stage_hq(d, q, w)
        assert unit == munit, what
        live = _live(hqn, hqm.shape[1])[:, :, None]
        bad = (hqn != mhqn) | (np.where(live, hqm, 0) != np.where(live, mhqm, 0)).any(axis=(1, 2))
        if bad.any():
            p = int(np.argmax(bad))
            pytest.fail("%s, device vs model at position %d: expected %s, got %s" % (
                what, p, mhqm[p, :mhqn[p]].tolist(), hqm[p, :hqn[p]].tolist()))
        assert np.array_equal(units, munits), what
        for u in range(units.shape[1]):
            k = int(units[0, u])
            assert np.array_equal(raw[u, :k], mraw[u, :k]), "%s: commands of unit %d" % (what, u)


def _unit_sizes(unit):
    return sorted(set(list(range(10)) + [unit - 1, unit, unit + 1, unit + 511, unit + 512, unit + 513, 2 * unit + 1,
                                         65535, 65536, 65537, 131073]))


@pytest.mark.parametrize("unit", [4096, 8192, 16384])
@pytest.mark.parametrize("q", [10, 11])
def test_hq_unit_sizes_equal_model(encoder, model, unit, q):
    """Parse units forced to 4 / 8 / 16 KiB (2 KiB is the default for these sizes: test_edge_sizes_deep_and_hq): sizes
    around one and two units, the 512-byte warm-up, and the 64 KiB window over which q11 pools its statistics."""
    import rust_brotli_b200 as rb
    src = golden_bytes("alice29.txt")
    with _option(encoder, rb._native.OPT_HQ_UNIT, unit, 0):
        for n in _unit_sizes(unit):
            d = src[:n]
            c = encoder.compress(d, q, 22)
            assert c == model.compress(d, q, 22, unit=unit, mb_units=(4 << 20) // unit)[0], n
            assert sys_decompress(c, max(n, 1)) == d, n


@pytest.mark.parametrize("q", [10, 11])
def test_hq_default_unit_bands_equal_model(encoder, model, q):
    """Size hints up to 256 KiB get 2 KiB parse units, up to 1 MiB 4 KiB, above that 8 KiB (q10) / 16 KiB (q11)."""
    from tools import datagen
    text = datagen.enwik_like(1048577, seed=12)
    for n in (262144, 262145, 1048576, 1048577):
        d = text[:n]
        c = encoder.compress(d, q, 22)
        assert c == model.compress(d, q, 22)[0], n
        assert sys_decompress(c, n) == d, n


def test_hq_size_hint_smaller_than_data(encoder, model):
    """A user's BROTLI_PARAM_SIZE_HINT of 100 000 on 4.6 MB: 2 KiB parse units over two 4 MiB metablocks (2048 units in the
    first).  The range call, the model and the C ABI must agree."""
    import rust_brotli_b200 as rb
    from tools import datagen
    d = datagen.enwik_like(4_600_000, seed=13)
    c = encoder.compress_range(d, 0, len(d), 10, 22, True, True, False, size_hint=100_000)
    assert c == model.compress_range(d, 0, len(d), 10, 22, True, True, False, size_hint=100_000)[0]
    s = rb._Stream(rb.BrotliEncoderParams(quality=10, lgwin=22, size_hint=100_000))
    try:
        via_abi = s.step(d, rb.BROTLI_OPERATION_FINISH)
    finally:
        s.close()
    assert sys_decompress(via_abi, len(d)) == d
    assert via_abi == c


@pytest.mark.parametrize("lgwin", [10, 11, 12, 14, 15])
@pytest.mark.parametrize("q", [10, 11])
def test_hq_small_windows(encoder, model, q, lgwin):
    """Windows of 1 to 32 KiB at quality 10 / 11, on alice29 (2 KiB units) and asyoulik + alice29 (4 KiB units): the stream
    equals the model's, decodes, and is no larger than libbrotlienc's at the same quality and window.  Measured (the model's
    stream, which the device reproduces): alice29 -1.22 % ... -0.46 % at q10, -0.55 % ... -0.32 % at q11; asyoulik + alice29
    -1.22 % ... -0.36 % at q10, -0.45 % ... -0.30 % at q11, over lgwin 10 - 15."""
    alice = golden_bytes("alice29.txt")
    for d in (alice, golden_bytes("asyoulik.txt") + alice):
        c = encoder.compress(d, q, lgwin)
        assert c == model.compress(d, q, lgwin)[0], len(d)
        assert sys_decompress(c, len(d)) == d
        ref = len(sys_compress(d, q, lgwin))
        assert len(c) <= ref, (len(d), len(c), ref)


@pytest.mark.parametrize("q", [10, 11])
def test_hq_ranges_past_zero(encoder, model, q):
    """Ranges that start inside the stream (abs_base > 0: shards of compress_multi, streamed pieces), including starts inside
    the first parse unit, past the 512-byte warm-up, at a unit seam and past the 64 KiB statistics window; then
    compress_multi with 3 shards, which must equal its shards compressed one by one and each shard the model's range."""
    import rust_brotli_b200 as rb
    d = golden_bytes("alice29.txt")
    for start in (1, 2, 3, 513, 2048, 70001):
        head = encoder.compress_range(d, 0, start, q, 22, True, False, True)
        tail = encoder.compress_range(d, start, len(d) - start, q, 22, False, True, False)
        assert sys_decompress(head + tail, len(d)) == d, start
        assert tail == model.compress_range(d, start, len(d) - start, q, 22, False, True, False)[0], start
    d = golden_bytes("asyoulik.txt") + d
    c = rb.compress_multi(rb.BrotliEncoderParams(quality=q, lgwin=22), d, 3)
    assert sys_decompress(c, len(d)) == d
    parts = []
    for i in range(3):
        a, b = i * len(d) // 3, (i + 1) * len(d) // 3
        win = (1 << 22) + 65536
        lo = ((a - win) & ~4095) if a > win else 0
        part = encoder.compress_range(d[lo:b], a - lo, b - a, q, 22, i == 0, i == 2, True, size_hint=b - a)
        assert part == model.compress_range(d[lo:b], a - lo, b - a, q, 22, i == 0, i == 2, True, size_hint=b - a)[0], i
        parts.append(part)
    assert b"".join(parts) == c


def _two_batch_input(n, seed):
    """PCG bytes with text islands; the islands repeat 16 MiB, 3 MB and 40 KB later, so copies cross the seam of the two sort
    batches of a lgwin 24 chunk (2^25 - 2^24 - 4096 = 16 773 120 payload bytes in the first)."""
    from tools import datagen
    a = np.frombuffer(datagen.pcg_random(n, seed=seed), dtype=np.uint8).copy()
    text = np.frombuffer(golden_bytes("alice29.txt"), dtype=np.uint8)
    seam = (1 << 25) - (1 << 24) - 4096
    for src, dst, ln in ((100_000, 100_000 + (1 << 24) - 20_000, 40_000),(seam - 3_000_000, seam - 30_000, 70_000),
                         (seam - 45_000, seam - 5_000, 40_000), (seam + 100_000, seam + 160_000, 30_000)):
        a[src:src + ln] = text[:ln]
        a[dst:dst + ln] = a[src:src + ln]
    return a.tobytes()


def test_hq_two_sort_batches_in_one_chunk(encoder, model):
    """quality 10, lgwin 24, 17 MB in one chunk: more than the 16 773 120 payload bytes of one sort batch, so the chunk is
    sorted in two batches (every long-prefix level re-sorts each) and copies cross the seam.  The stream equals the model's."""
    d = _two_batch_input(17_000_000, seed=22)
    c = encoder.compress(d, 10, 24)
    assert c == model.compress(d, 10, 24)[0]
    assert sys_decompress(c, len(d)) == d


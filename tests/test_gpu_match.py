"""GPU (H100): best[] of the quality 5..9 match stage against tests/match_ref.py, position by position.

The brute force restates the stage's contract without the kernels' headers, so a wrong score, window limit or dictionary
rule in bro_parse.cuh / bro_dict.cuh cannot hide on both sides.  Covered: every hasher / key width / depth of ChooseHasher
with both kernels (k_match_shallow at depth 16 / 32, k_match_deep at 64..256) and the on-demand search (k_rank_sig +
deep_best_warp, probed at every position and required to equal the up-front result), sizes around the first and last CTA,
ranges with a window in front of them, and 24 MiB chunks that take two sort batches.  The up-front results must also equal
the CPU model where the model is cheap."""
import numpy as np
import pytest

import match_ref
from conftest import golden_bytes

pytestmark = pytest.mark.gpu

MIB = 1 << 20
# (quality, lgwin, size hint): H5/14/16, H5/15/16, H6/15/16 (the bench path), H5/14/32, H6/15/32, H5/15/64, H6/15/64, H5/15/128,
# H9/15/256, and H6/15/256 at lgwin <= 16
CONFIGS = [(5, 22, MIB), (5, 22, 2 * MIB), (5, 22, 8 * MIB), (6, 22, MIB), (6, 22, 8 * MIB), (7, 22, 2 * MIB), (7, 22, 8 * MIB),
           (8, 22, MIB), (9, 22, MIB), (5, 16, 0), (8, 16, 0), (6, 10, 0), (6, 12, 0)]


@pytest.fixture(scope="module")
def inputs():
    from tools import datagen
    return {"text": datagen.enwik_like(400_000), "json": datagen.json_logs(400_000), "random": datagen.pcg_random(400_000),
            "alice": golden_bytes("alice29.txt")}


def _sample(n, k, seed=5):
    return np.random.default_rng(seed).integers(0, n, k)


def _check(encoder, d, q, w, hint=0, start=0, length=None, query=None, model=None, on_demand=True):
    """Up-front kernels == brute force (on the absolute positions `query`, default all), == the model if given; with depth
    >= 64 (and on_demand) the on-demand search == the up-front kernels at every position.  Returns the device result."""
    length = len(d) - start if length is None else length
    what = "q%d lgwin %d hint %d n=%d range %d+%d" % (q, w, hint, len(d), start, length)
    got = encoder.stage_match(d, q, w, hint, start, length)
    qi = np.arange(start, start + length) if query is None else np.unique(np.clip(query, start, start + length - 1))
    ref = match_ref.match_ref(d, q, w, hint, start, length, query=qi)
    diff = match_ref.first_difference(ref, got[qi - start], qi)
    assert diff is None, "%s, device vs brute force: %s" % (what, diff)
    if model is not None:
        mb = np.zeros(length + 1, dtype=np.uint32)
        model.compress_range(d, start, length, q, w, True, True, False, size_hint=hint, best_out=mb.ctypes.data)
        diff = match_ref.first_difference(mb[:length], got, np.arange(start, start + length))
        assert diff is None, "%s, device vs model: %s" % (what, diff)
    if on_demand and match_ref.config(q, w, hint or len(d))[2] >= 64:
        od = encoder.stage_match(d, q, w, hint, start, length, on_demand=True)
        diff = match_ref.first_difference(got, od, np.arange(start, start + length))
        assert diff is None, "%s, on-demand search vs up-front kernels: %s" % (what, diff)
    return got


@pytest.mark.parametrize("q,w,hint", CONFIGS)
def test_match_stage_equals_brute_force(encoder, model, inputs, q, w, hint):
    deep = match_ref.config(q, w, hint)[2] >= 64
    d, marks = match_ref.planted_input(w, with_positions=True)
    query = None
    if len(d) > 1_000_000:  # lgwin 22: the planted positions, the window edge, the end and a sample
        maxb = (1 << w) - 16
        query = np.concatenate([marks, np.arange(maxb - 64, maxb + 4096), np.arange(len(d) - 300, len(d)), _sample(len(d), 100_000)])
    _check(encoder, d, q, w, hint, query=query, model=model if len(d) < 1_000_000 else None)
    for name in ("alice", "text", "json", "random"):
        x = inputs[name]
        query = None
        if deep and name != "random":  # long buckets: a sample keeps the deep brute force short
            query = np.concatenate([np.arange(2000), np.arange(len(x) - 2000, len(x)), _sample(len(x), 40_000)])
        _check(encoder, x, q, w, hint, query=query, model=model)


@pytest.mark.parametrize("q,w,hint", [(5, 22, 8 * MIB), (6, 22, MIB), (7, 22, 2 * MIB), (9, 22, 0)])
def test_match_stage_sizes(encoder, model, q, w, hint):
    """The first and last CTA of a batch, one-entry buckets, the last 7 positions."""
    src = golden_bytes("alice29.txt") * 2
    for n in (1, 7, 8, 9, 255, 256, 257, 4095, 4096, 4097, 65537):
        _check(encoder, src[:n], q, w, hint, model=model)


@pytest.mark.parametrize("q,w,hint", [(5, 18, 0), (7, 18, 2 * MIB), (5, 16, 0), (9, 16, 0)])
def test_match_stage_ranges(encoder, model, q, w, hint):
    """Ranges that start past 0: the window in front of them (data_base and the batch origin > 0)."""
    d = match_ref.planted_input(16) + golden_bytes("alice29.txt")
    win = 1 << w
    for start, length in ((1, 70001), (4113, 50003), (win - 1, 30007), (win + 12345, 100001)):
        _check(encoder, d, q, w, hint, start, length, model=model)


@pytest.fixture(scope="module")
def big_text():
    from tools import datagen
    return datagen.enwik_like(24 * MIB, seed=6)


@pytest.mark.parametrize("w", [23, 24])
@pytest.mark.parametrize("q", [5, 7])
def test_match_stage_two_sort_batches(encoder, big_text, q, w):
    """A 24 MiB chunk with a window of 8 / 16 MiB takes two sort batches: at lgwin 23 the second is the last 4096 positions,
    at lgwin 24 it starts at 16 773 120 with its origin at 0.  Planted edges straddle the seam."""
    seam = (1 << 25) - (1 << w) - 4096
    pl, marks = match_ref.planted_input(16, with_positions=True)
    at = min(seam - 150_000, len(big_text) - len(pl) - 1000)
    d = big_text[:at] + pl + big_text[at + len(pl):]
    assert len(d) == 24 * MIB
    query = np.concatenate([np.arange(seam - 70_000, min(seam + 70_000, len(d))), np.arange(len(d) - 70_000, len(d)), marks + at,
                            _sample(len(d), 200_000)])
    _check(encoder, d, q, w, query=query, on_demand=False)
    with pytest.raises(RuntimeError):  # the on-demand path needs the chunk in one batch
        encoder.stage_match(d, q, w, on_demand=True)


def test_stage_match_q9_large_input_returns_matches(encoder):
    """At q9 an input of 4 MiB or more takes the on-demand path by default, which leaves ranks, not matches, in best[]; the
    hook switches it off and must return the matches of the up-front kernel (and the on-demand search the same)."""
    from tools import datagen
    d = datagen.json_logs(5_000_000)
    got = encoder.stage_match(d, 9, 22)
    query = np.unique(np.concatenate([np.arange(4000), _sample(len(d), 30_000)]))
    diff = match_ref.first_difference(match_ref.match_ref(d, 9, 22, query=query), got[query], query)
    assert diff is None, diff
    assert np.array_equal(encoder.stage_match(d, 9, 22, on_demand=True), got)

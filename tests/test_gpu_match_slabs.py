"""GPU (H100): best[] stored through the slab staging of k_match_shallow (match_store + k_best_place in bro_kernels.cuh).

A sort batch's payload is cut into slabs of 2^21 positions; every payload position leaves one record in its slab and the
placement kernel writes best[] from the records.  Checked here at bucket depth 16 (q5) and 32 (q6): best[] equals the
brute force of tests/match_ref.py around every slab edge and on a sample, for ranges with a window in front of them, payloads
that are not a multiple of the slab size and a chunk of two sort batches; and on the device, the records claimed in each slab of
the last batch equal the slab's size, so every record was placed exactly once."""
import numpy as np
import pytest

import match_ref

pytestmark = pytest.mark.gpu

MIB = 1 << 20
SLAB = 1 << 21


@pytest.fixture(scope="module")
def text24():
    from tools import datagen
    return datagen.enwik_like(24 * MIB, seed=11)


def _batches(w, start, length):
    """[b0, b1) of each sort batch of the range (run_chunk in bro_encoder.cu)."""
    payload_max = (1 << 25) - (1 << w) - 4096
    return [(b0, min(start + length, b0 + payload_max)) for b0 in range(start, start + length, payload_max)]


# (lgwin, range start, range length): lgwin 22 with the window partly / wholly in front of the range (batch origin 0 and > 0),
# 4 + 1 and 9 + 1 slabs, the last one short; lgwin 24, one 24 MiB chunk in two batches (7 + 1 slabs, then 4 + 1 slabs)
CASES = [(22, 3 * MIB + 123, 9 * MIB + 4321), (22, 5 * MIB + 77, 19 * MIB - 77), (24, 0, 24 * MIB)]


@pytest.mark.parametrize("w,start,length", CASES)
@pytest.mark.parametrize("q", [5, 6])
def test_slab_staged_best_equals_brute_force(encoder, text24, q, w, start, length):
    d = text24[:start + length]
    batches = _batches(w, start, length)
    got = encoder.stage_match(d, q, w, 0, start, length)
    cursors, sizes = encoder.stage_match_slabs()
    b0, b1 = batches[-1]
    expect = [min(SLAB, b1 - s) for s in range(b0, b1, SLAB)]
    assert sizes.tolist() == expect
    assert cursors.tolist() == expect, "records claimed per slab of the last batch"
    edges = [e for b0, b1 in batches for e in list(range(b0, b1, SLAB)) + [b1]]
    rng = np.random.default_rng(q * 100 + w)
    query = np.concatenate([np.arange(e - 1500, e + 1500) for e in edges] + [rng.integers(start, start + length, 60_000)])
    query = np.unique(np.clip(query, start, start + length - 1))
    ref = match_ref.match_ref(d, q, w, 0, start, length, query=query)
    diff = match_ref.first_difference(ref, got[query - start], query)
    assert diff is None, "q%d lgwin %d range %d+%d, device vs brute force: %s" % (q, w, start, length, diff)

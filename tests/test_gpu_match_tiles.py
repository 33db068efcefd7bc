"""GPU (H100): best[] placed through the tiles of k_best_bin / k_best_tile (bro_kernels.cuh).

After k_match_shallow has binned a sort batch's records by slab of 2^21 positions, k_best_bin reorders them by tile of 2^13
positions into a tile-major buffer, and k_best_tile writes each tile of best[] from a shared-memory image.  Checked here at
bucket depth 16 (q5) and 32 (q6): best[] equals the brute force of tests/match_ref.py around both edges of a few chosen tiles of
every batch (the first, the last, the two on each side of a slab edge, two random ones), around every slab edge and on a random
sample, for ranges with a window in front of them (batch origin 0 and > 0), payloads that are not a multiple of the tile size and
a chunk of two sort batches; and on the device, the records claimed in each tile of the last batch equal the tile's size, so
every record was placed exactly once."""
import numpy as np
import pytest

import match_ref

pytestmark = pytest.mark.gpu

MIB = 1 << 20
SLAB = 1 << 21
TILE = 1 << 13


@pytest.fixture(scope="module")
def text24():
    from tools import datagen
    return datagen.enwik_like(24 * MIB, seed=12)


def _batches(w, start, length):
    """[b0, b1) of each sort batch of the range (run_chunk in bro_encoder.cu)."""
    payload_max = (1 << 25) - (1 << w) - 4096
    return [(b0, min(start + length, b0 + payload_max)) for b0 in range(start, start + length, payload_max)]


def _edges(b0, b1, rng):
    """Both edges of the chosen tiles of batch [b0, b1) and every slab edge, as absolute positions."""
    nt = -(-(b1 - b0) // TILE)
    chosen = {0, nt - 1} | {int(t) for t in rng.integers(0, nt, 2)}
    for s in range(SLAB, b1 - b0, SLAB):
        chosen |= {s // TILE - 1, s // TILE}
    edges = set(range(b0, b1, SLAB)) | {b1}
    for t in chosen:
        edges |= {b0 + t * TILE, min(b1, b0 + (t + 1) * TILE)}
    return sorted(edges)


# (lgwin, range start, range length): lgwin 22 with the window partly / wholly in front of the range (batch origin 0 and > 0),
# payloads of 1152 + 1 and 2431 + 1 tiles, the last one short; lgwin 24, one 24 MiB chunk in two batches
CASES = [(22, 3 * MIB + 123, 9 * MIB + 4321), (22, 5 * MIB + 77, 19 * MIB - 77), (24, 0, 24 * MIB)]


@pytest.mark.parametrize("w,start,length", CASES)
@pytest.mark.parametrize("q", [5, 6])
def test_tile_placed_best_equals_brute_force(encoder, text24, q, w, start, length):
    d = text24[:start + length]
    batches = _batches(w, start, length)
    got = encoder.stage_match(d, q, w, 0, start, length)
    cursors, sizes = encoder.stage_match_tiles()
    b0, b1 = batches[-1]
    expect = [min(TILE, b1 - t) for t in range(b0, b1, TILE)]
    assert sizes.tolist() == expect
    assert cursors.tolist() == expect, "records claimed per tile of the last batch"
    rng = np.random.default_rng(q * 1000 + w)
    edges = [e for b0, b1 in batches for e in _edges(b0, b1, rng)]
    query = np.concatenate([np.arange(e - 1500, e + 1500) for e in edges] + [rng.integers(start, start + length, 40_000)])
    query = np.unique(np.clip(query, start, start + length - 1))
    ref = match_ref.match_ref(d, q, w, 0, start, length, query=query)
    diff = match_ref.first_difference(ref, got[query - start], query)
    assert diff is None, "q%d lgwin %d range %d+%d, device vs brute force: %s" % (q, w, start, length, diff)

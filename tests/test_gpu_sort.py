"""The sort stage position by position: a batch's sorted list equals numpy's stable argsort of the bucket keys.

The keys are restated in numpy: H5 ((load32 * 0x1e35a7bd) >> (32 - bits)), H6 ((load40 * 0x1fe35a7bd3579bd3) >> (64 - bits)) and
the long-prefix level hashes of quality 10 / 11 (tests/hq_ref.py).  Bytes past the end of the batch read as zero.
"""
import numpy as np
import pytest

import hq_ref

TILE = 4096


def _keys(data: bytes, hash_type: int, key_bits: int, level=None):
    a = np.frombuffer(data, dtype=np.uint8)
    n = len(a)
    w32, w64 = hq_ref._words(a, 48)
    with np.errstate(over="ignore"):
        if level is not None:
            return (hq_ref._level_hash(w64, 8 << level)[:n] >> np.uint64(64 - key_bits)).astype(np.int64)
        if hash_type == 6:
            v = w64[:n] & np.uint64(0xFFFFFFFFFF)
            return ((v * np.uint64(0x1fe35a7bd3579bd3)) >> np.uint64(64 - key_bits)).astype(np.int64)
        return (((w32[:n] * np.uint64(0x1e35a7bd)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - key_bits)).astype(np.int64)


def _input(n: int, seed: int) -> bytes:
    """Text with a zero run and a run of one repeated byte: buckets from a handful of positions to most of a tile, and whole
    tiles of one key (the look-back then crosses many tiles of zero count for every other digit)."""
    from tools import datagen
    a = np.frombuffer(datagen.enwik_like(n, seed=seed), dtype=np.uint8).copy()
    if n > 4 * TILE:
        a[n // 3:n // 3 + 3 * TILE + 77] = 0
        a[n // 2:n // 2 + TILE + 5] = ord("a")
    return a.tobytes()


def _check(encoder, data, quality, lgwin, hash_type, key_bits, level=None):
    got = encoder.stage_sort(data, quality, lgwin, level)
    key = _keys(data, hash_type, key_bits, level)
    want = np.argsort(key, kind="stable").astype(np.uint32)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "n=%d q%d lgwin %d level %s: %d sorted slots differ, first slot %d (tile %d): expected position %d " \
        "(key %d), got %d (key %s)" % (len(data), quality, lgwin, level, bad.size, bad[0], want[bad[0]] // TILE, want[bad[0]],
                                       key[want[bad[0]]], got[bad[0]], key[got[bad[0]]] if got[bad[0]] < len(data) else "-")


# (n, quality, lgwin, hash type and key bits the encoder picks for that size hint)
CASES = [
    (1000, 5, 22, 5, 14),                 # smaller than one tile, 14-bit keys
    (TILE, 5, 22, 5, 14),                 # exactly one tile
    (7 * TILE + 1234, 5, 22, 5, 14),      # a partial last tile
    (2 * 2**20 + 777, 5, 22, 5, 15),      # 15-bit keys
    (6 * 2**20 + 4095, 5, 22, 6, 15),     # H6 (5-byte hash), the bench configuration
]


@pytest.mark.gpu
@pytest.mark.parametrize("n,q,w,ht,bits", CASES)
def test_sorted_list_equals_stable_argsort(encoder, n, q, w, ht, bits):
    _check(encoder, _input(n, seed=n % 97), q, w, ht, bits)


@pytest.mark.gpu
def test_full_batch(encoder):
    """2^25 positions, the largest batch: 8192 tiles, positions use all 25 bits of the packed word."""
    _check(encoder, _input(1 << 25, seed=5), 5, 22, 6, 15)


@pytest.mark.gpu
@pytest.mark.parametrize("level", [0, 2])
def test_level_sort(encoder, level):
    """The long-prefix levels of quality 10 / 11 (8 and 32 bytes hashed), 15-bit keys."""
    _check(encoder, _input(3 * 2**20 + 333, seed=11), 10, 22, None, 15, level)


@pytest.mark.gpu
def test_consecutive_sorts_share_no_state(encoder):
    """A large sort, then a small one on the same lane, then the large one again: no look-back word or count of one sort
    leaks into the next."""
    big = _input(5 * 2**20 + 3, seed=2)
    _check(encoder, big, 5, 22, 6, 15)
    _check(encoder, _input(3 * TILE + 9, seed=3), 5, 22, 5, 14)
    _check(encoder, big, 5, 22, 6, 15)

"""Brute-force reference of the quality 5..9 match stage (best[] of k_match_shallow / k_match_deep and of the on-demand
search), in plain numpy.

It restates the contract of the stage without using its code (csrc/bro_parse.cuh, bro_dict.cuh).

Configuration, from (quality, lgwin, size hint): ChooseHasher, encode.rs:834-893 (DESIGN.md section 2.1):
  * q9: H9, 15-bit keys, depth 256;
  * q5..q8 with lgwin <= 16: H6, 15-bit keys, depth 256;
  * q5..q8 with a hint above 4 MiB and lgwin >= 19: H6, 15-bit keys, depth 2^(q-1);
  * otherwise H5, depth 2^(q-1), 14-bit keys when q < 7 and the hint is at most 1 MiB, else 15-bit keys.
Lengths are capped at 64 and the window is maxb = 2^lgwin - 16.

Per position p of the range [s, e) (absolute positions; the bytes in front of s are the window, bytes past e read as zero):
  * e - p < 8: best = 0 (no bucket match and no dictionary candidate);
  * maxl = min(64, e - p), mb = min(p, maxb);
  * key: H5 / H9 (load32 * 0x1e35a7bd mod 2^32) >> (32 - bits) (mod.rs:990-991); H6 (load40 * 0x1fe35a7bd3579bd3 mod 2^64)
    >> (64 - bits) (mod.rs:1138-1140);
  * candidates: the `depth` nearest c < p with the same key (every position is in its bucket, colliding ones too, and uses up
    depth); one counts if p - c <= mb and its common prefix with p is >= 4 bytes (capped at maxl);
  * score: H5 / H6 1920 + 135 len - 30 floor(log2 d) (backward_references/mod.rs:1878), H9 (7680 + 540 len - 120 floor(log2 d))
    >> 2 (mod.rs:685); best is the highest score above 2020, the nearest on equal scores, packed d << 8 | len;
  * no candidate: the static-dictionary candidate of mod.rs:1896-1988 with this library's slot table: the two slots at
    Hash14(load32); a slot is skipped if empty, if its word is longer than e - p, or if the matched length ml < 4 or
    ml + 10 <= word length wl; word_id = index + (OmitLast(wl - ml) << NDBITS[wl]); it is scored at distance mb + 1 + word_id,
    a score >= the best so far (2020 at first) wins, so the later slot wins ties; packed (wl - ml) << 26 | word_id << 8 | 0x80 | ml.
"""
import importlib.util
import os

import numpy as np

import hq_ref

LCAP = 64
MIN_SCORE = 2020
DICT_FLAG = 0x80
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def config(quality, lgwin, size_hint):
    """(hasher, key bits, depth) of quality 5..9."""
    q = max(quality, 5)
    assert q <= 9, "quality 10 / 11: see hq_ref.py"
    lgwin = min(max(lgwin, 10), 24)
    hint = min(size_hint, 0xFFFFFFFF)
    if q == 9:
        return 9, 15, 256
    if lgwin <= 16:
        return 6, 15, 256
    if hint > 1 << 22 and lgwin >= 19:
        return 6, 15, 1 << (q - 1)
    return 5, 14 if q < 7 and hint <= 1 << 20 else 15, 1 << (q - 1)


def keys(w64, hasher, bits):
    if hasher == 6:
        return ((w64 & np.uint64(0xFFFFFFFFFF)) * np.uint64(0x1fe35a7bd3579bd3)) >> np.uint64(64 - bits)
    return (((w64 & np.uint64(0xFFFFFFFF)) * np.uint64(0x1e35a7bd)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - bits)


def score(hasher, length, distance):
    lg = np.frexp(np.asarray(distance, dtype=np.float64))[1].astype(np.int64) - 1  # floor(log2 d), exact
    length = np.asarray(length, dtype=np.int64)
    if hasher == 9:
        return (7680 + 540 * length - 120 * lg) >> 2
    return 1920 + 135 * length - 30 * lg


_DICT = None


def dictionary():
    """(words u8[], NDBITS[32], offsets[32], slot table u16[32768], OmitLast transform id by cut 0..9).  Words and transforms
    come from the RFC 7932 tables of the system library, the slot table from this library's generator (it is data: which
    two words a bucket holds); the OmitLastN ids are looked up in the transform list."""
    global _DICT
    if _DICT is None:
        spec = importlib.util.spec_from_file_location("gen_dict", os.path.join(_ROOT, "rust-brotli_b200", "gen_dict.py"))
        g = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(g)
        data, bits, offs = g.load_dictionary()
        table = np.array(g.build_hash(data, bits, offs), dtype=np.int64)
        tr = g.load_transforms()
        omit = [tr.index((b"", cut, b"")) for cut in range(10)]  # type 0 = identity, 1..9 = omit last 1..9
        _DICT = (np.frombuffer(data + bytes(64), dtype=np.uint8), np.array(bits, np.int64), np.array(offs, np.int64), table,
                 np.array(omit, np.int64))
    return _DICT


def _dict_candidates(hasher, ap, w32, q, e_minus_p, mb):
    """Dictionary candidate (packed, 0 = none) of positions q of the zero-padded bytes ap."""
    words, ndbits, offs, table, omit = dictionary()
    k14 = (((w32[q] * np.uint64(0x1e35a7bd)) & np.uint64(0xFFFFFFFF)) >> np.uint64(18)).astype(np.int64)
    best = np.zeros(len(q), dtype=np.int64)
    best_score = np.full(len(q), MIN_SCORE, dtype=np.int64)
    for s in (0, 1):
        item = table[2 * k14 + s]
        wl, idx = item & 31, item >> 5
        ok = (item != 0) & (wl <= e_minus_p)
        base = offs[wl] + wl * idx
        ml = np.zeros(len(q), dtype=np.int64)
        alive = ok.copy()
        for j in range(24):
            alive &= (j < wl) & (ap[q + j] == words[base + j])
            ml += alive
        cut = wl - ml
        ok &= (ml >= 4) & (ml + 10 > wl)
        word_id = idx + (omit[np.minimum(cut, 9)] << ndbits[wl])
        sc = score(hasher, ml, mb + 1 + word_id)
        win = ok & (sc >= best_score)
        best = np.where(win, (cut << 26) | (word_id << 8) | DICT_FLAG | ml, best)
        best_score = np.where(win, sc, best_score)
    return best


def match_ref(data: bytes, quality: int, lgwin: int, size_hint: int = 0, start: int = 0, length=None, use_dict=True, query=None):
    """best[] of the positions `query` (absolute, sorted, inside the range; default: the whole range) of the range
    [start, start + length) of data.  size_hint 0 = len(data), as the encoder does."""
    if length is None:
        length = len(data) - start
    e = start + length
    hasher, bits, depth = config(quality, lgwin, size_hint or len(data))
    lgwin = min(max(lgwin, 10), 24)
    maxb = (1 << lgwin) - 16
    query = np.arange(start, e, dtype=np.int64) if query is None else np.asarray(query, dtype=np.int64)
    assert np.all(np.diff(query) > 0) and (not query.size or (query[0] >= start and query[-1] < e))
    out = np.zeros(len(query), dtype=np.uint32)
    lo = max(0, start - (1 << lgwin))  # entries farther back are out of the window of every position of the range
    a = np.frombuffer(data, dtype=np.uint8)[lo:e]
    w32, w64 = hq_ref._words(a, LCAP + 32)
    pos = np.arange(len(a), dtype=np.int64) + lo
    key = keys(w64[:len(a)], hasher, bits)
    maxl = np.minimum(LCAP, e - pos)
    mb = np.minimum(pos, maxb)
    sel = np.flatnonzero(e - query >= 8)
    qr = query[sel] - lo
    P, D, L = hq_ref._nearest_same_key(key, qr, depth, lambda q, c: w32[c] == w32[q], w64, maxl, limit=LCAP, maxb=mb)
    S = score(hasher, L, D)
    k = S > MIN_SCORE
    P, D, L, S = P[k], D[k], L[k], S[k]
    o = np.lexsort((D, -S, P))  # per position: highest score, then nearest
    P, D, L = P[o], D[o], L[o]
    first = np.ones(len(P), dtype=bool)
    first[1:] = P[1:] != P[:-1]
    P, D, L = P[first], D[first], L[first]
    res = np.zeros(len(qr), dtype=np.int64)
    res[np.searchsorted(qr, P)] = (D << 8) | L
    if use_dict:
        nd = np.flatnonzero(res == 0)
        ap = np.concatenate([a, np.zeros(64, dtype=np.uint8)])
        res[nd] = _dict_candidates(hasher, ap, w32, qr[nd], e - (qr[nd] + lo), mb[qr[nd]])
    out[sel] = res
    return out


def describe(v):
    v = int(v)
    if v == 0:
        return "none"
    if v & DICT_FLAG:
        _, ndbits, _, _, _ = dictionary()
        ml, cut, word_id = v & 0x7F, (v >> 26) & 0xF, (v >> 8) & 0x3FFFF
        nb = int(ndbits[ml + cut])
        return "dictionary word %d of length %d (transform %d), %d bytes matched, cut %d" % (
            word_id & ((1 << nb) - 1), ml + cut, word_id >> nb, ml, cut)
    return "distance %d length %d" % (v >> 8, v & 0xFF)


def first_difference(expected, got, query=None):
    """None if both best[] arrays agree, else a report of the first differing position (query: the absolute positions of
    the entries; default 0, 1, ..)."""
    expected, got = np.asarray(expected), np.asarray(got)
    assert expected.shape == got.shape
    bad = np.flatnonzero(expected != got)
    if not bad.size:
        return None
    i = int(bad[0])
    p = int(query[i]) if query is not None else i
    return "position %d (%d positions differ): expected %s, got %s" % (p, bad.size, describe(expected[i]), describe(got[i]))


# ---- inputs that reach every edge of the contract ----

def _collisions(rng, hasher, bits, count):
    """Pairs (x, y) of 8-byte strings with the same bucket key whose first four bytes differ; for H6 also pairs with the same
    first four bytes and a different fifth byte (found by search over every fifth byte of many prefixes)."""
    out = []
    v = rng.integers(0, 1 << 62, 1 << 20, dtype=np.int64).astype(np.uint64)
    k = keys(v, hasher, bits)
    o = np.argsort(k, kind="stable")
    ks = k[o]
    same = np.flatnonzero(ks[1:] == ks[:-1])
    for i in same:
        x, y = int(v[o[i]]), int(v[o[i + 1]])
        if (x ^ y) & 0xFFFFFFFF:
            out.append((x.to_bytes(8, "little"), y.to_bytes(8, "little")))
        if len(out) == count:
            break
    if hasher == 6:
        pre = rng.integers(0, 1 << 32, 4096, dtype=np.int64).astype(np.uint64)
        cand = (pre[:, None] | (np.arange(256, dtype=np.uint64)[None, :] << np.uint64(32))).ravel()
        k = keys(cand, 6, bits).reshape(4096, 256)
        found = 0
        for r in range(4096):
            u, first, cnt = np.unique(k[r], return_index=True, return_counts=True)
            j = np.flatnonzero(cnt > 1)
            if j.size:
                b5 = np.flatnonzero(k[r] == u[j[0]])[:2]
                out.append((int(cand[r * 256 + b5[0]]).to_bytes(8, "little"), int(cand[r * 256 + b5[1]]).to_bytes(8, "little")))
                found += 1
                if found == count:
                    break
    return out


def _dictionary_plants(rng):
    """Byte strings that hit the dictionary: whole words, cuts 1..10, hash collisions with a word, buckets whose two slots
    both match (equal and different scores)."""
    words, ndbits, offs, table, _ = dictionary()
    word = lambda item: bytes(words[offs[item & 31] + (item & 31) * (item >> 5):][:item & 31])
    items = [int(t) for t in table[0::2] if t and (t & 31) >= 14]
    rng.shuffle(items)
    out = []
    for cut, item in zip(range(11), items):
        w = word(item)
        out.append(w[:len(w) - cut] + bytes([w[len(w) - cut] ^ 0x55 if cut else 0x01]))
    # a 4-byte hash collision with a slot word: same Hash14, different first four bytes
    w = word(items[11])
    h = (int.from_bytes(w[:4], "little") * 0x1e35a7bd & 0xFFFFFFFF) >> 18
    v = rng.integers(0, 1 << 32, 1 << 20, dtype=np.int64).astype(np.uint64)
    hv = ((v * np.uint64(0x1e35a7bd)) & np.uint64(0xFFFFFFFF)) >> np.uint64(18)
    y = int(v[np.flatnonzero(hv == h)[0]]).to_bytes(4, "little")
    out.append(y + w[4:] + b"\x01")
    # buckets with two matching slots: the longer word in full, and only the common prefix (equal lengths matched)
    pairs = 0
    for b in range(16384):
        t0, t1 = int(table[2 * b]), int(table[2 * b + 1])
        if not (t0 and t1):
            continue
        w0, w1 = word(t0), word(t1)
        cp = next((i for i in range(min(len(w0), len(w1))) if w0[i] != w1[i]), min(len(w0), len(w1)))
        if cp >= 4 and cp + 10 > max(len(w0), len(w1)):
            long_ = w0 if len(w0) >= len(w1) else w1
            out.append(long_ + b"\x01")
            out.append(long_[:cp] + b"\x02")
            pairs += 1
            if pairs == 6:
                break
    return out


def planted_input(lgwin: int, seed: int = 7, with_positions: bool = False):
    """PCG bytes with planted structure at the edges of the contract: copies of lengths 3..200 around the 4 / 8 / 12 / 16-byte
    word steps and the 64-byte cap; distances 1-3 (overlapping runs), maxb - 1, maxb, maxb + 1 and exactly p from position 0;
    score ties where the nearer candidate must win (equal lengths in one octave; len L at d = 16..31 against L + 2 nine
    octaves farther, for L = 6 and 10, within one group of 16 bucket entries and across groups); buckets with 15, 16, 17, 31,
    32, 33, .., 255, 256, 257 earlier entries of which only the farthest continues; a bucket of ~1000 entries; key collisions
    (14- and 15-bit H5, H6, and H6 with equal first four bytes); dictionary words before and after p = maxb; copies that end
    9, 8 and 1 bytes before the end.  with_positions: also the positions where something was planted."""
    rng = np.random.Generator(np.random.PCG64(seed))
    maxb = (1 << lgwin) - 16
    dict_plants = _dictionary_plants(rng)
    coll = _collisions(rng, 5, 14, 4) + _collisions(rng, 5, 15, 4) + _collisions(rng, 6, 15, 4)
    n = max(300_000, maxb + 40_000)
    a = rng.integers(0, 256, n, dtype=np.uint8)
    marks = []

    def put(p, b):
        a[p:p + len(b)] = np.frombuffer(b, dtype=np.uint8)

    def copy(dst, src, ln):  # byte by byte: overlapping runs
        if dst - src >= ln:
            a[dst:dst + ln] = a[src:src + ln]
        else:
            for k in range(ln):
                a[dst + k] = a[src + k]
        a[dst + ln] = a[src + ln] ^ 0xA5  # ends exactly here
        marks.append(dst)

    def dict_group(p):
        for b in dict_plants:
            put(p, b)
            marks.append(p)
            p += len(b) + 8 + int(rng.integers(0, 8))
        return p

    p = dict_group(64)  # before maxb
    copy(p + 16, 0, 40)  # distance exactly p from position 0
    p += 120
    for d in (1, 2, 3):
        for ln in (5, 20, 70):
            copy(p + d, p, ln)
            p += ln + 40
    for ln in (3, 4, 7, 8, 9, 11, 12, 13, 15, 16, 17, 23, 24, 25, 63, 64, 65, 200):
        for d in (300, 5000):
            copy(p + d, p, ln)
            p += d + ln + 40
    # equal lengths in one octave (600 and 1000): the nearer wins
    for ln in (6, 12, 30):
        t = rng.integers(0, 256, ln, dtype=np.uint8).tobytes()
        for off in (0, 400, 1000):
            put(p + off, t + bytes([off % 251]))
        marks.append(p + 1000)
        p += 1000 + ln + 40
    # len L at d1 (16..31) against len L + 2 nine octaves farther: equal scores (H5 / H6 and H9 alike)
    for ln in (6, 10):
        for fill in (0, 20):  # 20 same-key entries between them: the far one is in another group of 16
            t = rng.integers(0, 256, ln + 2, dtype=np.uint8).tobytes()
            d1, d2 = 16 + int(rng.integers(0, 16)), 8192 + int(rng.integers(0, 8000))
            q = p + d2
            put(p, t + b"\x01")
            for k in range(fill):
                put(q - d1 - 60 * (k + 1), t[:5] + bytes([t[5] ^ 0x3C, k]))
            put(q - d1, t[:ln] + bytes([t[ln] ^ 0x11]))
            put(q, t + b"\x02")
            marks.append(q)
            p = q + ln + 40
    # buckets with k earlier entries of which only the farthest continues like the query
    for k in (15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257):
        head = rng.integers(0, 256, 8, dtype=np.uint8).tobytes()
        tail = rng.integers(0, 256, 24, dtype=np.uint8).tobytes()
        for r in range(k + 1):
            if r in (0, k):
                put(p, head + tail)
                p += 32
            else:
                put(p, head[:5] + bytes([head[5] ^ 0x77]) + bytes([r & 0xFF, r >> 8]))
                p += 8
        marks.append(p - 32)
    # one bucket of ~1000 entries, tails from a two-letter alphabet so that the lengths vary
    head = rng.integers(0, 256, 5, dtype=np.uint8).tobytes()
    for r in range(1000):
        put(p, head + (rng.integers(0, 2, 11, dtype=np.uint8) + 65).tobytes())
        marks.append(p)
        p += 16
    # key collisions: x, y share the bucket key; x again later finds x behind the collision
    for x, y in coll:
        put(p, x + b"\x09")
        put(p + 100, y + b"\x0A")
        put(p + 200, x + b"\x0B")
        marks.extend((p + 100, p + 200))
        p += 300
    assert p < n - 30_000
    p = max(p + 1000, maxb + 2048)
    for d in (maxb - 1, maxb, maxb + 1):
        copy(p, p - d, 20)
        p += 100
    p = dict_group(p + 64)  # after maxb
    assert p < n - 200
    for end in (n - 9, n - 8):  # copies that end 9 and 8 bytes before the end, and one at the very end
        copy(end - 24, end - 24 - 777, 24)
    a[n - 30:] = a[n - 30 - 999:n - 999]
    marks.append(n - 30)
    d = a.tobytes()
    return (d, np.unique(np.array(marks, dtype=np.int64))) if with_positions else d

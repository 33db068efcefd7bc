"""Brute-force reference of the quality 10 / 11 all-matches stage, in plain numpy.

It restates the contract of the stage (csrc/bro_hq.cuh, k_match_all / k_match_level) without using its code.  For a
position p of an n-byte input with n - p >= 8, maxl = min(384, n - p) and maxb = min(p, 2^lgwin - 16); lengths are exact
common-prefix lengths capped at maxl, and a candidate distance d needs d <= maxb:

  * short:  d < 16 (64 at quality 11), length >= 2;
  * bucket: length >= 4, the same H5 key ((load32 * 0x1e35a7bd) >> 17) and p - d among the 256 nearest earlier positions with
            that key (positions whose key collides but whose first four bytes differ use up depth);
  * level l = 0, 1, 2 (8, 16, 32 bytes), only when n - p >= bytes + 8: the same 15-bit key of the level hash, the same low 32
            bits of it, and p - d among the 1024 nearest earlier positions with that key.

A source's list is its Pareto front (a candidate is kept when it is strictly longer than every nearer one), the 8 longest kept.
The list of a position is the front of short + bucket; each level's list is then merged into it in turn (ties in distance go to
the earlier list) and again the 8 longest are kept.  Static-dictionary entries are not covered here.
"""
import numpy as np

LCAP = 384
MAXW = 8
DEPTH = 256
LEVEL_DEPTH = 1024
M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def _words(a, pad):
    """load32 and load64 (little endian) at every position of a zero-padded copy."""
    b = np.concatenate([a, np.zeros(pad, dtype=np.uint8)]).astype(np.uint64)
    m = len(a) + pad - 8
    w64 = np.zeros(m, dtype=np.uint64)
    for i in range(8):
        w64 |= b[i:i + m] << np.uint64(8 * i)
    return w64 & np.uint64(0xFFFFFFFF), w64


def _lcp(w64, p, c, cap, limit=LCAP):
    """Common-prefix length of positions p and c (arrays), at most cap (<= limit, the largest cap of the caller)."""
    out = np.zeros(len(p), dtype=np.int64)
    alive = np.arange(len(p))
    for j in range(0, limit, 8):
        if not alive.size:
            break
        x = w64[p[alive] + j] ^ w64[c[alive] + j]
        hit = x != 0
        if hit.any():
            xs = x[hit]
            low = xs & (~xs + np.uint64(1))
            out[alive[hit]] = j + (np.log2(low.astype(np.float64)).astype(np.int64) >> 3)
        out[alive[~hit]] = j + 8
        alive = alive[~hit]
    return np.minimum(out, cap)


def _level_hash(w64, nbytes):
    with np.errstate(over="ignore"):
        h = np.full(len(w64) - 32, (0x9E3779B97F4A7C15 * nbytes) & 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
        for k in range(0, nbytes, 8):
            h = (h ^ w64[k:k + len(h)]) * np.uint64(0xff51afd7ed558ccd)
            h ^= h >> np.uint64(32)
    return h


def _nearest_same_key(key, query, depth, accept, w64, maxl, limit=LCAP, maxb=None):
    """(p, distance, length) for every query position p and each of the `depth` nearest earlier positions with the same key
    for which accept(p, cand) holds.  A position stops collecting once it has a match of length maxl: nothing farther can
    be longer, so the fronts do not change.  With maxb (per position) it also stops at the first entry farther back than
    maxb[p]: every older one is out of the window too."""
    order = np.argsort(key, kind="stable")
    rank = np.empty(len(key), dtype=np.int64)
    rank[order] = np.arange(len(key))
    _, counts = np.unique(key, return_counts=True)
    ps, ds, ls = [], [], []
    q = query
    r = rank[q]
    for k in range(1, min(depth, int(counts.max()) - 1) + 1):
        ok = r >= k
        q, r = q[ok], r[ok]
        c = order[r - k]
        same = key[c] == key[q]
        q, r, c = q[same], r[same], c[same]  # the rest have fewer than k earlier entries in their bucket
        if maxb is not None:
            inw = q - c <= maxb[q]
            q, r, c = q[inw], r[inw], c[inw]
        if not q.size:
            break
        a = accept(q, c)
        ln = _lcp(w64, q[a], c[a], maxl[q[a]], limit)
        ps.append(q[a]); ds.append(q[a] - c[a]); ls.append(ln)
        full = np.zeros(len(q), dtype=bool)
        full[np.flatnonzero(a)[ln == maxl[q[a]]]] = True
        q, r = q[~full], r[~full]
    if not ps:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(ps), np.concatenate(ds), np.concatenate(ls)


def _front(p, d, ln, pri):
    """Pareto front per position (sorted by distance, then by pri), the MAXW longest kept."""
    o = np.lexsort((pri, d, p))
    p, d, ln = p[o], d[o], ln[o]
    v = p * 1024 + ln
    prev = np.concatenate([[-1], np.maximum.accumulate(v)[:-1]])
    k = (v > prev) & (ln >= 2)
    p, d, ln = p[k], d[k], ln[k]
    after = np.searchsorted(p, p, side="right") - 1 - np.arange(len(p))
    k = after < MAXW
    return p[k], d[k], ln[k]


def hq_ref(data: bytes, quality: int, lgwin: int, levels: int = 3):
    """Window matches of every position: (count[n] u8, entries[n][8][2] u32 (distance, length)), nearest first."""
    a = np.frombuffer(data, dtype=np.uint8)
    n = len(a)
    cnt = np.zeros(n, dtype=np.uint8)
    ent = np.zeros((n, MAXW, 2), dtype=np.uint32)
    if n < 8:
        return cnt, ent
    w32, w64 = _words(a, LCAP + 48)
    pos = np.arange(n, dtype=np.int64)
    maxl = np.minimum(LCAP, n - pos)
    maxb = np.minimum(pos, (1 << lgwin) - 16)
    query = pos[: n - 7]
    P, D, Ln = [], [], []
    # short distances
    for d in range(1, 64 if quality == 11 else 16):
        q = query[maxb[query] >= d]
        ln = _lcp(w64, q, q - d, maxl[q])
        k = ln >= 2
        P.append(q[k]); D.append(np.full(int(k.sum()), d, np.int64)); Ln.append(ln[k])
    # 4-byte bucket lists
    key = ((w32[:n] * np.uint64(0x1e35a7bd)) & np.uint64(0xFFFFFFFF)) >> np.uint64(17)
    bp, bd, bl = _nearest_same_key(key, query, DEPTH, lambda q, c: (w32[c] == w32[q]) & (q - c <= maxb[q]), w64, maxl)
    P.append(bp); D.append(bd); Ln.append(bl)
    P, D, Ln = (np.concatenate(x) for x in (P, D, Ln))
    P, D, Ln = _front(P, D, Ln, np.zeros(len(P), np.int64))
    for lv in range(levels):
        nb = 8 << lv
        h = _level_hash(w64, nb)[:n]
        lkey = h >> np.uint64(49)
        chk = h & np.uint64(0xFFFFFFFF)
        lq = query[n - query >= nb + 8]
        lp, ld, ll = _nearest_same_key(lkey, lq, LEVEL_DEPTH, lambda q, c: (chk[c] == chk[q]) & (q - c <= maxb[q]), w64, maxl)
        lp, ld, ll = _front(lp, ld, ll, np.zeros(len(lp), np.int64))
        P, D, Ln = _front(np.concatenate([P, lp]), np.concatenate([D, ld]), np.concatenate([Ln, ll]),
                          np.concatenate([np.zeros(len(P), np.int64), np.ones(len(lp), np.int64)]))
    first = np.searchsorted(P, P, side="left")
    slot = np.arange(len(P)) - first
    ent[P, slot, 0] = D
    ent[P, slot, 1] = Ln
    np.add.at(cnt, P, 1)
    return cnt, ent


def planted_input(lgwin: int, seed: int = 7) -> bytes:
    """PCG bytes with copies planted at the distances and lengths where the stage has an edge: distances 1-3, 15-17, 63-65
    (short ranges of q10 / q11) and 2^lgwin - 16 - 1 .. + 1 (the window limit: the last must not be found), lengths around
    the 4-byte bucket, the 8 / 16 / 32-byte levels and the 384-byte cap, overlapping runs, a zero run, and copies that end at
    the last bytes of the input."""
    rng = np.random.Generator(np.random.PCG64(seed))
    maxb = (1 << lgwin) - 16
    dists = [1, 2, 3, 15, 16, 17, 63, 64, 65, maxb - 1, maxb, maxb + 1]
    lens = [2, 3, 4, 7, 8, 9, 15, 16, 17, 23, 24, 39, 40, 41, 383, 384, 385]
    plan = [(d, ln) for d in dists for ln in lens]
    n = maxb + 2048 + sum(ln + 96 for _, ln in plan) + 4096 + 257 * 16 + 1025 * 24 + 64
    a = rng.integers(0, 256, n, dtype=np.uint8)
    p = maxb + 2048
    for d, ln in plan:
        for k in range(ln):  # byte by byte: d < ln overlaps
            a[p + k] = a[p + k - d]
        p += ln + 64 + int(rng.integers(0, 64))
    # a bucket filled exactly to its depth (256 records sharing 4 bytes; the last one queries them) and a level list filled
    # to its depth (1024 records sharing 8 bytes): only the farthest record continues like the query, two bytes further
    for depth, rec, head in ((256, 16, b"KEYQ"), (1024, 24, b"LEVELKEY")):
        h = len(head)
        for k in range(depth + 1):
            a[p:p + h] = np.frombuffer(head, dtype=np.uint8)
            if k in (0, depth):
                a[p + h:p + h + 2] = 0x5A
            elif a[p + h] == 0x5A:
                a[p + h] = 0x41
            p += rec
    a[p:p + 3000] = 0
    a[n - 100:n - 9] = a[n - 100 - 3000:n - 9 - 3000]  # ends at n - 9
    a[n - 9:] = a[n - 9 - 777:n - 777]  # ends at n
    return a.tobytes()


def window_part(hqn, hqm):
    """Splits stage output (hqn[n], hqm[n][16][2]) into its window entries as (count, entries[n][8][2]); asserts that the
    dictionary entries (bit 31 of the length word) all come after them."""
    n = len(hqn)
    j = np.arange(hqm.shape[1])
    live = j[None, :] < hqn[:, None].astype(np.int64)
    is_dict = (hqm[:, :, 1] >> 31).astype(bool) & live
    win = live & ~is_dict
    cnt = win.sum(axis=1)
    assert np.array_equal(win, j[None, :] < cnt[:, None]), "a dictionary entry precedes a window entry"
    ent = np.zeros((n, MAXW, 2), dtype=np.uint32)
    ent[:, :, :] = np.where(win[:, :MAXW, None], hqm[:, :MAXW, :], 0)
    return cnt.astype(np.uint8), ent


def first_difference(cnt_a, ent_a, cnt_b, ent_b):
    """None if both lists agree everywhere, else a report of the first position where they differ."""
    j = np.arange(MAXW)
    live_a = j[None, :] < cnt_a[:, None].astype(np.int64)
    live_b = j[None, :] < cnt_b[:, None].astype(np.int64)
    a = np.where(live_a[:, :, None], ent_a, 0)
    b = np.where(live_b[:, :, None], ent_b, 0)
    bad = (cnt_a != cnt_b) | (a != b).any(axis=(1, 2))
    if not bad.any():
        return None
    p = int(np.argmax(bad))
    fmt = lambda c, e: [(int(e[k, 0]), int(e[k, 1])) for k in range(int(c))]
    return "position %d (%d positions differ): expected %s, got %s" % (p, int(bad.sum()), fmt(cnt_a[p], ent_a[p]),
                                                                        fmt(cnt_b[p], ent_b[p]))

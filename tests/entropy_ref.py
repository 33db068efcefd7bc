"""Float64 / exact-integer reference of the entropy-coding decisions of quality 5..11, checked against the symbols of a stream.

The checks read a stream through tests/stream_audit.py (an RFC 7932 reader that knows the input) and share no code with the
encoder's headers, so a wrong threshold, off-by-one or tie rule in bro_split.cuh / bro_huffman.cuh / bro_common.cuh cannot be
reproduced on both sides.  What is restated, with the reference (dropbox/rust-brotli, src/enc/) cited:

  * the literal context decision: DecideOverLiteralContextModeling / ChooseContextMap / ShouldUseComplexStaticContextMap
    (encode.rs:1717-1927) in float64: 64-byte strides every 4096 bytes, the complex 13-context map only for a size hint of at
    least 1 MiB;
  * the greedy block splitter: BlockSplitterFinishBlock / ContextBlockSplitterFinishBlock / BrotliBuildMetaBlockGreedyInternal
    (metablock.rs:551-1021) in float64, replayed over the decoded symbols and guided by the stream's block switches;
  * the prefix codes: recounted histograms, the encoder's own count smoothing and length-limited Huffman rule (bro_huffman.cuh
    states them; they are integer rules, so the lengths must match exactly), Kraft completeness, and optimality against heapq
    Huffman or, where the 15-bit limit applies, package-merge;
  * the command and distance codes: ComputeDistanceCode (command.rs:48-68), CombineLengthCodes (:106-121) and
    PrefixEncodeCopyDistance (:134-173).

Entropies: BitsEntropy (bit_cost.rs:13-42) is max(Shannon bits, total count).  The reference evaluates it in f32 with
FastLog2u16, i.e. with each count truncated to u16; the encoder deliberately does not reproduce that truncation
(bro_split.cuh), so neither does this restatement.  The encoder computes entropies in Q16 fixed point: log2_q16 rounds
log2(x) to 1/65536 for x < 65536 and keeps only the top 16 bits of larger x (an underestimate of up to log2(1 + 2^-15) bits).
`entropy_terms` turns that into a rigorous bound on the error of every splitter margin; a decision whose float64 margin is
inside its bound is "ambiguous": the replay follows the stream there and counts it."""
import heapq
import math

import numpy as np

import stream_audit as sa

# ---- float64 entropies and the Q16 error bound ---------------------------------------------------------------------------
_LUT = np.floor(np.log2(np.maximum(np.arange(65536, dtype=np.float64), 1)) * 65536.0 + 0.5).astype(np.int64)  # lut[0] = 0


def log2_q16(x):
    """The encoder's fixed-point log2 (x >= 0, int64 array), restated to measure its distance from float64."""
    x = np.asarray(x, dtype=np.int64)
    s = np.maximum(np.frexp(np.maximum(x, 1).astype(np.float64))[1] - 16, 0)  # bit length - 16 for x >= 65536
    return (s << 16) + _LUT[x >> s]


def _err_per_unit(x):
    """Upper bound (bits) on |log2_q16(x) / 65536 - log2(x)|: half an LSB of rounding, plus the truncation of x >> s."""
    x = np.asarray(x, dtype=np.int64)
    s = np.maximum(np.frexp(np.maximum(x, 1).astype(np.float64))[1] - 16, 0)
    top = (x >> s).astype(np.float64)
    trunc = np.where(s > 0, np.log2(np.maximum(x, 1).astype(np.float64)) - s - np.log2(np.maximum(top, 1)), 0.0)
    return 0.5 / 65536 + trunc + 1e-12


def entropy_terms(h):
    """Per row of h (..., A) int64: (BitsEntropy in float64, its Q16 value / 65536, bound on |Q16 - float64|)."""
    h = np.asarray(h, dtype=np.int64)
    t = h.sum(axis=-1)
    hf = h.astype(np.float64)
    tf = t.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        xl = np.where(h > 0, hf * np.log2(np.maximum(hf, 1)), 0.0).sum(axis=-1)
        sh = np.where(t > 0, tf * np.log2(np.maximum(tf, 1)) - xl, 0.0)
    e64 = np.maximum(sh, tf)
    q = (t * log2_q16(t) - (h * log2_q16(h)).sum(axis=-1))
    eq = np.maximum(q, t << 16) / 65536.0
    bound = tf * _err_per_unit(t) + (hf * _err_per_unit(h)).sum(axis=-1) + 1e-9 * (1 + e64)
    return e64, eq, bound


def shannon64(h):
    h = np.asarray(h, dtype=np.float64)
    t = h.sum()
    return float(t * math.log2(t) - sum(c * math.log2(c) for c in h if c > 0)) if t > 0 else 0.0


# ---- literal context decision (encode.rs:1717-1927) ---------------------------------------------------------------------
SIMPLE2 = [0, 0, 1, 1] + [0] * 60                                # kStaticContextMapSimpleUTF8, encode.rs:1728
CONT3 = [1, 1, 2, 2] + [0] * 60                                  # kStaticContextMapContinuation, encode.rs:1723
COMPLEX13 = [11, 11, 12, 12, 0, 0, 0, 0, 1, 1, 9, 9, 2, 2, 2, 2, 1, 1, 1, 1, 8, 3, 3, 3, 1, 1, 1, 1, 2, 2, 2, 2, 8, 4, 4, 4,
             8, 7, 4, 4, 8, 0, 0, 0, 3, 3, 3, 3, 5, 5, 10, 5, 5, 5, 10, 5, 6, 6, 6, 6, 6, 6, 6, 6]  # encode.rs:1782
STATIC_MAPS = {1: [0] * 64, 2: SIMPLE2, 3: CONT3, 13: COMPLEX13}   # keyed by the number of contexts
MAP_NAMES = {1: "none", 2: "simple-2", 3: "continuation-3", 13: "complex-13"}


def context_decision(data, start, length, quality, size_hint):
    """(number of literal contexts, [(margin bits, bound bits)] of the comparisons that decided it).  Margins are in total
    bits over the sample (the reference divides both sides by the sample size)."""
    if quality < 5 or length < 64:
        return 1, []
    d = np.frombuffer(bytes(data), dtype=np.uint8)
    strides = [s for s in range(start, start + length - 63, 4096)]
    margins = []
    if size_hint >= 1 << 20:  # ShouldUseComplexStaticContextMap, encode.rs:1802-1871
        comb = np.zeros(32, dtype=np.int64)
        ctx = np.zeros((13, 32), dtype=np.int64)
        lut0, lut1 = sa.UTF8_LUT0, sa.UTF8_LUT1
        cm = np.array(COMPLEX13)
        for s in strides:
            w = d[s:s + 64]
            prev1, prev2, lit = w[1:63], w[0:62], w[2:64]
            c = cm[lut0[prev1] | lut1[prev2]]
            np.add.at(comb, lit >> 3, 1)
            np.add.at(ctx, (c, lit >> 3), 1)
        total = int(comb.sum())
        s1, b1 = _shannon_with_bound(comb)
        s2, b2 = 0.0, 0.0
        for i in range(13):
            a, b = _shannon_with_bound(ctx[i])
            s2 += a
            b2 += b
        m_a = s2 - 3.0 * total            # entropy[2] > 3.0
        m_b = (s1 - s2) - 0.2 * total     # entropy[1] - entropy[2] < 0.2
        margins += [(m_a, b2), (m_b, b1 + b2)]
        if not (m_a > 0 or m_b < 0):
            return 13, margins
    lut = np.array([0, 0, 1, 2])
    big = np.zeros(9, dtype=np.int64)     # DecideOverLiteralContextModeling, encode.rs:1895-1919
    for s in strides:
        w = lut[d[s:s + 64] >> 6]
        np.add.at(big, w[:-1] * 3 + w[1:], 1)
    mono = np.array([big[0::3].sum(), big[1::3].sum(), big[2::3].sum()])
    two = np.array([big[i::6].sum() for i in range(6)])
    e1, b1 = _shannon_with_bound(mono)
    e2a, b2a = _shannon_with_bound(two[:3])
    e2b, b2b = _shannon_with_bound(two[3:])
    e2, b2 = e2a + e2b, b2a + b2b
    e3, b3 = 0.0, 0.0
    for i in range(3):
        a, b = _shannon_with_bound(big[3 * i:3 * i + 3])
        e3 += a
        b3 += b
    if quality < 7:
        e3, b3 = e1 * 10, b1 * 10
    total = float(mono.sum())
    ma, mb, mc = (e1 - e2) - 0.2 * total, (e1 - e3) - 0.2 * total, (e2 - e3) - 0.02 * total  # ChooseContextMap :1771-1779
    margins += [(ma, b1 + b2), (mb, b1 + b3)]
    if ma < 0 and mb < 0:
        return 1, margins
    margins.append((mc, b2 + b3))
    return (2 if mc < 0 else 3), margins


def _shannon_with_bound(h):
    h = np.asarray(h, dtype=np.int64)
    t = int(h.sum())
    if t == 0:
        return 0.0, 0.0
    s = shannon64(h)
    b = t * float(_err_per_unit([t])[0]) + float((h * _err_per_unit(h)).sum()) + 1e-9 * (1 + s)
    return s, b


def stream_context_map(mb):
    """Number of contexts of the static map the stream's literal context map encodes (1, 2, 3, 13), or raise."""
    nt = mb.ntypes[0]
    for nctx in (1, 2, 3, 13):
        if mb.nlit_trees != nt * nctx:
            continue
        want = [t * nctx + STATIC_MAPS[nctx][c] for t in range(nt) for c in range(64)]
        if mb.lit_cmap == want:
            return nctx
    raise AssertionError("literal context map is none of the static maps (%d types, %d trees)" % (nt, mb.nlit_trees))


# ---- prefix codes -------------------------------------------------------------------------------------------------------
def smooth_counts(counts):
    """bro_huffman.cuh huff_smooth_counts, restated: runs of counts within (c - m)^2 <= 4 m + slack of the running mean,
    at least 4 long and at least 1/4 in use, are flattened to their rounded mean; codes with < 16 used symbols are left."""
    c = [int(x) for x in counts]
    used, total = sum(1 for x in c if x), sum(c)
    if used < 16:
        return c
    slack = min(16, total >> 8)
    length = len(c)
    while length and c[length - 1] == 0:
        length -= 1
    i = 0
    while i < length:
        s, n, nz = c[i], 1, int(c[i] != 0)
        j = i + 1
        while j < length:
            dev = c[j] * n - s
            if dev * dev > n * (4 * s + slack * n):
                break
            s += c[j]
            nz += c[j] != 0
            n += 1
            j += 1
        if n >= 4 and nz * 4 >= n:
            mean = max(1, (s + n // 2) // n)
            c[i:j] = [mean] * (j - i)
        i = j
    return c


def huffman_lengths(counts, limit=15):
    """(lengths, unlimited maximum depth, repaired) of bro_huffman.cuh's rule, restated: a two-queue merge over the used
    symbols sorted by (count, symbol), a leaf winning ties; if deeper than `limit`, clamp, lengthen the least frequent
    symbols below the limit until the Kraft sum fits, then shorten the most frequent while the slack allows it."""
    used = sorted((c, s) for s, c in enumerate(counts) if c)
    lengths = [0] * len(counts)
    n = len(used)
    if n == 0:
        return lengths, 0, False
    if n == 1:
        lengths[used[0][1]] = 1
        return lengths, 1, False
    w = [c for c, _ in used] + [0] * (n - 1)
    parent = [0] * (2 * n - 1)
    leaf, inner, nxt = 0, n, n
    for _ in range(n - 1):
        pick = []
        for _ in range(2):
            if leaf < n and (inner >= nxt or w[leaf] <= w[inner]):
                pick.append(leaf)
                leaf += 1
            else:
                pick.append(inner)
                inner += 1
        w[nxt] = w[pick[0]] + w[pick[1]]
        parent[pick[0]] = parent[pick[1]] = nxt
        nxt += 1
    depth = [0] * (2 * n - 1)
    for v in range(2 * n - 3, -1, -1):
        depth[v] = depth[parent[v]] + 1
    nd = depth[:n]
    maxd = max(nd)
    repaired = maxd > limit
    if repaired:
        excess = -(1 << limit)
        for i in range(n):
            nd[i] = min(nd[i], limit)
            excess += 1 << (limit - nd[i])
        i = 0
        while excess > 0 and i < n:
            if nd[i] >= limit:
                i += 1
                continue
            excess -= 1 << (limit - nd[i] - 1)
            nd[i] += 1
        for i in range(n - 1, -1, -1):
            if excess >= 0:
                break
            while nd[i] > 1 and (1 << (limit - nd[i])) <= -excess and (i + 1 == n or nd[i] - 1 >= nd[i + 1]):
                excess += 1 << (limit - nd[i])
                nd[i] -= 1
    for (c, s), l in zip(used, nd):
        lengths[s] = l
    return lengths, maxd, repaired


def huffman_cost(counts):
    """Optimal unrestricted prefix-code cost sum(count * length) by heapq Huffman."""
    h = [c for c in counts if c]
    if len(h) <= 1:
        return sum(h)
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        a = heapq.heappop(h) + heapq.heappop(h)
        cost += a
        heapq.heappush(h, a)
    return cost


def package_merge_cost(counts, limit=15):
    """Optimal cost sum(count * length) over codes with lengths <= limit (package-merge, Larmore and Hirschberg 1990)."""
    leaves = sorted(c for c in counts if c)
    n = len(leaves)
    if n <= 1:
        return sum(leaves)
    # each item: (weight, number of leaves of each symbol it contains) kept as a count vector over the sorted leaves
    base = [(w, np.eye(1, n, i, dtype=np.int64)[0]) for i, w in enumerate(leaves)]
    cur = list(base)
    for _ in range(limit - 1):
        pk = [(cur[2 * k][0] + cur[2 * k + 1][0], cur[2 * k][1] + cur[2 * k + 1][1]) for k in range(len(cur) // 2)]
        cur = sorted(base + pk, key=lambda x: x[0])
    lengths = sum(v for _, v in cur[:2 * n - 2])
    return int(np.dot(lengths, leaves))


def kraft_sum(lengths):
    return sum(1 << (15 - l) for l in lengths if l)


def check_code(code, counts, what, smooth, stats):
    """Compare one prefix code of the stream with the recount `counts` of the symbols read with it.  Returns None or a
    description of the first difference; updates `stats` (repaired codes, gaps to package-merge)."""
    counts = [int(x) for x in counts]
    sm = smooth_counts(counts) if smooth else counts
    used = [s for s, c in enumerate(sm) if c]
    got = code.lengths
    if len(used) <= 1:
        want_sym = used[0] if used else 0
        if code.kind != "single" or code.simple_symbols[0] != want_sym:
            return "%s: expected the one-symbol code of symbol %d, stream has a %s code" % (what, want_sym, code.kind)
        return None
    want, maxd, repaired = huffman_lengths(sm)
    for s, c in enumerate(counts):
        if c and not got[s]:
            return "%s, symbol %d: used %d times, has no code" % (what, s, c)
    for s in range(len(sm)):
        if bool(got[s]) != bool(sm[s]):
            return "%s, symbol %d: count %d after smoothing, stream length %d" % (what, s, sm[s], got[s])
    if max(got) > 15 or kraft_sum(got) != 1 << 15:
        return "%s: lengths exceed 15 or the Kraft sum is %d / 32768" % (what, kraft_sum(got))
    if len(used) <= 4:
        if code.kind != "simple":
            return "%s: %d used symbols but a %s code" % (what, len(used), code.kind)
        order = sorted(used, key=lambda s: (got[s], s))
        if code.simple_symbols != order:
            return "%s: simple code lists %s, expected %s" % (what, code.simple_symbols, order)
    elif code.kind != "complex":
        return "%s: %d used symbols but a %s code" % (what, len(used), code.kind)
    for s in used:
        if got[s] != want[s]:
            return "%s, symbol %d: stream length %d, reference %d (count %d, smoothed %d)" % (what, s, got[s], want[s], counts[s], sm[s])
    cost = sum(c * l for c, l in zip(sm, got))
    if not repaired:
        opt = huffman_cost(sm)
        if cost != opt:
            return "%s: cost %d bits, Huffman optimum %d" % (what, cost, opt)
    else:
        opt = package_merge_cost(sm)
        stats["repaired"] += 1
        stats["max_unlimited_depth"] = max(stats["max_unlimited_depth"], maxd)
        gap = (cost - opt) / opt
        stats["gaps"].append((cost - opt, gap))
        if cost < opt or gap > REPAIR_GAP_MAX:
            return "%s: cost %d bits, package-merge optimum %d (gap %.4f %%)" % (what, cost, opt, 100 * gap)
    stats["codes"] += 1
    return None


REPAIR_GAP_MAX = 0.01  # the Kraft repair may cost at most 1 % over the length-limited optimum (measured gaps: README)


# ---- per-metablock recount and code checks ------------------------------------------------------------------------------
def blocklen_code(n):
    for c in range(25, -1, -1):
        if n >= sa.BL_OFFSET[c]:
            return c
    raise ValueError(n)


def recount(mb):
    """Exact histograms of the symbols read with each prefix code: literal trees, command codes (per block type), distance
    trees (explicit distances only), block-type and block-count codes per category."""
    lit = np.bincount(mb.lit_trees.astype(np.int64) * 256 + np.frombuffer(mb.lit_bytes, dtype=np.uint8),
                      minlength=256 * mb.nlit_trees).reshape(mb.nlit_trees, 256) if len(mb.lit_bytes) else \
        np.zeros((mb.nlit_trees, 256), dtype=np.int64)
    cmd = np.zeros((mb.ntypes[1], 704), dtype=np.int64)
    dist = np.zeros((mb.ndist_trees, mb.dist_alphabet), dtype=np.int64)
    for c in mb.cmds:
        cmd[c[4], c[3]] += 1
        if c[5] >= 0:
            dist[mb.dist_cmap[4 * c[7] + c[8]], c[5]] += 1
    types, lens = [], []
    for cat in range(3):
        th = np.zeros(mb.ntypes[cat] + 2, dtype=np.int64)
        lh = np.zeros(26, dtype=np.int64)
        for k, (_, tc, _, ln) in enumerate(mb.switches[cat]):
            if k:
                th[tc] += 1
            if ln is not None:
                lh[blocklen_code(ln)] += 1
        types.append(th)
        lens.append(lh)
    return lit, cmd, dist, types, lens


def check_codes(mb, where, stats, smooth=True):
    lit, cmd, dist, types, lens = recount(mb)
    for t in range(mb.nlit_trees):
        r = check_code(mb.lit_codes[t], lit[t], "%s, literal tree %d" % (where, t), smooth, stats)
        if r:
            return r
    for t in range(mb.ntypes[1]):
        r = check_code(mb.cmd_codes[t], cmd[t], "%s, command code %d" % (where, t), smooth, stats)
        if r:
            return r
    for t in range(mb.ndist_trees):
        r = check_code(mb.dist_codes[t], dist[t], "%s, distance tree %d" % (where, t), smooth, stats)
        if r:
            return r
    for cat, name in enumerate(("literal", "command", "distance")):
        if mb.ntypes[cat] > 1:
            for code, h, kind in ((mb.type_code[cat], types[cat], "block-type"), (mb.len_code[cat], lens[cat], "block-count")):
                r = check_code(code, h, "%s, %s %s code" % (where, name, kind), False, stats)
                if r:
                    return r
    return None


# ---- command and distance codes (command.rs) ----------------------------------------------------------------------------
def insert_code(n):
    return max(c for c in range(24) if sa.INS_BASE[c] <= n)


def copy_code(n):
    return max(c for c in range(24) if sa.COPY_BASE[c] <= n)


def command_symbol(ins, cpy, implicit):
    """CombineLengthCodes (command.rs:106-121)."""
    ic, cc = insert_code(ins), copy_code(cpy)
    bits64 = (cc & 7) | ((ic & 7) << 3)
    if implicit and ic < 8 and cc < 16:
        return bits64 if cc < 8 else bits64 | 64
    sub = 2 * ((cc >> 3) + 3 * (ic >> 3))
    return ((sub << 5) + 0x40 + ((0x520D40 >> sub) & 0xC0)) | bits64


def distance_code(distance, max_distance, ring):
    """ComputeDistanceCode (command.rs:48-68); ring entries that are None are unknown to the encoder."""
    if distance <= max_distance:
        r = [x if x is not None else -(1 << 40) for x in ring]
        o0, o1 = distance + 3 - r[0], distance + 3 - r[1]
        if distance == r[0]:
            return 0
        if distance == r[1]:
            return 1
        if 0 <= o0 < 7:
            return (0x09750468 >> (4 * o0)) & 0xF
        if 0 <= o1 < 7:
            return (0x0FDB1ACE >> (4 * o1)) & 0xF
        if distance == r[2]:
            return 2
        if distance == r[3]:
            return 3
    return distance + 15


def prefix_encode_distance(code, npostfix, ndirect):
    """PrefixEncodeCopyDistance (command.rs:134-173): (symbol, extra bits value)."""
    if code < 16 + ndirect:
        return code, 0
    dist = (1 << (npostfix + 2)) + code - 16 - ndirect
    bucket = dist.bit_length() - 2
    postfix = dist & ((1 << npostfix) - 1)
    prefix = (dist >> bucket) & 1
    offset = (2 + prefix) << bucket
    nbits = bucket - npostfix
    return 16 + ndirect + ((2 * (nbits - 1) + prefix) << npostfix) + postfix, (dist - offset) >> npostfix


def check_commands(mb, lgwin, where):
    """Every command's symbol and distance code against command.rs.  The encoder starts each metablock with an unknown
    distance cache (bro_finalize.cuh: metablocks are independent), so only ring entries pushed inside the metablock count.
    Dictionary references must be explicit: ComputeDistanceCode's max_distance guard gives them distance + 15.  The
    encoder's compute_distance_code has no such guard, which cannot matter: finalize_unit sends dictionary references as
    distance + 15 without calling it, and a window copy never exceeds max_distance."""
    max_backward = (1 << lgwin) - 16
    n = len(mb.cmds)
    for k, (pos, ins, cpy, cs, _, dsym, dextra, _, _, distance, is_dict, ring, pushes) in enumerate(mb.cmds):
        if distance is None:  # ends the metablock inside its insert: InitInsertCommand, command.rs:38-44
            if k != n - 1 or cs != command_symbol(ins, 4, False):
                return "%s, command %d at %d: insert-only command has symbol %d, expected %d" % (where, k, pos, cs, command_symbol(ins, 4, False))
            continue
        max_distance = min(pos + ins, max_backward)
        known = [ring[i] if i < pushes else None for i in range(4)]
        want = distance_code(distance, max_distance, known)
        got = 0 if cs < 128 else (dsym if dsym < 16 else distance + 15)
        if got != want:
            return "%s, command %d at %d: distance %d sent as code %d, shortest is %d (ring %s)" % (where, k, pos, distance, got, want, known)
        want_cs = command_symbol(ins, cpy, want == 0)
        if cs != want_cs:
            return "%s, command %d at %d: command symbol %d, expected %d (insert %d, copy %d, distance code %d)" % (
                where, k, pos, cs, want_cs, ins, cpy, want)
        if cs >= 128:
            ws, we = prefix_encode_distance(want, mb.npostfix, mb.ndirect)
            if (dsym, dextra) != (ws, we):
                return "%s, command %d at %d: distance symbol %d extra %d, expected %d extra %d" % (where, k, pos, dsym, dextra, ws, we)
    return None


# ---- the greedy block splitter (metablock.rs:551-1021), guided replay ----------------------------------------------------
SPLIT_PARAMS = {0: (256, 512, 400.0), 1: (704, 1024, 500.0), 2: (64, 512, 100.0)}  # metablock.rs:885-928


def category_symbols(mb, cat, nctx):
    """Symbol sequence the splitter of `cat` sees, as indices ctx * A + symbol."""
    if cat == 0:
        cls = np.array(STATIC_MAPS[nctx], dtype=np.int64)[mb.lit_ctx] if nctx > 1 else np.zeros(len(mb.lit_ctx), dtype=np.int64)
        return cls * 256 + np.frombuffer(mb.lit_bytes, dtype=np.uint8)
    if cat == 1:
        return np.array([c[3] for c in mb.cmds], dtype=np.int64)
    return np.array([c[5] for c in mb.cmds if c[5] >= 0], dtype=np.int64)


def replay_split(mb, cat, nctx, where, report):
    """Replays the greedy splitter of one category over the stream's symbols.  At every FinishBlock the float64 margins
    diff0 - thr, diff1 - thr and diff0 - 20 - diff1 are computed with a bound on their Q16 error; the stream's decision must
    be possible under every margin outside its bound.  Returns None or a description of the first disagreement;
    `report` collects decision counts, ambiguous cases and the largest Q16-vs-float64 margin error seen."""
    A, min_block, thr = SPLIT_PARAMS[cat]
    max_types = 256 // nctx if nctx > 1 else 256
    HA = nctx * A
    syms = category_symbols(mb, cat, nctx)
    count = len(syms)
    nt = mb.ntypes[cat]
    blocks = [(t, ln) for _, _, t, ln in mb.switches[cat]] if nt > 1 else [(0, float("inf"))]
    hist = []                      # per type: (nctx, A) int64
    le = [None, None]              # last entropies: (float64 per ctx, q16 per ctx, bound per ctx)
    last_type = [0, 0]
    num_types = 0
    merge_count = 0
    target = min_block
    b, acc = 0, 0                  # stream block and symbols of it accounted for
    pos = 0

    def ent(h):
        return entropy_terms(h)

    def finish(cur, bs, at):
        nonlocal num_types, merge_count, target, b, acc
        if num_types == 0:
            hist.append(cur)
            e = ent(cur)
            le[0] = le[1] = e
            num_types = 1
            acc = bs
            report["decisions"] += 1
            return None
        ec = ent(cur)
        comb = [cur + hist[last_type[0]], cur + hist[last_type[1]]]
        e0, e1 = ent(comb[0]), ent(comb[1])
        d0 = float((e0[0] - ec[0] - le[0][0]).sum())
        d1 = float((e1[0] - ec[0] - le[1][0]).sum())
        q0 = float((e0[1] - ec[1] - le[0][1]).sum())
        q1 = float((e1[1] - ec[1] - le[1][1]).sum())
        b0 = float((e0[2] + ec[2] + le[0][2]).sum())
        b1 = float((e1[2] + ec[2] + le[1][2]).sum())
        margins = [(d0 - thr, q0 - thr, b0), (d1 - thr, q1 - thr, b1), (d0 - 20.0 - d1, q0 - 20.0 - q1, b0 + b1)]
        for m64, mq, bd in margins:
            err = abs(mq - m64)
            report["max_margin_error"] = max(report["max_margin_error"], err)
            if err > bd:
                return "%s: Q16 margin error %.6g exceeds its bound %.6g" % (at, err, bd)
        # the stream's decision
        if acc < blocks[b][1]:
            action = "merge"
        elif acc == blocks[b][1] and b + 1 < len(blocks):
            t = blocks[b + 1][0]
            action = "new" if t == num_types else "second" if t == last_type[1] else None
            if action is None:
                return "%s: block %d has type %d, neither new (%d) nor second-last (%d)" % (at, b + 1, t, num_types, last_type[1])
        else:
            return "%s: stream block %d ends at %d symbols, replay has %d" % (at, b, blocks[b][1], acc)
        # which decisions float64 allows: a comparison inside its bound may go either way
        def can(m, bd, want_positive):
            return (m[0] > 0) == want_positive or abs(m[0]) <= bd

        room = num_types < max_types
        new_ok = room and can(margins[0], b0, True) and can(margins[1], b1, True)
        not_new_ok = (not room) or can(margins[0], b0, False) or can(margins[1], b1, False)
        second_ok = not_new_ok and can(margins[2], b0 + b1, True)
        merge_ok = not_new_ok and can(margins[2], b0 + b1, False)
        allowed = {"new": new_ok, "second": second_ok, "merge": merge_ok}
        f_new = room and d0 > thr and d1 > thr
        f_action = "new" if f_new else "second" if d1 < d0 - 20.0 else "merge"
        ambiguous = sum(allowed.values()) > 1
        report["decisions"] += 1
        report["ambiguous"] += ambiguous
        report["disagree_in_bound"] += (f_action != action)
        report[action] += 1
        if not allowed[action]:
            return "%s: stream %s, float64 %s (diff0 %.3f, diff1 %.3f bits, threshold %g, %d types; bounds %.3g / %.3g)" % (
                at, action, f_action, d0, d1, thr, num_types, b0, b1)
        if action == "new":
            hist.append(cur)
            last_type[1], last_type[0] = last_type[0], num_types
            le[1], le[0] = le[0], ec
            num_types += 1
            merge_count = 0
            target = min_block
            b += 1
            acc = bs
        elif action == "second":
            last_type[0], last_type[1] = last_type[1], last_type[0]
            hist[last_type[0]] = comb[1]
            le[1], le[0] = le[0], e1
            merge_count = 0
            target = min_block
            b += 1
            acc = bs
        else:
            hist[last_type[0]] = comb[0]
            le[0] = e0
            if num_types == 1:
                le[1] = e0
            merge_count += 1
            if merge_count > 1:
                target += min_block
            acc += bs
        return None

    while True:
        take = min(target, count - pos)
        chunk = syms[pos:pos + take]
        cur = np.bincount(chunk, minlength=HA).reshape(nctx, A).astype(np.int64)
        at = "%s, %s splitter, symbol %d" % (where, ("literal", "command", "distance")[cat], pos + take)
        pos += take
        if take == target:
            r = finish(cur, target, at)
            if r:
                return r
            if pos == count:
                r = finish(np.zeros((nctx, A), dtype=np.int64), min_block, at + " (final)")
                break
        else:
            r = finish(cur, max(take, min_block), at + " (final)")
            break
    if r:
        return r
    if num_types != nt:
        return "%s, %s splitter: replay ends with %d types, stream has %d" % (where, ("literal", "command", "distance")[cat], num_types, nt)
    if nt > 1 and (b != len(blocks) - 1 or acc != blocks[b][1]):
        return "%s, %s splitter: replay ends in block %d at %d, stream has %d blocks, last of %d" % (
            where, ("literal", "command", "distance")[cat], b, acc, len(blocks), blocks[-1][1])
    return None


def new_report():
    return {"decisions": 0, "ambiguous": 0, "disagree_in_bound": 0, "new": 0, "second": 0, "merge": 0, "max_margin_error": 0.0,
            "ctx_ambiguous": 0, "codes": 0, "repaired": 0, "max_unlimited_depth": 0, "gaps": [], "metablocks": 0, "maps": {}}


def audit_stream(stream, data, quality, size_hint=0, report=None):
    """All checks on one stream of `data`; raises AssertionError with a position report.  Returns the report."""
    report = report if report is not None else new_report()
    lgwin, mbs = sa.audit(stream, data)
    hint = size_hint or len(data)
    for i, mb in enumerate(mbs):
        if mb.raw:
            continue
        where = "metablock %d" % i
        report["metablocks"] += 1
        if quality < 10:
            nctx = stream_context_map(mb)
            report["maps"][MAP_NAMES[nctx]] = report["maps"].get(MAP_NAMES[nctx], 0) + 1
            if nctx > 1:
                assert all(m == 2 for m in mb.cmodes), "%s: static context maps need UTF8 mode, stream has %s" % (where, mb.cmodes)
            want, margins = context_decision(data, mb.start, mb.mlen, quality, hint)
            if want != nctx:
                assert any(abs(m) <= bd for m, bd in margins), "%s: %s literal context map, float64 chooses %s (margins %s)" % (
                    where, MAP_NAMES[nctx], MAP_NAMES[want], ["%.2f+-%.2g" % mb_ for mb_ in margins])
            report["ctx_ambiguous"] += any(abs(m) <= bd for m, bd in margins)
            assert (mb.npostfix, mb.ndirect) == (0, 0), "%s: NPOSTFIX / NDIRECT %d / %d below quality 10" % (where, mb.npostfix, mb.ndirect)
            for cat in range(3):
                r = replay_split(mb, cat, nctx if cat == 0 else 1, where, report)
                assert r is None, r
        r = check_codes(mb, where, report)
        assert r is None, r
        r = check_commands(mb, lgwin, where)
        assert r is None, r
    return report


# ---- inputs that reach the edges ----------------------------------------------------------------------------------------
def _fib_literals(rng, nsym=26, base=0x80):
    f = [1, 1]
    while len(f) < nsym:
        f.append(f[-1] + f[-2])
    d = np.repeat(np.arange(base, base + nsym, dtype=np.uint8), f)
    rng.shuffle(d)
    return d.tobytes()


def _few_symbols(rng, k, n, base=0xA0):
    return (base + rng.integers(0, k, n, dtype=np.uint8)).astype(np.uint8).tobytes()


def _tolerance_runs(rng, slack=16):
    """Literal counts at the smoothing tolerance: after a run with mean m, counts m +- (isqrt(4 m + slack) and one more),
    and sparse runs with exactly 1 / 4 of their symbols in use."""
    counts = np.zeros(256, dtype=np.int64)
    m = 100
    for k, s in enumerate(range(0x40, 0x80, 8)):
        r = int(math.isqrt(4 * m + slack)) + (k % 3 - 1)
        counts[s:s + 7] = m
        counts[s + 7] = m + r if k % 2 else max(1, m - r)
    for s in range(0xC0, 0x100, 16):
        counts[s:s + 16:4] = 2         # 4 of 16 in use
    d = np.repeat(np.arange(256, dtype=np.uint8), counts)
    rng.shuffle(d)
    return d.tobytes()


def _de_bruijn(k, n, base):
    """De Bruijn sequence B(k, n) over bytes base .. base + k - 1: no n-gram repeats, so nothing to copy."""
    a, seq = [0] * (k * n), []

    def db(t, p):
        if t > n:
            if n % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return bytes(base + x for x in seq)


def _segments(rng, text, json, nseg, seglen):
    """Alternating text / random / JSON segments and segments over distinct byte subsets (new block types), lengths
    around multiples of the 512-symbol minimum block."""
    out = []
    for k in range(nseg):
        n = seglen * (1 + k % 3) + (k % 5 - 2)
        kind = k % 4
        if kind == 0:
            o = int(rng.integers(0, len(text) - n))
            out.append(text[o:o + n])
        elif kind == 1:
            out.append(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
        elif kind == 2:
            o = int(rng.integers(0, len(json) - n))
            out.append(json[o:o + n])
        else:
            sub = rng.choice(256, 12, replace=False).astype(np.uint8)
            out.append(sub[rng.integers(0, 12, n)].tobytes())
    return b"".join(out)


def planted_cases(golden, datagen, big=False):
    """(name, data, quality, lgwin, size hint) cases, each reaching an edge of the entropy stage."""
    rng = np.random.default_rng(7)
    text = datagen.enwik_like(1_200_000, seed=3)
    json = datagen.json_logs(600_000, seed=5)
    cases = [
        ("fibonacci-26", _fib_literals(rng) + text[:20000], 5, 22, 0),
        ("fibonacci-30", _fib_literals(rng, 30, 0x40), 7, 22, 0),
        ("tolerance", _tolerance_runs(rng) + _tolerance_runs(rng, 4), 5, 22, 0),
    ]
    for k in (1, 2, 3, 4, 15, 16, 17):
        cases.append(("%d-symbols" % k, _few_symbols(rng, k, 3000) + bytes(range(0x30, 0x30 + k)) * 3, 5, 22, 0))
    cases += [
        ("segments", _segments(rng, text, json, 120, 512), 5, 22, 0),
        ("segments-q9", _segments(rng, text, json, 60, 1024), 9, 16, 0),
        ("type-cap", _segments(rng, text, json, 1100, 512), 5, 22, (1 << 20) - 1),
        ("type-cap-complex13", _segments(rng, text, json, 200, 520)[:200_000] + text[:300_000], 5, 22, 1 << 20),
        ("no-distances", _de_bruijn(16, 4, 0x90), 5, 22, 0),
        ("incompressible", rng.integers(0, 256, 300_000, dtype=np.uint8).tobytes() + text[:50000], 5, 22, 0),
        ("hint-below-1MiB", text[:600_000], 5, 22, (1 << 20) - 1),
        ("hint-1MiB", text[:600_000], 5, 22, 1 << 20),
        ("hint-1MiB-q7", text[:600_000], 7, 22, 1 << 20),
    ]
    for name in ("alice29.txt", "asyoulik.txt", "random_then_unicode", "compressed_file", "quickfox_repeated"):
        for q in (5, 7, 9):
            for w in (16, 22):
                cases.append(("%s-q%d-w%d" % (name, q, w), golden(name), q, w, 0))
    cases.append(("json-q9", datagen.json_logs(1_500_000), 9, 22, 0))
    if big:
        cases.append(("two-4MiB-metablocks", datagen.enwik_like((8 << 20) + 100_000, seed=9), 5, 22, 0))
    return cases


def hq_cases(golden, datagen):
    return [("alice29-q%d" % q, golden("alice29.txt"), q, 22, 0) for q in (10, 11)] + \
           [("asyoulik-q10-w16", golden("asyoulik.txt"), 10, 16, 0), ("json-q11", datagen.json_logs(300_000), 11, 22, 0),
            ("fibonacci-q10", _fib_literals(np.random.default_rng(7)), 10, 22, 0)]

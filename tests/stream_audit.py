"""Symbol-level audit reader of a brotli stream (RFC 7932), given the input it must decode to.

An independent decoder: it shares no code with the encoder's headers or the CPU model, and it keeps what a size-only
decoder throws away.  For every compressed metablock it returns the header (MLEN, NBLTYPES and the block-type / block-count
codes per category, context modes, context maps, NPOSTFIX / NDIRECT, the code lengths of every prefix code and, for simple
codes, the symbol order) and a record of every symbol of the body:

  * commands: position of the first literal, insert / copy length, command symbol and its block type, the distance symbol
    and extra bits and its block type and context (or "implicit"), the distance, whether it is a dictionary reference, and
    the distance ring in force before the command together with how many of its entries were pushed inside this metablock;
  * literals: value, block type, 6-bit context id and the prefix code (tree) it was read with;
  * block switches per category: symbol rank at which the block starts, type code, the type it selects, block count.

Literal contexts are computed from the known input, and every byte the stream produces (literals, window copies and
static-dictionary words, transformed through the system's libbrotlicommon) is checked against that input as it is
produced, so nothing is audited on a stream that was mis-read.  Uncompressed and metadata metablocks are recognised and
skipped (an uncompressed one is recorded with `raw=True`).  Symbols are decoded through tables indexed by the next
`maxlen` bits of the stream, not bit by bit."""
import ctypes

import numpy as np

K_CL_ORDER = [1, 2, 3, 4, 0, 5, 17, 6, 16, 7, 8, 9, 10, 11, 12, 13, 14, 15]
INS_BASE = [0, 1, 2, 3, 4, 5, 6, 8, 10, 14, 18, 26, 34, 50, 66, 98, 130, 194, 322, 578, 1090, 2114, 6210, 22594]
INS_EXTRA = [0, 0, 0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 7, 8, 9, 10, 12, 14, 24]
COPY_BASE = [2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 14, 18, 22, 30, 38, 54, 70, 102, 134, 198, 326, 582, 1094, 2118]
COPY_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 7, 8, 9, 10, 24]
BL_OFFSET = [1, 5, 9, 13, 17, 25, 33, 41, 49, 65, 81, 97, 113, 145, 177, 209, 241, 305, 369, 497, 753, 1265, 2289, 4337, 8433, 16625]
BL_NBITS = [2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 6, 6, 7, 8, 9, 10, 11, 12, 13, 24]
# RFC 7932 section 5: insert / copy code offsets of the 11 cells of the command alphabet
CELL_INS = [0, 0, 0, 0, 8, 8, 0, 16, 8, 16, 16]
CELL_COPY = [0, 8, 0, 8, 0, 8, 16, 0, 16, 8, 16]
SHORT_IDX = [0, 1, 2, 3, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1]
SHORT_OFF = [0, 0, 0, 0, -1, 1, -2, 2, -3, 3, -1, 1, -2, 2, -3, 3]


class StreamError(ValueError):
    pass


# ---- literal context ids (RFC 7932 section 7.1), as tables over all (p1, p2) -------------------------------------------
def _utf8_lut0():
    a = [0, 0, 0, 0, 0, 0, 0, 0, 0, 4, 4, 0, 0, 4, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 8, 12, 16, 12, 12,
         20, 12, 16, 24, 28, 12, 12, 32, 12, 36, 12, 44, 44, 44, 44, 44, 44, 44, 44, 44, 44, 32, 32, 24, 40, 28, 12, 12, 48,
         52, 52, 52, 48, 52, 52, 52, 48, 52, 52, 52, 52, 52, 48, 52, 52, 52, 52, 52, 48, 52, 52, 52, 52, 52, 24, 12, 28, 12,
         12, 12, 56, 60, 60, 60, 56, 60, 60, 60, 56, 60, 60, 60, 60, 60, 56, 60, 60, 60, 60, 60, 56, 60, 60, 60, 60, 60, 24,
         12, 28, 12, 0]
    return a + [c & 1 for c in range(128, 192)] + [2 + (c & 1) for c in range(192, 256)]


def _utf8_lut1():
    out = []
    for c in range(256):
        if c < 32 or c in (32, 127) or 128 <= c < 224:
            out.append(0)
        elif c >= 224:
            out.append(2)
        elif 48 <= c <= 57 or 65 <= c <= 90:
            out.append(2)
        elif 97 <= c <= 122:
            out.append(3)
        else:
            out.append(1)
    return out


def _signed3(c):
    return 0 if c == 0 else 1 if c < 16 else 2 if c < 64 else 3 if c < 128 else 4 if c < 192 else 5 if c < 240 else 6 if c < 255 else 7


UTF8_LUT0 = np.array(_utf8_lut0(), dtype=np.uint8)
UTF8_LUT1 = np.array(_utf8_lut1(), dtype=np.uint8)
SIGNED_LUT = np.array([_signed3(c) for c in range(256)], dtype=np.uint8)


def context_ids(data, mode):
    """6-bit literal context id of every position of `data` for context mode 0..3 (p1, p2 = 0 before the start)."""
    d = np.frombuffer(bytes(data), dtype=np.uint8)
    p1 = np.concatenate([[0], d[:-1]]).astype(np.uint8) if len(d) else d
    p2 = np.concatenate([[0, 0], d[:-2]]).astype(np.uint8)[:len(d)] if len(d) else d
    if mode == 0:
        return p1 & 0x3F
    if mode == 1:
        return p1 >> 2
    if mode == 2:
        return UTF8_LUT0[p1] | UTF8_LUT1[p2]
    return (SIGNED_LUT[p1] << 3) | SIGNED_LUT[p2]


# ---- static dictionary (system libbrotlicommon) ----------------------------------------------------------------------------
_DICT = None


def _dictionary():
    global _DICT
    if _DICT is None:
        class D(ctypes.Structure):
            _fields_ = [("size_bits_by_length", ctypes.c_uint8 * 32), ("offsets_by_length", ctypes.c_uint32 * 32),
                        ("data_size", ctypes.c_size_t), ("data", ctypes.POINTER(ctypes.c_uint8))]
        lib = ctypes.CDLL("libbrotlicommon.so.1")
        lib.BrotliGetDictionary.restype = ctypes.POINTER(D)
        lib.BrotliGetTransforms.restype = ctypes.c_void_p
        lib.BrotliTransformDictionaryWord.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        lib.BrotliTransformDictionaryWord.restype = ctypes.c_int
        d = lib.BrotliGetDictionary().contents
        _DICT = (lib, bytes(d.data[:d.data_size]), list(d.size_bits_by_length), list(d.offsets_by_length), lib.BrotliGetTransforms())
    return _DICT


def dictionary_word(copy_len, word_id):
    """Bytes of static-dictionary reference `word_id` of length `copy_len` (RFC 7932 section 8), or None if invalid."""
    lib, data, bits, offs, transforms = _dictionary()
    if not 4 <= copy_len <= 24 or bits[copy_len] == 0:
        return None
    nb = bits[copy_len]
    idx, tr = word_id & ((1 << nb) - 1), word_id >> nb
    if tr >= 121:
        return None
    w = data[offs[copy_len] + idx * copy_len: offs[copy_len] + (idx + 1) * copy_len]
    out = ctypes.create_string_buffer(64)
    n = lib.BrotliTransformDictionaryWord(out, w, copy_len, transforms, tr)
    return out.raw[:n]


# ---- bits and prefix codes --------------------------------------------------------------------------------------------------
class BitReader:
    def __init__(self, data):
        self.d = bytes(data) + bytes(16)
        self.n = len(data) * 8
        self.pos = 0

    def peek(self):  # at least 56 bits from pos
        p = self.pos
        return int.from_bytes(self.d[p >> 3:(p >> 3) + 8], "little") >> (p & 7)

    def bits(self, n):
        if n == 0:
            return 0
        v = self.peek() & ((1 << n) - 1) if n <= 56 else sum(((self.d[(self.pos + i) >> 3] >> ((self.pos + i) & 7)) & 1) << i for i in range(n))
        self.pos += n
        if self.pos > self.n:
            raise StreamError("read past the end of the stream")
        return v


class PrefixCode:
    """Canonical prefix code over `lengths` (RFC 7932 section 3.2) with a decode table over the next `maxlen` bits."""

    def __init__(self, lengths, kind="complex", simple_symbols=None, tree_select=None):
        self.lengths = list(lengths)
        self.kind = kind                      # "single" (one symbol, no bits), "simple" or "complex"
        self.simple_symbols = simple_symbols  # simple codes: the symbols in stream order
        self.tree_select = tree_select
        used = [(l, s) for s, l in enumerate(self.lengths) if l]
        if kind == "single":
            self.maxlen = 0
            self.table = [simple_symbols[0]]
            return
        kraft = sum(1 << (15 - l) for l, _ in used)
        if kraft != 1 << 15 or any(l > 15 for l, _ in used):
            raise StreamError("prefix code is not complete: Kraft sum %d / 32768" % kraft)
        self.maxlen = max(l for l, _ in used)
        table = np.zeros(1 << self.maxlen, dtype=np.int64)
        bl = [0] * 17
        for l, _ in used:
            bl[l] += 1
        nxt, code = [0] * 17, 0
        for i in range(1, 17):
            code = (code + bl[i - 1]) << 1
            nxt[i] = code
        for s, l in enumerate(self.lengths):
            if l:
                c = nxt[l]
                nxt[l] += 1
                r = int(format(c, "0%db" % l)[::-1], 2)  # the stream is LSB first, codes are MSB first
                table[r::1 << l] = s | (l << 16)
        self.table = table.tolist()

    def read(self, br):
        if self.maxlen == 0:
            return self.table[0]
        v = self.table[br.peek() & ((1 << self.maxlen) - 1)]
        br.pos += v >> 16
        return v & 0xFFFF


def read_prefix_code(br, alphabet):
    hskip = br.bits(2)
    if hskip == 1:  # simple code (RFC 7932 section 3.4)
        nsym = br.bits(2) + 1
        nb = max(1, (alphabet - 1).bit_length())
        syms = [br.bits(nb) for _ in range(nsym)]
        if any(s >= alphabet for s in syms) or len(set(syms)) != nsym:
            raise StreamError("bad simple code symbols %s" % syms)
        lengths = [0] * alphabet
        if nsym == 1:
            return PrefixCode(lengths, "single", syms)
        tree_select = None
        if nsym == 2:
            ls = [1, 1]
        elif nsym == 3:
            ls = [1, 2, 2]
        else:
            tree_select = br.bits(1)
            ls = [1, 2, 3, 3] if tree_select else [2, 2, 2, 2]
        for s, l in zip(syms, ls):
            lengths[s] = l
        return PrefixCode(lengths, "simple", syms, tree_select)
    cl = [0] * 18
    space, num = 32, 0
    fixed = PrefixCode([2, 4, 3, 2, 2, 4])
    for i in range(hskip, 18):
        v = fixed.read(br)
        cl[K_CL_ORDER[i]] = v
        if v:
            space -= 32 >> v
            num += 1
            if space <= 0:
                break
    if num == 1:
        clc = PrefixCode([0] * 18, "single", [cl.index(next(v for v in cl if v))])
    else:
        clc = PrefixCode(cl)
    lengths = [0] * alphabet
    i, prev, rep, rep_len, space = 0, 8, 0, 0, 32768
    while i < alphabet and space > 0:
        s = clc.read(br)
        if s < 16:
            lengths[i] = s
            i += 1
            rep = 0
            if s:
                prev = s
                space -= 32768 >> s
        else:
            extra = br.bits(2 if s == 16 else 3)
            new_len = prev if s == 16 else 0
            if rep_len != new_len:
                rep, rep_len = 0, new_len
            old = rep
            if rep > 0:
                rep = (rep - 2) << (2 if s == 16 else 3)
            rep += extra + 3
            delta = rep - old
            if i + delta > alphabet:
                raise StreamError("code length repeat past the alphabet")
            for _ in range(delta):
                lengths[i] = rep_len
                i += 1
            if rep_len:
                space -= delta * (32768 >> rep_len)
    code = PrefixCode(lengths)
    code.cl_lengths = cl
    return code


def read_block_len(br, code):
    c = code.read(br)
    return BL_OFFSET[c] + br.bits(BL_NBITS[c])


def read_var_len_uint8(br):
    if br.bits(1) == 0:
        return 0
    nb = br.bits(3)
    return (1 << nb) + br.bits(nb) if nb else 1


def read_context_map(br, size):
    """(number of trees, map, its prefix code) of a context map (RFC 7932 section 7.3)."""
    n = read_var_len_uint8(br) + 1
    if n == 1:
        return 1, [0] * size, None
    rlemax = br.bits(4) + 1 if br.bits(1) else 0
    code = read_prefix_code(br, n + rlemax)
    cm = []
    while len(cm) < size:
        s = code.read(br)
        if s == 0:
            cm.append(0)
        elif s <= rlemax:
            cm.extend([0] * ((1 << s) + br.bits(s)))
        else:
            cm.append(s - rlemax)
    if len(cm) > size:
        raise StreamError("context map run past its end")
    if br.bits(1):  # inverse move-to-front
        mtf = list(range(256))
        for i, v in enumerate(cm):
            x = mtf[v]
            cm[i] = x
            del mtf[v]
            mtf.insert(0, x)
    return n, cm, code


# ---- the stream ---------------------------------------------------------------------------------------------------------------
class Metablock:
    """One metablock.  Header fields: start (output offset), mlen, is_last, raw, ntypes[3], type_code[3] / len_code[3]
    (PrefixCode or None), first_len[3], cmodes, lit_cmap, dist_cmap, nlit_trees, ndist_trees, npostfix, ndirect, lit_codes,
    cmd_codes, dist_codes.  Body: see `audit`."""

    def __init__(self, start):
        self.start = start
        self.raw = False


def _ctx_tables(data):
    return [context_ids(data, m).tolist() for m in range(4)]


def audit(stream, data):
    """Decode `stream`, which must decode to `data`; returns (lgwin, [Metablock]).

    Per compressed metablock:
      cmds: list of tuples (pos, ins, copy, cmd_sym, cmd_type, dist_sym, dist_extra, dist_type, dist_ctx, distance, is_dict,
            ring, pushes) -- dist_sym is -1 for the implicit distance of a command symbol < 128 and for a command that ends
            the metablock inside its insert (then distance is None); ring is the 4-entry ring before the command, most recent
            first, and `pushes` how many of its entries were pushed inside this metablock (at most 4);
      lit_bytes / lit_types / lit_ctx / lit_trees: one entry per literal, in stream order;
      switches[cat]: [(rank, type_code, type, block_len)] -- the first entry is the initial block (type_code None)."""
    data = bytes(data)
    br = BitReader(stream)
    if br.bits(1) == 0:
        lgwin = 16
    else:
        n = br.bits(3)
        if n:
            lgwin = 17 + n
        else:
            n = br.bits(3)
            if n == 1:
                raise StreamError("large-window streams are not audited")
            lgwin = 17 if n == 0 else 8 + n
    max_backward = (1 << lgwin) - 16
    ctx_tab = None
    out = 0                          # bytes produced so far
    ring = [16, 15, 11, 4]           # most recent first
    mbs = []
    while True:
        mb = Metablock(out)
        islast = br.bits(1)
        if islast and br.bits(1):    # ISLASTEMPTY
            break
        mn = br.bits(2)
        if mn == 3:                  # metadata
            if br.bits(1):
                raise StreamError("reserved bit set")
            sk = br.bits(2)
            ln = br.bits(8 * sk) + 1 if sk else 0
            br.pos = (br.pos + 7) & ~7
            br.pos += 8 * ln
            if islast:
                break
            continue
        mlen = br.bits(4 * (mn + 4)) + 1
        mb.mlen, mb.is_last = mlen, bool(islast)
        if out + mlen > len(data):
            raise StreamError("metablock at %d runs past the input (%d + %d > %d)" % (out, out, mlen, len(data)))
        if not islast and br.bits(1):  # uncompressed
            br.pos = (br.pos + 7) & ~7
            got = br.d[br.pos >> 3:(br.pos >> 3) + mlen]
            if got != data[out:out + mlen]:
                raise StreamError("uncompressed metablock at %d differs from the input" % out)
            br.pos += 8 * mlen
            mb.raw = True
            out += mlen
            mbs.append(mb)
            continue
        if ctx_tab is None:
            ctx_tab = _ctx_tables(data)
        mb.ntypes, mb.type_code, mb.len_code, mb.first_len = [], [], [], []
        for cat in range(3):
            nt = read_var_len_uint8(br) + 1
            mb.ntypes.append(nt)
            if nt > 1:
                mb.type_code.append(read_prefix_code(br, nt + 2))
                mb.len_code.append(read_prefix_code(br, 26))
                mb.first_len.append(read_block_len(br, mb.len_code[cat]))
            else:
                mb.type_code.append(None)
                mb.len_code.append(None)
                mb.first_len.append(1 << 28)
        mb.npostfix = br.bits(2)
        mb.ndirect = br.bits(4) << mb.npostfix
        mb.cmodes = [br.bits(2) for _ in range(mb.ntypes[0])]
        mb.nlit_trees, mb.lit_cmap, mb.lit_cmap_code = read_context_map(br, 64 * mb.ntypes[0])
        mb.ndist_trees, mb.dist_cmap, mb.dist_cmap_code = read_context_map(br, 4 * mb.ntypes[2])
        mb.lit_codes = [read_prefix_code(br, 256) for _ in range(mb.nlit_trees)]
        mb.cmd_codes = [read_prefix_code(br, 704) for _ in range(mb.ntypes[1])]
        mb.dist_alphabet = 16 + mb.ndirect + (48 << mb.npostfix)
        mb.dist_codes = [read_prefix_code(br, mb.dist_alphabet) for _ in range(mb.ndist_trees)]
        mb.header_bits = br.pos
        _body(br, mb, data, ctx_tab, ring, out, max_backward)
        out += mlen
        mbs.append(mb)
        if islast:
            break
    if out != len(data):
        raise StreamError("stream decodes to %d bytes, input has %d" % (out, len(data)))
    return lgwin, mbs


def _body(br, mb, data, ctx_tab, ring, out0, max_backward):
    ntypes = mb.ntypes
    btype = [0, 0, 0]
    prev_types = [[0, 1], [0, 1], [0, 1]]   # (last, second last) as the decoder keeps them
    blen = list(mb.first_len)
    switches = [[(0, None, 0, mb.first_len[c] if ntypes[c] > 1 else None)] for c in range(3)]
    rank = [0, 0, 0]

    def switch(cat):
        c = mb.type_code[cat].read(br)
        pt = prev_types[cat]
        t = pt[1] if c == 0 else ((pt[0] + 1) % ntypes[cat] if c == 1 else c - 2)
        if t >= ntypes[cat]:
            raise StreamError("block type %d >= NBLTYPES %d" % (t, ntypes[cat]))
        prev_types[cat] = [t, pt[0]]
        btype[cat] = t
        blen[cat] = read_block_len(br, mb.len_code[cat])
        switches[cat].append((rank[cat], c, t, blen[cat]))

    lit_bytes, lit_types, lit_ctx, lit_trees = bytearray(), bytearray(), [], []
    cmds = []
    lit_codes, cmd_codes, dist_codes = mb.lit_codes, mb.cmd_codes, mb.dist_codes
    lit_cmap, dist_cmap = mb.lit_cmap, mb.dist_cmap
    pushes = 0
    pos, end = out0, out0 + mb.mlen
    while pos < end:
        if blen[1] == 0:
            switch(1)
        blen[1] -= 1
        rank[1] += 1
        cmd_type = btype[1]
        cs = cmd_codes[cmd_type].read(br)
        cell = cs >> 6
        icode = CELL_INS[cell] + ((cs >> 3) & 7)
        ccode = CELL_COPY[cell] + (cs & 7)
        ins = INS_BASE[icode] + br.bits(INS_EXTRA[icode])
        cpy = COPY_BASE[ccode] + br.bits(COPY_EXTRA[ccode])
        cmd_pos = pos
        if pos + ins > end:
            raise StreamError("insert of %d at %d runs past the metablock end %d" % (ins, pos, end))
        # literals
        j = 0
        while j < ins:
            if blen[0] == 0:
                switch(0)
            t = btype[0]
            k = min(ins - j, blen[0])           # literals before the next block switch
            ctab = ctx_tab[mb.cmodes[t]]
            base = 64 * t
            for p in range(pos, pos + k):
                cx = ctab[p]
                tree = lit_cmap[base + cx]
                code = lit_codes[tree]
                if code.maxlen:
                    ps = br.pos
                    v = code.table[(int.from_bytes(br.d[ps >> 3:(ps >> 3) + 4], "little") >> (ps & 7)) & ((1 << code.maxlen) - 1)]
                    br.pos = ps + (v >> 16)
                    b = v & 0xFFFF
                else:
                    b = code.table[0]
                if b != data[p]:
                    raise StreamError("literal at %d decodes to %d, input has %d" % (p, b, data[p]))
                lit_ctx.append(cx)
                lit_trees.append(tree)
            lit_bytes += data[pos:pos + k]
            lit_types += bytes([t]) * k
            blen[0] -= k
            rank[0] += k
            pos += k
            j += k
        if br.pos > br.n:
            raise StreamError("read past the end of the stream")
        if pos >= end:
            cmds.append((cmd_pos, ins, cpy, cs, cmd_type, -1, 0, None, None, None, False, tuple(ring), pushes))
            break
        ring_before, pushes_before = tuple(ring), pushes
        if cs < 128:
            dsym, dextra, dtype, dctx = -1, 0, None, None
            distance = ring[0]
        else:
            if blen[2] == 0:
                switch(2)
            blen[2] -= 1
            rank[2] += 1
            dtype = btype[2]
            dctx = 3 if cpy > 4 else cpy - 2
            dsym = dist_codes[dist_cmap[4 * dtype + dctx]].read(br)
            dextra = 0
            if dsym < 16:
                distance = ring[SHORT_IDX[dsym]] + SHORT_OFF[dsym]
                if distance <= 0:
                    raise StreamError("short distance code %d gives distance %d" % (dsym, distance))
            elif dsym < 16 + mb.ndirect:
                distance = dsym - 15
            else:
                x = dsym - mb.ndirect - 16
                nbits = 1 + (x >> (mb.npostfix + 1))
                hcode = x >> mb.npostfix
                lcode = x & ((1 << mb.npostfix) - 1)
                offset = ((2 + (hcode & 1)) << nbits) - 4
                dextra = br.bits(nbits)
                distance = ((offset + dextra) << mb.npostfix) + lcode + mb.ndirect + 1
        max_distance = min(pos, max_backward)
        is_dict = distance > max_distance
        if is_dict:
            word = dictionary_word(cpy, distance - max_distance - 1)
            if word is None:
                raise StreamError("invalid dictionary reference at %d: length %d, distance %d" % (pos, cpy, distance))
            if data[pos:pos + len(word)] != word:
                raise StreamError("dictionary word at %d differs from the input" % pos)
            covered = len(word)
        else:
            covered = cpy
            if pos + cpy > end:
                raise StreamError("copy at %d runs past the metablock end" % pos)
            src = pos - distance
            if distance >= cpy:
                ok = data[src:src + cpy] == data[pos:pos + cpy]
            else:
                ok = all(data[src + i] == data[pos + i] for i in range(cpy))
            if not ok:
                raise StreamError("copy at %d (distance %d, length %d) differs from the input" % (pos, distance, cpy))
            if dsym != 0 and cs >= 128:
                ring[1:4] = ring[0:3]
                ring[0] = distance
                pushes = min(4, pushes + 1)
        cmds.append((cmd_pos, ins, cpy, cs, cmd_type, dsym, dextra, dtype, dctx, distance, is_dict, ring_before, pushes_before))
        pos += covered
        if pos > end:
            raise StreamError("copy at %d runs past the metablock end" % (pos - covered))
    mb.cmds = cmds
    mb.lit_bytes, mb.lit_types = bytes(lit_bytes), bytes(lit_types)
    mb.lit_ctx, mb.lit_trees = np.array(lit_ctx, dtype=np.int32), np.array(lit_trees, dtype=np.int32)
    mb.switches = switches
    mb.counts = list(rank)

"""Deterministic synthetic inputs for the BASELINE.json configs (SURVEY.md section 8d).

Nothing here reads files outside the repository.  All generators are seeded and vectorised
with numpy so that 100 MB takes seconds.

  enwik_like(n, seed=8)   -- Wikipedia-XML-shaped UTF-8 text: Zipfian pseudo-word vocabulary driven by an
                             order-1 Markov chain (each word has a few preferred successors), wrapped in
                             <page><title>..</title><text>..</text></page> records with [[link]] / {{tmpl}} markup.
                             Tuned so that brotli q5/lgwin22 lands at a ratio of about 0.3 (real enwik8 ~0.3).
  json_logs(n, seed=4)    -- newline-delimited JSON log records with Zipfian keys/values and increasing timestamps.
  tiled(block, n)         -- a small block repeated to n bytes (configs 3 and 5 tile a 10 KB / 176 KB file).
  pcg_random(n, seed=3)   -- incompressible bytes.
"""
import numpy as np


def _make_vocab(rng, nwords):
    """Pseudo-words: syllable-based so that letter statistics look like a natural language."""
    cons = np.array(list("bcdfghjklmnprstvwz") + ["th", "st", "ch", "sh", "tr", "pr", "nd", "ng", "ll", "ss"], dtype=object)
    cons_p = rng.dirichlet(np.ones(len(cons)) * 2.0)
    vow = np.array(list("aeiou") + ["ea", "ou", "ie", "ai", "oo"], dtype=object)
    vow_p = np.array([0.2, 0.27, 0.17, 0.17, 0.07, 0.03, 0.03, 0.02, 0.02, 0.02])
    vow_p = vow_p / vow_p.sum()
    words = []
    seen = set()
    # short words first (they will be the most frequent ranks)
    while len(words) < nwords:
        rank = len(words)
        nsyl = 1 + int(rng.random() < min(0.9, 0.25 + rank / 400.0)) + int(rng.random() < min(0.8, rank / 3000.0)) \
            + int(rng.random() < min(0.5, rank / 20000.0))
        w = ""
        for _ in range(nsyl):
            if rng.random() < 0.8:
                w += cons[rng.choice(len(cons), p=cons_p)]
            w += vow[rng.choice(len(vow), p=vow_p)]
            if rng.random() < 0.35:
                w += cons[rng.choice(len(cons), p=cons_p)]
        if w in seen:
            continue
        seen.add(w)
        words.append(w)
    return words


def _gather_strings(blob, offs, lens, ids):
    """Concatenate blob[offs[i]:offs[i]+lens[i]] for i in ids (vectorised)."""
    l = lens[ids]
    total = int(l.sum())
    starts = np.cumsum(l) - l
    idx = np.arange(total, dtype=np.int64) - np.repeat(starts, l) + np.repeat(offs[ids], l)
    return blob[idx]


def enwik_like(nbytes, seed=8, nwords=60000, nsucc=6, p_follow=0.28):
    rng = np.random.default_rng(seed)
    words = _make_vocab(rng, nwords)
    # token table: plain words (with trailing space), capitalised variants, punctuation and markup tokens
    toks = [w + " " for w in words]
    nplain = len(toks)
    specials = [". ", ", ", ".\n", "; ", ": ", "? ", "\n\n", "''", "'''", " (", ") ", "== ", " ==\n", "* ", "&quot;", "&amp;",
                "1", "2", "3", "19", "20", "0", "5", "8", "<ref>", "</ref> ", "|", "}} ", "]] ", "[[", "{{", "http://www.",
                ".com/ ", "[[Category:", "&lt;", "&gt;", "-", "= "]
    toks += specials
    blob = np.frombuffer("".join(toks).encode("utf-8"), dtype=np.uint8)
    lens = np.array([len(t.encode("utf-8")) for t in toks], dtype=np.int64)
    offs = np.cumsum(lens) - lens
    ntok = len(toks)
    # unigram: Zipf over words, specials get a fixed share
    ranks = np.arange(1, nplain + 1, dtype=np.float64)
    p_words = 1.0 / ranks ** 1.02
    p_words *= 0.80 / p_words.sum()
    p_spec = rng.dirichlet(np.ones(len(specials)) * 0.7) * 0.20
    p_uni = np.concatenate([p_words, p_spec])
    cdf_uni = np.cumsum(p_uni)
    cdf_uni /= cdf_uni[-1]
    # preferred successors (order-1 structure): each token gets nsucc successors drawn from the unigram law
    succ = np.searchsorted(cdf_uni, rng.random((ntok, nsucc))).astype(np.int32)
    succ = np.minimum(succ, ntok - 1)
    avg_len = float((lens * p_uni).sum() / p_uni.sum())
    ntokens = int(nbytes / avg_len * 1.08) + 4096
    nchains = 8192
    steps = (ntokens + nchains - 1) // nchains
    state = np.minimum(np.searchsorted(cdf_uni, rng.random(nchains)), ntok - 1).astype(np.int32)
    out = np.empty((steps, nchains), dtype=np.int32)
    for s in range(steps):
        follow = rng.random(nchains) < p_follow
        pick = rng.integers(0, nsucc, nchains)
        # geometric preference among the successors
        pick = np.minimum(pick, rng.integers(0, nsucc, nchains))
        nxt_f = succ[state, pick]
        nxt_u = np.minimum(np.searchsorted(cdf_uni, rng.random(nchains)), ntok - 1).astype(np.int32)
        state = np.where(follow, nxt_f, nxt_u).astype(np.int32)
        out[s] = state
    ids = out.T.reshape(-1)  # each chain is one contiguous "article"
    body = _gather_strings(blob, offs, lens, ids)
    # wrap articles into <page> records: insert headers at chain boundaries
    chain_bytes = lens[out.T].sum(axis=1)
    bounds = np.cumsum(chain_bytes) - chain_bytes
    pieces = []
    title_ids = np.minimum(np.searchsorted(cdf_uni[:nplain] / cdf_uni[nplain - 1], rng.random((nchains, 2))), nplain - 1)
    total = 0
    for c in range(nchains):
        if total >= nbytes:
            break
        t = (words[title_ids[c, 0]] + " " + words[title_ids[c, 1]]).title()
        hdr = ("  <page>\n    <title>%s</title>\n    <id>%d</id>\n    <revision>\n      <id>%d</id>\n"
               "      <timestamp>2006-03-%02dT%02d:%02d:%02dZ</timestamp>\n      <contributor>\n        <username>%s</username>\n"
               "        <id>%d</id>\n      </contributor>\n      <text xml:space=\"preserve\">" %
               (t, 1000 + c * 7, 15900000 + c * 131, 1 + c % 28, c % 24, (c * 7) % 60, (c * 13) % 60,
                words[title_ids[c, 1]].title(), 1000 + (c * 37) % 90000)).encode()
        ftr = b"</text>\n    </revision>\n  </page>\n"
        seg = body[bounds[c]:bounds[c] + chain_bytes[c]]
        pieces.append(np.frombuffer(hdr, dtype=np.uint8))
        pieces.append(seg)
        pieces.append(np.frombuffer(ftr, dtype=np.uint8))
        total += len(hdr) + len(seg) + len(ftr)
    data = np.concatenate(pieces)
    while len(data) < nbytes:  # extremely unlikely; repeat deterministically
        data = np.concatenate([data, data[: nbytes - len(data)]])
    return data[:nbytes].tobytes()


def json_logs(nbytes, seed=4):
    rng = np.random.default_rng(seed)
    words = _make_vocab(rng, 5000)
    levels = ["INFO", "INFO", "INFO", "DEBUG", "WARN", "ERROR"]
    svcs = ["auth", "gateway", "billing", "search", "indexer", "mailer", "scheduler", "storage"]
    keys = ["user", "req", "path", "status", "dur_ms", "host", "region", "shard", "retry", "bytes"]
    n_rec = nbytes // 250 + 1024
    zipf = np.minimum(rng.zipf(1.3, (n_rec, 12)), len(words)) - 1
    lv = rng.integers(0, len(levels), n_rec)
    sv = np.minimum(rng.zipf(1.5, n_rec), len(svcs)) - 1
    nk = rng.integers(2, 6, n_rec)
    nums = rng.integers(0, 100000, (n_rec, 6))
    dts = rng.integers(1, 900, n_rec)
    ts = 1700000000000 + np.cumsum(dts)
    out = []
    total = 0
    for i in range(n_rec):
        msg = " ".join(words[j] for j in zipf[i, : 3 + (i % 6)])
        kv = ",".join('"%s":%s' % (keys[(i + k * 3) % len(keys)],
                                   ('"%s"' % words[zipf[i, 8 + (k % 4)]]) if k % 2 else str(nums[i, k]))
                      for k in range(nk[i]))
        rec = '{"ts":%d,"level":"%s","svc":"%s","msg":"%s","kv":{%s}}\n' % (ts[i], levels[lv[i]], svcs[sv[i]], msg, kv)
        out.append(rec)
        total += len(rec)
        if total >= nbytes:
            break
    data = "".join(out).encode()
    while len(data) < nbytes:
        data += data[: nbytes - len(data)]
    return data[:nbytes]


def tiled(block: bytes, nbytes: int) -> bytes:
    reps = nbytes // len(block) + 1
    return (block * reps)[:nbytes]


def pcg_random(nbytes, seed=3):
    return np.random.Generator(np.random.PCG64(seed)).integers(0, 256, nbytes, dtype=np.uint8).tobytes()


if __name__ == "__main__":
    import sys, time
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
    t = time.time()
    d = enwik_like(n)
    print("generated", len(d), "bytes in %.1fs" % (time.time() - t))
    sys.stdout.write(d[:1500].decode("utf-8", "replace"))

"""CPU: quality 9.5 (BROTLI_PARAM_Q9_5) in the parameter rule and the CPU model of the pipeline.

  * default_enc_params without Q9_5 gives the parameters it gave before Q9_5 existed (restated below), at every quality, window
    and size-hint class; with Q9_5 it gives the hasher of tests/q95_cases.py:hasher_q95, the hash-chain parse family and the
    quality 10 / 11 metablock builder;
  * the model's 9.5 streams of tests/q95_cases.py decode through libbrotlidec and equal their sha256 goldens (the device must
    produce the same bytes: tests/test_gpu_q95.py)."""
import pytest

import q95_cases as C
from oracle.harness import sys_decompress

MIB = 1 << 20
HINTS = [0, 1000, 256 << 10, MIB, MIB + 1, 4 * MIB, 4 * MIB + 1, 0xFFFFFFFF]


def _without_q95(q, w, hint):
    """The parameter rule before Q9_5: (hash_type, key_bits, hash_len, depth, n_last, lcap, unit, mb_units, hq_levels)."""
    q = min(max(q, 5), 11)
    w = min(max(w, 10), 24)
    if q >= 10:
        unit = 2048 if hint and hint <= 256 << 10 else 4096 if hint and hint <= MIB else (16384 if q >= 11 else 8192)
        return (5, 15, 4, 256, 16, 384, unit, (4 << 20) // unit, 3)
    if q == 9:
        h = (9, 15, 4, 256, 16)
    elif w <= 16:
        h = (6, 15, 5, 256, 16)
    else:
        nl = 4 if q < 7 else 10 if q < 9 else 16
        if hint > 4 * MIB and w >= 19:
            h = (6, 15, 5, 1 << (q - 1), nl)
        else:
            h = (5, 14 if q < 7 and hint <= MIB else 15, 4, 1 << (q - 1), nl)
    return h + (64, 4096, 1024, 0)


def _fields(p):
    return (p.hash_type, p.key_bits, p.hash_len, p.depth, p.n_last, p.lcap, p.unit, p.mb_units, p.hq_levels)


def test_params_without_q95_unchanged(model):
    from tools.model_harness import EncParams
    names = [f[0] for f in EncParams._fields_]
    for q in range(0, 13):
        for w in (10, 16, 17, 18, 19, 22, 24, 25):
            for hint in HINTS:
                p = model.params(q, w, 1 << 20, hint)
                assert _fields(p) == _without_q95(q, w, hint or (1 << 20)), (q, w, hint)
                assert (p.zopfli, p.hq_meta) == ((1, 1) if q >= 10 else (0, 0)), (q, w, hint)
                assert p.hq_split == 1 and p.ctx_model == 1 and p.use_dict == 1
                # with Q9_5 quality 5..9 differ at most in the H6 threshold
                r = model.params(q, w, 1 << 20, hint, q9_5=True)
                if q < 10:
                    same = [n for n in names if n not in ("hash_type", "hash_len", "key_bits")]
                    assert all(getattr(r, n) == getattr(p, n) for n in same), (q, w, hint)


def test_params_with_q95(model):
    for q in range(5, 12):
        for w in (10, 16, 17, 18, 19, 22, 24):
            for hint in HINTS:
                p = model.params(q, w, 1 << 20, hint, q9_5=True)
                ht, kb, depth = C.hasher_q95(q, w, hint or (1 << 20))
                assert (p.hash_type, p.key_bits, p.depth) == (ht, kb, depth), (q, w, hint)
                assert p.hash_len == (5 if ht == 6 else 4)
                assert p.n_last == (16 if q >= 9 or w <= 16 else 4 if q < 7 else 10)
                assert (p.zopfli, p.hq_meta) == (0, 1 if q >= 10 else 0)
                assert (p.lcap, p.unit, p.mb_units, p.hq_levels) == (64, 4096, 1024, 0)
    # the H6 threshold at quality 5..8: above 1 MiB with Q9_5, above 4 MiB without
    assert model.params(7, 22, 1, 2 * MIB, q9_5=True).hash_type == 6
    assert model.params(7, 22, 1, 2 * MIB).hash_type == 5


@pytest.fixture(scope="module")
def case_inputs():
    return {}


@pytest.mark.parametrize("name", list(C.CASES))
def test_model_q95_golden(model, case_inputs, name):
    inp, q, w, hint, kw = C.CASES[name]
    if inp not in case_inputs:
        case_inputs.clear()
        case_inputs[inp] = C.inputs(inp)
    d = case_inputs[inp]
    c, _ = model.compress(d, q, w, size_hint=hint, q9_5=True, **kw)
    assert sys_decompress(c, len(d)) == d, name
    assert C.sha(c) == C.GOLDEN[name], "%s: model stream changed (%d B)" % (name, len(c))


def test_model_q95_sits_between_q9_and_q10(model):
    """On alice29 (lgwin 22) 9.5 is smaller than q9 and larger than q10, 9.5x smaller than 9.5 and larger than q11."""
    d = C.inputs("alice")
    size = {k: len(model.compress(d, q, 22, q9_5=q95)[0]) for k, q, q95 in
            (("q9", 9, False), ("9.5", 10, True), ("9.5x", 11, True), ("q10", 10, False), ("q11", 11, False))}
    assert size["q9"] > size["9.5"] > size["q10"], size
    assert size["9.5"] > size["9.5x"] > size["q11"], size

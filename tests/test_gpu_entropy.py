"""Entropy stage (after the parse) against tests/entropy_ref.py, symbol by symbol, on the device's streams.

The stream is read back by tests/stream_audit.py with the input known.  For every metablock:
  * the literal context map must be the one the float64 restatement of DecideOverLiteralContextModeling chooses;
  * the greedy splitter's block switches must be decisions float64 allows at every FinishBlock (guided replay; a margin
    inside its bound on the Q16 error may go either way and is counted as ambiguous);
  * every prefix code must equal the encoder's smoothing + length-limited Huffman rule over the recounted histogram
    exactly, be complete, and cost no more than the optimum (heapq Huffman, or package-merge where the 15-bit limit
    applies: the Kraft repair may lose at most entropy_ref.REPAIR_GAP_MAX);
  * every distance must be sent with the shortest code ComputeDistanceCode gives over the ring entries pushed inside the
    metablock, and the implicit-distance command form used exactly where CombineLengthCodes allows it.
Quality 10 / 11 run the per-code and distance checks only (BrotliSplitBlock, clustering and context-map construction are
not restated here).  Each device stream must also equal the CPU model's."""
import pytest

import entropy_ref as er
from conftest import golden_bytes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cases():
    from tools import datagen
    return {c[0]: c for c in er.planted_cases(golden_bytes, datagen, big=True)}


@pytest.fixture(scope="module")
def hq_cases():
    from tools import datagen
    return {c[0]: c for c in er.hq_cases(golden_bytes, datagen)}


def _device_stream(encoder, d, q, w, hint):
    return encoder.compress_range(d, 0, len(d), q, w, True, True, False, size_hint=hint)


NAMES = ["fibonacci-26", "fibonacci-30", "tolerance", "1-symbols", "2-symbols", "3-symbols", "4-symbols", "15-symbols",
         "16-symbols", "17-symbols", "segments", "segments-q9", "type-cap", "type-cap-complex13", "no-distances",
         "incompressible", "hint-below-1MiB", "hint-1MiB", "hint-1MiB-q7", "json-q9", "two-4MiB-metablocks"]


@pytest.mark.parametrize("name", NAMES)
def test_device_entropy_stage_planted(encoder, model, cases, name):
    _, d, q, w, hint = cases[name]
    c = _device_stream(encoder, d, q, w, hint)
    report = er.audit_stream(c, d, q, hint)
    assert c == model.compress_range(d, 0, len(d), q, w, True, True, False, size_hint=hint)[0], "%s: device != model" % name
    if name.startswith("fibonacci-30") or name == "two-4MiB-metablocks":
        assert report["repaired"] > 0, "%s: no code reached the Kraft repair" % name
    if name == "type-cap":
        assert report["new"] >= 255, report  # the 256-type cap of the command / literal splitters is reached
    if name == "type-cap-complex13":
        assert report["maps"] == {"complex-13": 1} and report["new"] >= 19, report
    print(name, {k: v for k, v in report.items() if k != "gaps"}, "repair gaps", report["gaps"])


@pytest.mark.parametrize("name", ["alice29.txt", "asyoulik.txt", "random_then_unicode", "compressed_file", "quickfox_repeated"])
def test_device_entropy_stage_golden(encoder, model, name):
    d = golden_bytes(name)
    for q in (5, 7, 9):
        for w in (16, 22):
            c = _device_stream(encoder, d, q, w, 0)
            er.audit_stream(c, d, q)
            assert c == model.compress(d, q, w)[0], "%s q%d lgwin %d: device != model" % (name, q, w)


@pytest.mark.parametrize("name", ["alice29-q10", "alice29-q11", "asyoulik-q10-w16", "json-q11", "fibonacci-q10"])
def test_device_entropy_codes_hq(encoder, model, hq_cases, name):
    _, d, q, w, hint = hq_cases[name]
    c = _device_stream(encoder, d, q, w, hint)
    report = er.audit_stream(c, d, q, hint)
    assert c == model.compress(d, q, w)[0], "%s: device != model" % name
    if name == "fibonacci-q10":
        assert report["repaired"] > 0

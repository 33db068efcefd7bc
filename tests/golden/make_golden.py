"""Regenerates tests/golden/: copies the reference's small test inputs (public test vectors, not source code) and
records, for each (file, quality, lgwin): the size produced by the C restatement in oracle/ (with sha256 of its
stream), the size produced by Google's libbrotlienc 1.1.0 (the code the reference was ported from), and the size +
sha256 of the CPU model of the GPU pipeline.

  python tests/golden/make_golden.py [TESTDATA_DIR]

TESTDATA_DIR is the reference's testdata/ directory to copy the inputs from; without it the inputs already stored here are
used and only golden_sizes.json is rewritten."""
import hashlib, json, os, shutil, sys
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.harness import Oracle, sys_compress, sys_decompress
from tools.model_harness import Model

FILES = ["alice29.txt", "asyoulik.txt", "random_then_unicode", "quickfox_repeated", "random_org_10k.bin", "backward65536",
         "64x", "ukkonooa", "monkey", "x", "xyzzy", "10x10y", "aaabaaaa", "empty", "quickfox", "compressed_file"]
CONFIGS = [(5, 20), (5, 22), (6, 22), (7, 22), (8, 22), (9, 22), (9, 16), (5, 24), (5, 18), (10, 22), (11, 22), (11, 24), (10, 16)]
# quality >= 10: oracle/brotli_ref.c restates the q4..q9 path only; the size reference there is libbrotlienc 1.1.0 (the C code
# the reference was ported from: alice29 q10 = 47 477 B, q11 = 46 487 B against the reference's own KATs 47 488 / 46 493,
# src/bin/integration_tests.rs:408-449) -- "oracle_size" then holds that size and "size_reference" says so.

def main(src=None):
    here = os.path.dirname(os.path.abspath(__file__))
    o, m = Oracle(), Model()
    table = {}
    for f in FILES:
        if src:
            shutil.copyfile(os.path.join(src, f), os.path.join(here, f))
        d = open(os.path.join(here, f), "rb").read()
        for q, w in CONFIGS:
            sc = sys_compress(d, q, w)
            if q >= 10:
                mc, _ = m.compress(d, q, w)
                assert sys_decompress(mc, len(d)) == d
                table["%s|q%d|w%d" % (f, q, w)] = {
                    "input_size": len(d), "oracle_size": len(sc), "size_reference": "libbrotlienc", "libbrotlienc_size": len(sc),
                    "model_size": len(mc), "model_sha256": hashlib.sha256(mc).hexdigest()}
                continue
            oc, st = o.compress(d, q, w)
            assert sys_decompress(oc, len(d)) == d
            mc, _ = m.compress(d, q, w)
            assert sys_decompress(mc, len(d)) == d
            table["%s|q%d|w%d" % (f, q, w)] = {
                "input_size": len(d), "oracle_size": len(oc), "oracle_sha256": hashlib.sha256(oc).hexdigest(),
                "oracle_equals_libbrotlienc": oc == sc, "libbrotlienc_size": len(sc), "hasher": st.hasher_type,
                "model_size": len(mc), "model_sha256": hashlib.sha256(mc).hexdigest()}
    json.dump(table, open(os.path.join(here, "golden_sizes.json"), "w"), indent=1, sort_keys=True)
    print("wrote", len(table), "entries")

if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)

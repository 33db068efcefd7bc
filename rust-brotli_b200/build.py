"""In-tree build of libbrotli_b200.so for sm_90a (H100; nvcc cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libbrotli_b200.so")
SOURCES = ["bro_encoder.cu", "bro_capi.cu", "bro_broccoli.cu", "bro_concat.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 (Hopper); the TMA bulk copies and mbarriers need sm_90
DEPS = ["bro_common.cuh", "bro_huffman.cuh", "bro_meta.cuh", "bro_parse.cuh", "bro_split.cuh", "bro_finalize.cuh",
        "bro_kernels.cuh", "bro_kernels_hq.cuh", "bro_hq.cuh", "bro_bsplit.cuh", "bro_encoder.h", "bro_dict.cuh", "bro_dict_data.inc",
        "bro_concat.cuh"]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    # this file too: a library built with other flags (another architecture) is stale
    files = [os.path.join(CSRC, f) for f in SOURCES + DEPS] + [os.path.join(ROOT, "include", h) for h in ("brotli_b200.h", "broccoli.h")]
    files.append(os.path.abspath(__file__))
    return any(os.path.exists(f) and os.path.getmtime(f) > t for f in files)


def build(force=False, verbose=False):
    inc = os.path.join(CSRC, "bro_dict_data.inc")
    if not os.path.exists(inc):  # generated: RFC 7932 dictionary (from the system libbrotlicommon) + our hash table
        subprocess.check_call([sys.executable, os.path.join(HERE, "gen_dict.py")])
    if not force and not needs_build():
        return OUT
    objs = []
    procs = []
    for f in SOURCES:
        obj = os.path.join(CSRC, f.replace(".cu", ".o"))
        cmd = ["nvcc"] + ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
               "-I", CSRC, "-I", os.path.join(ROOT, "include"), "-c", os.path.join(CSRC, f), "-o", obj]
        if verbose:
            cmd[1:1] = ["-Xptxas", "-v"]
        procs.append(subprocess.Popen(cmd))
        objs.append(obj)
    for p in procs:
        if p.wait() != 0:
            raise RuntimeError("nvcc failed")
    subprocess.check_call(["nvcc"] + ARCH + ["-shared", "-o", OUT] + objs + ["-lcudart"])
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))

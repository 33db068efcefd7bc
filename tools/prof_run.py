"""Small driver for ncu: N compressions of the 100 MB bench workload, HBM resident."""
import ctypes, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import rust_brotli_b200 as rb
from tools import datagen

def main():
    nbytes = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000_000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    q = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    kind = sys.argv[4] if len(sys.argv) > 4 else "text"
    if kind == "text": d = datagen.enwik_like(nbytes)
    elif kind == "random": d = datagen.pcg_random(nbytes)
    elif kind == "json": d = datagen.json_logs(nbytes)
    elif kind == "zeros": d = bytes(nbytes)
    else: d = datagen.tiled(open(os.path.join(ROOT, "tests", "golden", kind), "rb").read(), nbytes)
    enc = rb.DeviceEncoder(0)
    enc.set_option(rb._native.OPT_TIMING, 1)
    enc.set_option(rb._native.OPT_LANES, int(os.environ.get("B200_LANES", "4")))
    enc.set_option(rb._native.OPT_DICT, int(os.environ.get("B200_DICT", "1")))
    t_in = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
    t_out = torch.empty(len(d) + (1 << 20), dtype=torch.uint8, device="cuda")
    for i in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        n = enc.compress_device(t_in.data_ptr(), len(d), t_out.data_ptr(), t_out.numel(), q, 22)
        dt = time.perf_counter() - t
        tm, nl = enc.timings()
        print("rep", i, "bytes", n, "wall %.2f ms" % (dt * 1e3), {k: round(v, 3) for k, v in tm.items()}, "launches", nl, flush=True)

if __name__ == "__main__":
    main()

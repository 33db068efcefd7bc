"""GPU: the stream-ordered device path against the blocking one, on 100 MB of enwik-shaped text at q5, lgwin 22, HBM-resident.

Reports the host time of one async call (the enqueue alone: nothing waits), and the wall time of 10 back-to-back steps of the
blocking call (b200_encoder_compress_range, device_io 1), of the async call (enqueued 10 times, one synchronise at the end) and of
a CUDA graph replay of one captured async call.  The three are alternated in one run; every round prints one JSON line, and the
last line has the medians with the card's name and power limit.  Not part of bench.py."""
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        return q
    except Exception as e:  # the measurement stands without it
        return "unknown (%s)" % e


def main():
    import torch
    import rust_brotli_b200 as rb
    from tools import datagen
    n, q, w, steps, rounds = 100_000_000, 5, 22, 10, int(os.environ.get("ROUNDS", "3"))
    d = datagen.enwik_like(n)
    enc = rb.DeviceEncoder(0)
    L = enc._L
    cap = L.b200_max_compressed_size(n) + 64
    d_in = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
    out_b = torch.empty(cap, dtype=torch.uint8, device="cuda")
    out_a = torch.empty(cap, dtype=torch.uint8, device="cuda")
    size_a = torch.zeros(1, dtype=torch.int64, device="cuda")
    out_g = torch.empty(cap, dtype=torch.uint8, device="cuda")
    size_g = torch.zeros(1, dtype=torch.int64, device="cuda")
    osz = ctypes.c_size_t(0)

    def blocking():
        if not L.b200_encoder_compress_range(enc._h, q, w, 0, ctypes.c_void_p(d_in.data_ptr()), n, 0, n, 1, 1, 0,
                                             ctypes.c_void_p(out_b.data_ptr()), cap, ctypes.byref(osz), 1):
            raise RuntimeError("blocking call failed")

    def enqueue():
        enc.compress_async(d_in.data_ptr(), n, out_a.data_ptr(), cap, size_a.data_ptr(), q, w,
                           torch.cuda.current_stream().cuda_stream)

    enc.reserve(q, w, n)
    torch.cuda.synchronize()
    blocking()  # warm-up of every path outside the capture
    enqueue()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        enc.compress_async(d_in.data_ptr(), n, out_g.data_ptr(), cap, size_g.data_ptr(), q, w,
                           torch.cuda.current_stream().cuda_stream)
    g.replay()
    torch.cuda.synchronize()
    k = osz.value
    ref = bytes(out_b[:k].cpu().numpy())
    same = (int(size_a.item()) == k and int(size_g.item()) == k and ref == bytes(out_a[:k].cpu().numpy())
            == bytes(out_g[:k].cpu().numpy()))
    if not same:
        raise SystemExit("outputs differ: blocking %d, async %d, graph %d bytes" % (k, int(size_a.item()), int(size_g.item())))

    def timed(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3

    res = {"blocking": [], "async": [], "graph": [], "enqueue": []}
    for r in range(rounds):
        res["blocking"].append(timed(blocking))
        res["async"].append(timed(enqueue))
        res["graph"].append(timed(g.replay))
        torch.cuda.synchronize()  # one async call alone: host time of the enqueue
        t = time.perf_counter()
        enqueue()
        res["enqueue"].append((time.perf_counter() - t) * 1e3)
        torch.cuda.synchronize()
        print(json.dumps({"round": r, "ms_10_steps": {x: round(v[-1], 2) for x, v in res.items() if x != "enqueue"},
                          "enqueue_ms": round(res["enqueue"][-1], 3)}), flush=True)
    med = {x: statistics.median(v) for x, v in res.items()}
    print(json.dumps({"input": "enwik_like 100 MB, HBM-resident", "quality": q, "lgwin": w, "compressed_bytes": k, "steps": steps,
                      "rounds": rounds, "median_ms_10_steps": {x: round(med[x], 2) for x in ("blocking", "async", "graph")},
                      "median_enqueue_ms": round(med["enqueue"], 3),
                      "GB_per_s": {x: round(steps * n / med[x] / 1e6, 2) for x in ("blocking", "async", "graph")},
                      "card": card()}), flush=True)
    enc.close()


if __name__ == "__main__":
    main()

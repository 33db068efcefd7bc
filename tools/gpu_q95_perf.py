"""GPU: quality 9.5 between q9 and q10 -- throughput and compressed size of q9, 9.5 (quality 10 + Q9_5), 9.5x (quality 11 + Q9_5),
q10 and q11 on 100 MB of enwik-shaped text and 100 MB of JSON logs (tools/datagen.py), lgwin 22.

Each configuration compresses a device-resident tensor through compress_tensor(params=...) (one complete stream, as
BrotliEncoderCompressStream with one FINISH makes it); a run is timed with the host clock around the call and a device
synchronise.  Every configuration is warmed up once, then the configurations alternate in each of ROUNDS rounds (default 3),
the bytes of every round must be identical, and the medians are reported with the card's name and power limit.  One JSON line
per (input, configuration), then a summary line; with OUT=<file> the lines are also written there.  Not part of bench.py."""
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIGS = [("q9", 9, False), ("9.5", 10, True), ("9.5x", 11, True), ("q10", 10, False), ("q11", 11, False)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the measurement stands without it
        return "unknown (%s)" % e


def main():
    import torch
    import rust_brotli_b200 as rb
    from tools import datagen
    if not torch.cuda.is_available():
        raise SystemExit("gpu_q95_perf needs a CUDA device")
    n, rounds = int(os.environ.get("BYTES", "100000000")), int(os.environ.get("ROUNDS", "3"))
    enc = rb.DeviceEncoder(0)
    lines = []
    for name, gen in (("text", datagen.enwik_like), ("json", datagen.json_logs)):
        t = torch.frombuffer(bytearray(gen(n)), dtype=torch.uint8).cuda()

        def run(q, q95):
            p = rb.BrotliEncoderParams(quality=q, lgwin=22, q9_5=q95)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out, size = rb.compress_tensor(t, params=p, encoder=enc)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            return dt, int(size.item()), out

        sizes, times = {}, {c[0]: [] for c in CONFIGS}
        for label, q, q95 in CONFIGS:  # warm-up: modules, workspaces
            _, sizes[label], _ = run(q, q95)
        for _ in range(rounds):
            for label, q, q95 in CONFIGS:
                dt, sz, _ = run(q, q95)
                assert sz == sizes[label], (name, label, sz, sizes[label])
                times[label].append(dt)
        for label, q, q95 in CONFIGS:
            med = statistics.median(times[label])
            rec = {"input": name, "config": label, "quality": q, "q9_5": q95, "lgwin": 22, "bytes_in": n, "bytes_out": sizes[label],
                   "ratio": round(n / sizes[label], 4), "vs_q9_pct": round((sizes[label] / sizes["q9"] - 1) * 100, 3),
                   "vs_q10_pct": round((sizes[label] / sizes["q10"] - 1) * 100, 3), "median_s": round(med, 4),
                   "MBps": round(n / med / 1e6, 1), "runs_s": [round(x, 4) for x in times[label]]}
            lines.append(rec)
            print(json.dumps(rec), flush=True)
        del t
    summary = {"card": card(), "rounds": rounds, "timing": "host clock around compress_tensor + torch.cuda.synchronize, medians"}
    lines.append(summary)
    print(json.dumps(summary))
    enc.close()
    if os.environ.get("OUT"):
        with open(os.environ["OUT"], "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()

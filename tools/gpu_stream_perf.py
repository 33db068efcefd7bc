"""GPU: a device-resident stream (DeviceStreamEncoder) against the host stream API (CompressorWriter), both flushing every k bytes
of 100 MB of enwik-shaped text at q5, lgwin 22, for k = 64 KiB, 1 MiB, 8 MiB and 24 MiB.

The host writer takes its input from host memory, and each FLUSH re-uploads the window plus the new bytes and waits for the
piece.  The device stream takes slices of a device tensor and never waits: one synchronise ends the run.  The two alternate in
each round, the bytes of every round must be identical, and the last line gives the medians with the card's name and power limit.
Not part of bench.py."""
import io
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


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
    n, rounds = 100_000_000, int(os.environ.get("ROUNDS", "3"))
    ks = [64 << 10, 1 << 20, 8 << 20, 24 << 20]
    d = datagen.enwik_like(n)
    d_in = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
    params = rb.BrotliEncoderParams(quality=5, lgwin=22)

    def host(k):
        sink = io.BytesIO()
        w = rb.CompressorWriter(sink, 4096, params=params)
        for o in range(0, n, k):
            w.write(d[o:o + k])
            w.flush()
        w.close()
        return sink.getvalue()

    def device(k):
        s = rb.DeviceStreamEncoder(params)
        for o in range(0, n, k):
            s.flush(d_in[o:o + k])
        s.finish()
        out, size, status = s.output()
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        got = bytes(out[:int(size.item())].cpu().numpy())
        s.close()
        return got

    def timed(f, k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f(k)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    device(ks[-1])  # warm-up: the encoder's workspace
    host(ks[-1])
    res = {k: {"host": [], "device": []} for k in ks}
    for r in range(rounds):
        for k in ks:
            th, bh = timed(host, k)
            td, bd = timed(device, k)
            assert bh == bd, "device stream bytes differ from the host stream (k=%d)" % k
            res[k]["host"].append(th)
            res[k]["device"].append(td)
            print(json.dumps({"round": r, "k": k, "host_s": round(th, 4), "device_s": round(td, 4), "bytes": len(bh)}), flush=True)
    summary = {"card": card(), "n": n, "quality": 5, "lgwin": 22, "rounds": rounds}
    for k in ks:
        h, dv = statistics.median(res[k]["host"]), statistics.median(res[k]["device"])
        summary["k=%d" % k] = {"host_MBps": round(n / h / 1e6, 1), "device_MBps": round(n / dv / 1e6, 1), "speedup": round(h / dv, 3)}
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()

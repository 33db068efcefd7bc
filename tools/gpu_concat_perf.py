"""Throughput of b200_concat_async against a device-to-device cudaMemcpyAsync of the same byte count.

Splices 1 GiB of catable streams (uncompressed 16 MiB metablocks, synthetic) in three layouts -- 8 x 128 MiB, 16 384 x 64 KiB,
262 144 x 4 KiB -- and times, with CUDA events, the splice and a copy of the output's byte count alternately in the same run.
Prints one JSON line per layout: GB/s of output for both, their ratio, the card and its power limit.

    python tools/gpu_concat_perf.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def headers(slen):
    """Byte offsets and 4-byte headers of one catable stream of slen bytes: [window 22] ISLAST 0, MNIBBLES 6, MLEN - 1,
    ISUNCOMPRESSED, data; the last byte is the empty last metablock 0x03."""
    block = 1 << 24
    payload_total = slen - 1
    out, pos, first = [], 0, True
    while pos < payload_total:
        room = payload_total - pos - 4
        n = min(block, room)
        bits = []

        def put(k, v):
            bits.extend((v >> i) & 1 for i in range(k))
        if first:
            put(4, ((22 - 17) << 1) | 1)
        put(1, 0); put(2, 2); put(24, n - 1); put(1, 1)
        bits += [0] * (-len(bits) % 8)
        out.append((pos, bytes(sum(bits[i + j] << j for j in range(8)) for i in range(0, len(bits), 8))))
        pos += 4 + n
        first = False
    assert pos == payload_total
    return out


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def main():
    import torch
    import rust_brotli_b200 as rb
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    L = rb._broccoli()
    total = 1 << 30
    card = torch.cuda.get_device_name(0)
    plim = power_limit()
    for count in (8, 16384, 262144):
        slen = total // count
        buf = torch.randint(0, 256, (total,), dtype=torch.uint8, device="cuda")
        v = buf.view(count, slen)
        for off, h in headers(slen):
            v[:, off:off + 4] = torch.tensor(list(h), dtype=torch.uint8, device="cuda")
        v[:, slen - 1] = 3
        ptrs = torch.arange(count, dtype=torch.int64, device="cuda") * slen + buf.data_ptr()
        sizes = torch.full((count,), slen, dtype=torch.int64, device="cuda")
        ws = torch.empty(L.b200_concat_workspace_size(count), dtype=torch.uint8, device="cuda")
        cap = total + 3
        out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        size = torch.zeros(1, dtype=torch.int64, device="cuda")
        res = torch.zeros(2, dtype=torch.int32, device="cuda")
        st = torch.cuda.current_stream()

        def splice():
            assert L.b200_concat_async(ptrs.data_ptr(), sizes.data_ptr(), count, 0, out.data_ptr(), cap, size.data_ptr(),
                                       res.data_ptr(), ws.data_ptr(), ws.numel(), st.cuda_stream)
        splice()
        torch.cuda.synchronize()
        assert res.tolist() == [0, -1], res.tolist()
        nout = int(size.item())
        src, dst = buf[:nout], torch.empty(nout, dtype=torch.uint8, device="cuda")
        for _ in range(3):
            splice()
            dst.copy_(src)
        t_s, t_c = [], []
        for _ in range(a.iters):
            e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            e[0].record(); splice(); e[1].record()
            e[2].record(); dst.copy_(src); e[3].record()
            torch.cuda.synchronize()
            t_s.append(e[0].elapsed_time(e[1]))
            t_c.append(e[2].elapsed_time(e[3]))
        ms_s, ms_c = sorted(t_s)[len(t_s) // 2], sorted(t_c)[len(t_c) // 2]
        print(json.dumps({"layout": "%d x %d B" % (count, slen), "out_bytes": nout, "splice_ms": round(ms_s, 4),
                          "copy_ms": round(ms_c, 4), "splice_GBps": round(nout / ms_s / 1e6, 1), "copy_GBps": round(nout / ms_c / 1e6, 1),
                          "ratio_to_copy": round(ms_c / ms_s, 3), "card": card, "power_limit": plim}), flush=True)
        del buf, out, dst, ws, ptrs, sizes


if __name__ == "__main__":
    main()

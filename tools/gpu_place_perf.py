"""GPU: per-launch device time of the q5 match stage's kernels on the bench workload (100 MB of enwik-shaped text, quality 5,
lgwin 22, bench.py's input), taken with torch.profiler (CUDA activities) over STEPS steps (default 3) with the chunks serialised
on one lane (OPT_LANES = 1), after two warm-up steps.

For k_match_shallow and for each kernel that places best[] (k_best_bin + k_best_tile, or k_best_place in builds before them)
it prints one JSON line: launches, min / mean / max µs per launch, and the achieved rate of the bytes the kernel has to move,
computed from the shapes (every payload position once per step), against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s
(not measured).  The card's name, power limit and clocks are read in the same run.  It times the library of the tree it runs from
(B200_LIB: another build of the same sources, tools/build_variant.sh); to time an earlier commit, run a copy of this file from
that commit's checkout.  Not part of bench.py."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WORKLOAD_BYTES = 100_000_000
DATASHEET_GBS = 3350.0
# bytes per payload position that each kernel must read + write
BYTES_PER_POS = {
    "k_best_place": 8 + 4,   # the (position, value) record, the best[] word
    "k_best_bin": 8 + 8,     # the record from the slab-major staging, the record to the tile-major buffer
    "k_best_tile": 8 + 4,    # the record, the best[] word
}
KERNELS = ["k_match_shallow", "k_best_place", "k_best_bin", "k_best_tile"]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the measurement stands without it
        return "unknown (%s)" % e


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile
    import rust_brotli_b200 as rb
    from tools import datagen
    if not torch.cuda.is_available():
        raise SystemExit("gpu_place_perf needs a CUDA device")
    steps = int(os.environ.get("STEPS", "3"))
    data = datagen.enwik_like(WORKLOAD_BYTES, seed=8)
    enc = rb.DeviceEncoder(0)
    enc.set_option(rb._native.OPT_LANES, 1)
    d_in = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    cap = rb.lib().b200_max_compressed_size(len(data)) + 4096
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")

    def step():
        return enc.compress_device(d_in.data_ptr(), len(data), d_out.data_ptr(), cap, 5, 22)

    sizes = {step() for _ in range(2)}
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            sizes.add(step())
        torch.cuda.synchronize()
    assert len(sizes) == 1, sizes
    times = {k: [] for k in KERNELS}
    for e in prof.events():
        for k in KERNELS:
            if k in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                times[k].append(e.time_range.elapsed_us())
    info = {"card": card(), "lib": os.environ.get("B200_LIB") or "in-tree", "compressed_bytes": sizes.pop(), "steps": steps}
    print(json.dumps(info), flush=True)
    place_us = 0.0
    for k in KERNELS:
        t = times[k]
        if not t:
            continue
        rec = {"kernel": k, "launches": len(t), "us_min": round(min(t), 1), "us_mean": round(sum(t) / len(t), 1), "us_max": round(max(t), 1)}
        if k in BYTES_PER_POS:
            place_us += sum(t)
            gbs = BYTES_PER_POS[k] * WORKLOAD_BYTES * steps / (sum(t) * 1e-6) / 1e9
            rec.update({"bytes_per_position": BYTES_PER_POS[k], "achieved_gbs": round(gbs, 1),
                        "of_datasheet_hbm": round(gbs / DATASHEET_GBS, 3)})
        print(json.dumps(rec), flush=True)
    launches = len(times["k_match_shallow"]) or 1
    print(json.dumps({"placement_us_per_batch": round(place_us / launches, 1),
                      "note": "sum of the placement kernels' time per k_match_shallow launch (one sort batch)"}), flush=True)


if __name__ == "__main__":
    main()

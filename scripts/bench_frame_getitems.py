#!/usr/bin/env python
"""bench_frame_getitems.py -- sparse reads from a frame: K random 64-item ranges of an 8 GiB frame (32 chunks of
256 MiB; bench.c words made on the device, lz4, shuffle, typesize 4, clevel 5), read three ways:

  host_lists  one blosc_b200_frame_getitems call, the range lists in host memory (planned on the host)
  dev_lists   the same call with the lists as int64 CUDA tensors (planned on the GPU)
  full        one blosc_b200_frame_decompress of the whole frame, then a torch index of the same ranges

for K in 1, 16, 256, 4096, 65536, 1048576, with the frame in device memory and then in pinned host memory (dest is
device memory in both).  All results are checked equal before anything is timed.  Each time is the median of --reps
host-timed calls, each ending in a synchronise, after --warmup untimed ones.  Prints the GPU's name and power limit
(read in the same run), one JSON line per (frame residency, K), and the per-kernel CUDA-event times of one call of each
frame_getitems arm (the plan kernels, the chunk plans' and the frame plan's, are "plan").
    python scripts/bench_frame_getitems.py [--reps R] [--warmup W] [--ks 1,16,256,4096,65536,1048576]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import __graft_entry__ as g

WORKLOAD = ("lz4", 1, 4, 5, 8 << 30, 256 << 20)      # compressor, doshuffle, typesize, clevel, nbytes, chunksize
ITEMS = 64


def power_limit():
    """the board's power limit in watts, read with nvidia-smi (None where it cannot be read)"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), min(ts), max(ts)


def bench_words_dev(nbytes):
    """bench.c's words (tests/datagen.py bench_words), made on the device"""
    i = torch.arange(nbytes // 4, dtype=torch.int32, device="cuda")
    return (((i << 26) ^ (i << 18) ^ (i << 11) ^ (i << 3) ^ i) & ((1 << 19) - 1)).view(torch.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ks", default="1,16,256,4096,65536,1048576")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_frame_getitems.py measures on a GPU"
    comp, shuf, ts, clevel, nbytes, cs = WORKLOAD
    pkg = g.load_package()
    d_src = bench_words_dev(nbytes)
    fb = pkg.frame_bound(nbytes, ts, cs)
    d_frame = torch.empty(fb, dtype=torch.uint8, device="cuda")
    fb = pkg.frame_compress(clevel, shuf, ts, nbytes, d_src, d_frame, fb, comp, 0, cs)
    assert fb > 0
    del d_src
    frames = {"device": d_frame[:fb].clone(), "pinned_host": d_frame[:fb].cpu().pin_memory()}
    del d_frame
    d_full = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    nit = nbytes // ts
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit(), "frame_bytes": fb,
                      "workload": "lz4-shuffle-ts4-cl5-8GiB-256MiB-chunks", "items_per_range": ITEMS,
                      "reps": args.reps, "warmup": args.warmup}), flush=True)
    for where, frame in frames.items():
        for k in [int(x) for x in args.ks.split(",")]:
            starts = np.random.default_rng(k).integers(0, nit - ITEMS, k).astype(np.uint64)
            counts = np.full(k, ITEMS, np.uint64)
            rb = ITEMS * ts
            out_host = torch.zeros(k * rb, dtype=torch.uint8, device="cuda")
            out_dev = torch.zeros(k * rb, dtype=torch.uint8, device="cuda")
            d_starts = torch.from_numpy(starts.astype(np.int64)).cuda()
            d_counts = torch.from_numpy(counts.astype(np.int64)).cuda()
            idx = (d_starts * ts)[:, None] + torch.arange(rb, device="cuda")[None, :]
            idx = idx.reshape(-1)

            def host_lists():
                assert pkg.frame_getitems(frame, fb, starts, counts, out_host) == k * rb

            def dev_lists():
                assert pkg.frame_getitems(frame, fb, d_starts, d_counts, out_dev) == k * rb

            def full():
                assert pkg.frame_decompress(frame, fb, d_full, nbytes) == nbytes
                return d_full[idx]

            host_lists(); dev_lists()
            out_full = full()
            torch.cuda.synchronize()
            assert torch.equal(out_host, out_dev) and torch.equal(out_host, out_full), (where, k)
            del out_full
            line = {"frame": where, "k": k}
            for name, fn in (("host_lists", host_lists), ("dev_lists", dev_lists), ("full", full)):
                med, lo, hi = median_ms(fn, args.reps, args.warmup)
                line[name + "_ms"] = round(med, 4)
                line[name + "_range_ms"] = [round(lo, 4), round(hi, 4)]
            line["dev_speedup_vs_host"] = round(line["host_lists_ms"] / line["dev_lists_ms"], 2)
            line["dev_speedup_vs_full"] = round(line["full_ms"] / line["dev_lists_ms"], 2)
            print(json.dumps(line), flush=True)
            for name, fn in (("host_lists", host_lists), ("dev_lists", dev_lists), ("full", full)):
                pkg.set_profiling(True); pkg.prof_reset()
                fn()
                torch.cuda.synchronize()
                prof = pkg.prof_get(); pkg.set_profiling(False)
                print(json.dumps({"frame": where, "k": k, "arm": name,
                                  "kernels_ms": {n: [round(v[0], 4), v[1]] for n, v in prof.items() if v[1]}}),
                      flush=True)


if __name__ == "__main__":
    main()

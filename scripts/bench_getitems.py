#!/usr/bin/env python
"""bench_getitems.py -- sparse reads from one chunk: K random 64-item ranges of the cfg 2 chunk (256 MiB bench.c
buffer, lz4, shuffle, typesize 4, clevel 5), read four ways:

  loop          K blosc_getitem calls (only up to --loop-max ranges)
  getitems      one blosc_b200_getitems call, the range lists in host memory (planned on the host)
  getitems_dev  the same call with the lists as CUDA tensors (planned on the GPU)
  full          one blosc_decompress_ctx of the whole chunk, then a torch index of the same ranges

for K in 1, 16, 256, 4096, 65536, 1048576, with the chunk in device memory and then in pinned host memory (dest is
device memory in both).  All results are checked equal before anything is timed.  Each time is the median of --reps
host-timed calls, each ending in a stream synchronise, after --warmup untimed ones.  Prints the GPU's name and power
limit (read in the same run), one JSON line per (chunk residency, K), and the per-kernel CUDA-event times of one call
of each getitems arm (the GPU plan's kernels are "plan").
    python scripts/bench_getitems.py [--reps R] [--warmup W] [--ks 1,16,256,4096,65536,1048576] [--loop-max 4096]"""
import argparse
import json
import os
import statistics
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import __graft_entry__ as g
from datagen import bench_words

WORKLOAD = ("lz4", 1, 4, 5, 256 << 20)      # compressor, doshuffle, typesize, clevel, nbytes
ITEMS = 64


def power_limit():
    """the board's power limit in watts, read with nvidia-smi (None where it cannot be read)"""
    import subprocess
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ks", default="1,16,256,4096,65536,1048576")
    ap.add_argument("--loop-max", type=int, default=4096)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_getitems.py measures on a GPU"
    comp, shuf, ts, clevel, nbytes = WORKLOAD
    pkg = g.load_package()
    d_src = torch.from_numpy(bench_words(nbytes)).cuda()
    d_chunk = torch.zeros(nbytes + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(clevel, shuf, ts, nbytes, d_src, d_chunk, nbytes + 16, comp)
    assert cb > 0
    chunks = {"device": d_chunk[:cb].clone(), "pinned_host": d_chunk[:cb].cpu().pin_memory()}
    d_full = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    nit = nbytes // ts
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit(), "cbytes": cb,
                      "workload": "lz4-shuffle-ts4-cl5-256MiB", "items_per_range": ITEMS, "reps": args.reps,
                      "warmup": args.warmup}), flush=True)
    for where, chunk in chunks.items():
        for k in [int(x) for x in args.ks.split(",")]:
            starts = np.random.default_rng(k).integers(0, nit - ITEMS, k).astype(np.int32)
            counts = np.full(k, ITEMS, np.int32)
            rb = ITEMS * ts
            out_loop = torch.zeros(k * rb, dtype=torch.uint8, device="cuda")
            out_many = torch.zeros(k * rb, dtype=torch.uint8, device="cuda")
            out_dev = torch.zeros(k * rb, dtype=torch.uint8, device="cuda")
            d_starts, d_counts = torch.from_numpy(starts).cuda(), torch.from_numpy(counts).cuda()
            idx = (torch.from_numpy(starts.astype(np.int64) * ts).cuda()[:, None]
                   + torch.arange(rb, device="cuda")[None, :]).reshape(-1)
            base = out_loop.data_ptr()
            st_list = starts.tolist()

            def loop():
                for r, s in enumerate(st_list):
                    assert pkg.lib.blosc_getitem(pkg._ptr(chunk), s, ITEMS, base + r * rb) == rb

            def many():
                assert pkg.getitems(chunk, starts, counts, out_many) == k * rb

            def many_dev():
                assert pkg.getitems(chunk, d_starts, d_counts, out_dev) == k * rb

            def full():
                assert pkg.decompress_ctx(chunk, d_full, nbytes) == nbytes
                return d_full[idx]

            arms = [("getitems", many), ("getitems_dev", many_dev), ("full", full)]
            if k <= args.loop_max:
                arms.insert(0, ("loop", loop))
                loop()
            many(); many_dev()
            out_full = full()
            torch.cuda.synchronize()
            if k <= args.loop_max:
                assert torch.equal(out_loop, out_many), (where, k)
            assert torch.equal(out_many, out_dev) and torch.equal(out_many, out_full), (where, k)
            assert torch.equal(out_many, d_src[idx])
            line = {"chunk": where, "k": k}
            for name, fn in arms:
                med, lo, hi = median_ms(fn, args.reps, args.warmup)
                line[name + "_ms"] = round(med, 4)
                line[name + "_range_ms"] = [round(lo, 4), round(hi, 4)]
            if "loop_ms" in line:
                line["speedup_vs_loop"] = round(line["loop_ms"] / line["getitems_ms"], 2)
            line["speedup_vs_full"] = round(line["full_ms"] / line["getitems_ms"], 2)
            line["dev_speedup_vs_full"] = round(line["full_ms"] / line["getitems_dev_ms"], 2)
            print(json.dumps(line), flush=True)
            for name, fn in (("getitems", many), ("getitems_dev", many_dev)):
                pkg.set_profiling(True); pkg.prof_reset()
                fn()
                prof = pkg.prof_get(); pkg.set_profiling(False)
                print(json.dumps({"chunk": where, "k": k, "arm": name,
                                  "kernels_ms": {n: round(v[0], 4) for n, v in prof.items() if v[1]}}), flush=True)


if __name__ == "__main__":
    main()

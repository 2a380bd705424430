#!/usr/bin/env python
"""bench_getslice.py -- boxes of N-d arrays read from a 256 MiB chunk and from an 8 GiB frame of 32 such chunks
(bench.c words made on the device, lz4, shuffle, typesize 4, clevel 5), read three ways:

  getslice   one blosc_b200_getslice / blosc_b200_frame_getslice call with the box
  getitems   one blosc_b200_getitems / blosc_b200_frame_getitems call with one range per innermost run, the range lists
             as CUDA tensors (int32 for the chunk, int64 for the frame; planned on the GPU)
  full       a full blosc_decompress_ctx / frame_decompress, then a torch slice made contiguous

The boxes: a few rows (16 runs), a 2-D tile, a 3-D sub-cube and a column of 2^24 runs of one item.  The data is in
device memory, then in pinned host memory; dest is device memory.  All three results are checked equal first.  The
arms are then alternated --reps times in the same process, each call host-timed up to a device synchronise, after
--warmup untimed calls of each; medians and ranges are printed as one JSON line per (data, residency, box), after a
line with the GPU's name and power limit read in the same run, and followed by the CUDA-event kernel times of one
getslice call.
    python scripts/bench_getslice.py [--reps R] [--warmup W] [--no-frame]"""
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
import torch

import __graft_entry__ as g

TS, CHUNK = 4, 256 << 20
NCHUNKS = 32
ITEMS = CHUNK // TS                                   # 2^26 items a chunk
# (name, shape, start, stop) over one chunk's 2^26 items; the frame's boxes scale the first dimension by NCHUNKS
BOXES = (("rows", (1 << 16, 1024), (30000, 0), (30016, 1000)),
         ("tile", (8192, 8192), (1000, 2000), (3048, 4048)),
         ("cube", (256, 512, 512), (64, 128, 128), (128, 256, 256)),
         ("column", (1 << 24, 4), (0, 1), (1 << 24, 2)))
FRAME_BOXES = (("rows", (NCHUNKS << 16, 1024), (65530, 0), (65546, 1000)),                 # across chunks 0 and 1
               ("tile", (NCHUNKS * 8192, 8192), (7000, 2000), (9048, 4048)),
               ("cube", (NCHUNKS * 256, 512, 512), (230, 128, 128), (294, 256, 256)),
               ("column", (NCHUNKS << 24, 4), (3 << 23, 1), ((3 << 23) + (1 << 24), 2)))


def power_limit():
    """the board's power limit in watts, read with nvidia-smi (None where it cannot be read)"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def bench_words_dev(nbytes):
    """bench.c's words (tests/datagen.py bench_words), made on the device"""
    i = torch.arange(nbytes // 4, dtype=torch.int32, device="cuda")
    return (((i << 26) ^ (i << 18) ^ (i << 11) ^ (i << 3) ^ i) & ((1 << 19) - 1)).view(torch.uint8)


def runs_dev(shape, start, stop, dtype):
    """the box as one range per innermost run, on the device: flat starts and counts"""
    ext = [e - s for s, e in zip(start, stop)]
    stride = [1] * len(shape)
    for k in range(len(shape) - 2, -1, -1):
        stride[k] = stride[k + 1] * shape[k + 1]
    r = 1
    for e in ext[:-1]:
        r *= e
    p = torch.arange(r, dtype=torch.int64, device="cuda")
    flat = torch.full_like(p, start[-1])
    for k in range(len(shape) - 2, -1, -1):
        flat += (start[k] + p % ext[k]) * stride[k]
        p //= ext[k]
    return flat.to(dtype), torch.full((r,), ext[-1], dtype=dtype, device="cuda")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-frame", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_getslice.py measures on a GPU"
    pkg = g.load_package()
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit(),
                      "workload": "lz4-shuffle-ts4-cl5-256MiB-chunk, frame of 32", "reps": args.reps,
                      "warmup": args.warmup}), flush=True)
    d_src = bench_words_dev(CHUNK)
    d_chunk = torch.empty(CHUNK + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(5, 1, TS, CHUNK, d_src, d_chunk, CHUNK + 16, "lz4")
    assert cb > 0
    del d_src
    datas = [("chunk", "device", d_chunk[:cb].clone()), ("chunk", "pinned_host", d_chunk[:cb].cpu().pin_memory())]
    del d_chunk
    if not args.no_frame:
        nbytes = NCHUNKS * CHUNK
        d_src = bench_words_dev(nbytes)
        fb = pkg.frame_bound(nbytes, TS, CHUNK)
        d_frame = torch.empty(fb, dtype=torch.uint8, device="cuda")
        fb = pkg.frame_compress(5, 1, TS, nbytes, d_src, d_frame, fb, "lz4", 0, CHUNK)
        assert fb > 0
        del d_src
        datas += [("frame", "device", d_frame[:fb].clone()), ("frame", "pinned_host", d_frame[:fb].cpu().pin_memory())]
        del d_frame
    for kind, where, data in datas:
        size = data.numel()
        nbytes = CHUNK if kind == "chunk" else NCHUNKS * CHUNK
        d_full = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        for name, shape, start, stop in (BOXES if kind == "chunk" else FRAME_BOXES):
            nout = TS
            for s, e in zip(start, stop):
                nout *= e - s
            st, nn = runs_dev(shape, start, stop, torch.int32 if kind == "chunk" else torch.int64)
            outs = {a: torch.empty(nout, dtype=torch.uint8, device="cuda") for a in ("getslice", "getitems")}
            sl = tuple(slice(s, e) for s, e in zip(start, stop))

            def getslice():
                if kind == "chunk":
                    assert pkg.getslice(data, shape, start, stop, outs["getslice"]) == nout
                else:
                    assert pkg.frame_getslice(data, size, shape, start, stop, outs["getslice"]) == nout

            def getitems():
                if kind == "chunk":
                    assert pkg.getitems(data, st, nn, outs["getitems"]) == nout
                else:
                    assert pkg.frame_getitems(data, size, st, nn, outs["getitems"]) == nout

            def full():
                if kind == "chunk":
                    assert pkg.decompress_ctx(data, d_full, nbytes) == nbytes
                else:
                    assert pkg.frame_decompress(data, size, d_full, nbytes) == nbytes
                return d_full.view(torch.int32).view(*shape)[sl].contiguous().view(torch.uint8).reshape(-1)

            arms = (("getslice", getslice), ("getitems", getitems), ("full", full))
            getslice(); getitems()
            ref = full()
            torch.cuda.synchronize()
            assert torch.equal(outs["getslice"], ref) and torch.equal(outs["getitems"], ref), (kind, where, name)
            del ref
            for _, fn in arms:
                for _ in range(args.warmup):
                    fn()
            times = {a: [] for a, _ in arms}
            for _ in range(args.reps):
                for a, fn in arms:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    times[a].append((time.perf_counter() - t0) * 1e3)
            line = {"data": kind, "residency": where, "box": name, "shape": shape, "start": start, "stop": stop,
                    "runs": st.numel(), "out_bytes": nout}
            for a, _ in arms:
                line[a + "_ms"] = round(statistics.median(times[a]), 4)
                line[a + "_range_ms"] = [round(min(times[a]), 4), round(max(times[a]), 4)]
            print(json.dumps(line), flush=True)
            pkg.set_profiling(True); pkg.prof_reset()
            getslice()
            torch.cuda.synchronize()
            prof = pkg.prof_get(); pkg.set_profiling(False)
            print(json.dumps({"data": kind, "residency": where, "box": name, "arm": "getslice",
                              "kernels_ms": {n: [round(v[0], 4), v[1]] for n, v in prof.items() if v[1]}}), flush=True)
            del st, nn, outs
        del d_full


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""bench_getslices.py -- batches of K equal patches at seeded random corners, read from a 256 MiB chunk and from an
8 GiB frame of 32 such chunks (bench.c words made on the device, lz4, shuffle, typesize 4, clevel 5), three ways:

  getslices  one blosc_b200_getslices / blosc_b200_frame_getslices call, the corners an int64 CUDA tensor
  loop       K blosc_b200_getslice / frame_getslice calls, one per patch (up to K = 256; the corners are read on the
             host once, outside the timing)
  full       a full blosc_decompress_ctx / frame_decompress, then one torch gather of the K patches (advanced indexing)

The patches: 64x64x64 cubes of the chunk read as (256, 512, 512) and of the frame read as (8192, 512, 512), and
256x256 tiles of the chunk read as (8192, 8192); K = 1, 16, 256, 4096.  The data and dest are device memory.  All arms'
outputs are checked equal first.  The arms are then alternated --reps times in the same process, each call host-timed
up to a device synchronise, after --warmup untimed calls of each; medians and ranges are printed as one JSON line per
(data, patch, K), after a line with the GPU's name and power limit read in the same run.
    python scripts/bench_getslices.py [--reps R] [--warmup W] [--no-frame]"""
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

TS, CHUNK, NCHUNKS = 4, 256 << 20, 32
KS = (1, 16, 256, 4096)
LOOP_MAX_K = 256
CASES = (("chunk", "cube", (256, 512, 512), (64, 64, 64)),
         ("chunk", "tile", (8192, 8192), (256, 256)),
         ("frame", "cube", (NCHUNKS * 256, 512, 512), (64, 64, 64)))


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


def gather_index(starts, extent):
    """advanced-indexing tensors that pick K patches of `extent` at `starts` (K, ndim), broadcast to (K, *extent)"""
    k, nd = starts.shape
    idx = []
    for d in range(nd):
        view = [k] + [1] * nd
        ar = [1] * (nd + 1)
        ar[d + 1] = extent[d]
        idx.append(starts[:, d].view(view) + torch.arange(extent[d], device="cuda").view(ar))
    return tuple(idx)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-frame", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_getslices.py measures on a GPU"
    pkg = g.load_package()
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit(),
                      "workload": "lz4-shuffle-ts4-cl5-256MiB-chunk, frame of 32", "reps": args.reps,
                      "warmup": args.warmup}), flush=True)
    datas = {}
    d_src = bench_words_dev(CHUNK)
    d_chunk = torch.empty(CHUNK + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(5, 1, TS, CHUNK, d_src, d_chunk, CHUNK + 16, "lz4")
    assert cb > 0
    datas["chunk"] = (d_chunk[:cb].clone(), CHUNK)
    del d_src, d_chunk
    if not args.no_frame:
        nbytes = NCHUNKS * CHUNK
        d_src = bench_words_dev(nbytes)
        fb = pkg.frame_bound(nbytes, TS, CHUNK)
        d_frame = torch.empty(fb, dtype=torch.uint8, device="cuda")
        fb = pkg.frame_compress(5, 1, TS, nbytes, d_src, d_frame, fb, "lz4", 0, CHUNK)
        assert fb > 0
        datas["frame"] = (d_frame[:fb].clone(), nbytes)
        del d_src, d_frame
    gen = torch.Generator(device="cuda").manual_seed(2026)
    for kind, patch, shape, extent in CASES:
        if kind not in datas:
            continue
        data, nbytes = datas[kind]
        size = data.numel()
        d_full = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        pb = TS
        for e in extent:
            pb *= e
        for k in KS:
            starts = torch.stack([torch.randint(0, s - e + 1, (k,), device="cuda", generator=gen)
                                  for s, e in zip(shape, extent)], dim=1)
            idx = gather_index(starts, extent)
            h_starts = starts.cpu().tolist()
            nout = k * pb
            outs = {a: torch.empty(nout, dtype=torch.uint8, device="cuda") for a in ("getslices", "loop")}
            one = pkg.getslice if kind == "chunk" else \
                (lambda d, sh, st, sp, o: pkg.frame_getslice(d, size, sh, st, sp, o))

            def getslices():
                if kind == "chunk":
                    assert pkg.getslices(data, shape, extent, starts, outs["getslices"]) == nout
                else:
                    assert pkg.frame_getslices(data, size, shape, extent, starts, outs["getslices"]) == nout

            def loop():
                o = outs["loop"]
                for i, c in enumerate(h_starts):
                    assert one(data, shape, c, [a + e for a, e in zip(c, extent)], o[i * pb:(i + 1) * pb]) == pb

            def full():
                if kind == "chunk":
                    assert pkg.decompress_ctx(data, d_full, nbytes) == nbytes
                else:
                    assert pkg.frame_decompress(data, size, d_full, nbytes) == nbytes
                return d_full.view(torch.int32).view(*shape)[idx].reshape(-1).view(torch.uint8)

            arms = [("getslices", getslices)] + ([("loop", loop)] if k <= LOOP_MAX_K else []) + [("full", full)]
            for a, fn in arms:
                if a != "full":
                    fn()
            ref = full()
            torch.cuda.synchronize()
            for a, _ in arms:
                if a != "full":
                    assert torch.equal(outs[a], ref), (kind, patch, k, a)
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
            line = {"data": kind, "patch": patch, "shape": shape, "extent": extent, "k": k, "out_bytes": nout}
            for a, _ in arms:
                line[a + "_ms"] = round(statistics.median(times[a]), 4)
                line[a + "_range_ms"] = [round(min(times[a]), 4), round(max(times[a]), 4)]
            print(json.dumps(line), flush=True)
            del outs, idx, starts
        del d_full


if __name__ == "__main__":
    main()

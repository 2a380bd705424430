#!/usr/bin/env python
"""bench_getoindex.py -- orthogonal index selections (numpy's a[np.ix_(...)]) read from a 256 MiB chunk and from an
8 GiB frame of 32 such chunks (bench.c words made on the device, lz4, shuffle, typesize 4, clevel 5), read up to three
ways:

  oindex     one blosc_b200_getoindex / blosc_b200_frame_getoindex call, the lists int64 CUDA tensors
  getslices  one blosc_b200_getslices / blosc_b200_frame_getslices call with one corner per selected row, the corners a
             CUDA tensor; only where the list is on the rows alone (a row is then one box)
  full       a full blosc_decompress_ctx / frame_decompress, then torch advanced indexing

The selections, on the chunk read as 8192 x 8192 float32 (the frame: 262144 x 8192): 1024 random rows x all columns,
with the list unsorted and sorted; all rows x 256 random columns; 512 random rows x 512 random columns (np.ix_); and a
1-d list of 10^5 random items.  The data is in device memory, then in pinned host memory; dest is device memory.  All
results are checked equal first.  The arms are then alternated --reps times in the same process, each call host-timed
up to a device synchronise, after --warmup untimed calls of each; medians and ranges are printed as one JSON line per
(data, residency, selection), after a line with the GPU's name and power limit read in the same run, and followed by
the CUDA-event kernel times of one oindex call.
    python scripts/bench_getoindex.py [--reps R] [--warmup W] [--no-frame]"""
import argparse
import json
import os
import statistics
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch

import __graft_entry__ as g
from bench_getslice import bench_words_dev, power_limit

TS, CHUNK = 4, 256 << 20
NCHUNKS = 32
SIDE = 8192                                            # a chunk is SIDE x SIDE items


def selections(rows, gen):
    """(name, shape, selection, rows_only) over `rows` x SIDE items; rows_only: the list is on the rows alone"""
    r = torch.randperm(rows, device="cuda", generator=gen)[:1024]
    c = torch.randperm(SIDE, device="cuda", generator=gen)[:256]
    r2 = torch.randperm(rows, device="cuda", generator=gen)[:512]
    c2 = torch.randperm(SIDE, device="cuda", generator=gen)[:512]
    flat = torch.randint(0, rows * SIDE, (100000,), device="cuda", generator=gen)
    return (("rows_1024", (rows, SIDE), [r, slice(None)], True),
            ("rows_1024_sorted", (rows, SIDE), [r.sort().values, slice(None)], True),
            ("cols_256", (rows, SIDE), [slice(None), c], False),
            ("ix_512x512", (rows, SIDE), [r2, c2], False),
            ("flat_1e5", (rows * SIDE,), [flat], True))


def torch_index(a, sel):
    """a[np.ix_(...)] of a torch tensor, slices kept"""
    out = a
    for k, s in enumerate(sel):
        out = out[(slice(None),) * k + (s,)]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-frame", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_getoindex.py measures on a GPU"
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
        gen = torch.Generator(device="cuda").manual_seed(7)
        for name, shape, sel, rows_only in selections(SIDE if kind == "chunk" else NCHUNKS * SIDE, gen):
            nout = TS
            for s, n in zip(sel, shape):
                nout *= n if isinstance(s, slice) else s.numel()
            arms = ["oindex"] + (["getslices"] if rows_only else []) + ["full"]
            outs = {a: torch.empty(nout, dtype=torch.uint8, device="cuda") for a in arms[:-1]}
            if rows_only:                               # one corner per selected row: (row, 0), extent (1, SIDE)
                corners = torch.stack([sel[0], torch.zeros_like(sel[0])], 1) if len(shape) == 2 else sel[0].view(-1, 1)
                corners, extent = corners.contiguous(), ((1, SIDE) if len(shape) == 2 else (1,))

            def oindex_arm():
                if kind == "chunk":
                    assert pkg.getoindex(data, shape, sel, outs["oindex"]) == nout
                else:
                    assert pkg.frame_getoindex(data, size, shape, sel, outs["oindex"]) == nout

            def getslices_arm():
                if kind == "chunk":
                    assert pkg.getslices(data, shape, extent, corners, outs["getslices"]) == nout
                else:
                    assert pkg.frame_getslices(data, size, shape, extent, corners, outs["getslices"]) == nout

            def full_arm():
                if kind == "chunk":
                    assert pkg.decompress_ctx(data, d_full, nbytes) == nbytes
                else:
                    assert pkg.frame_decompress(data, size, d_full, nbytes) == nbytes
                return torch_index(d_full.view(torch.int32).view(*shape), sel).contiguous().view(torch.uint8).reshape(-1)

            fns = {"oindex": oindex_arm, "getslices": getslices_arm, "full": full_arm}
            for a in arms[:-1]:
                fns[a]()
            ref = full_arm()
            torch.cuda.synchronize()
            for a in arms[:-1]:
                assert torch.equal(outs[a], ref), (kind, where, name, a)
            del ref
            for a in arms:
                for _ in range(args.warmup):
                    fns[a]()
            times = {a: [] for a in arms}
            for _ in range(args.reps):
                for a in arms:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fns[a]()
                    torch.cuda.synchronize()
                    times[a].append((time.perf_counter() - t0) * 1e3)
            line = {"data": kind, "residency": where, "sel": name, "shape": shape, "out_bytes": nout}
            for a in arms:
                line[a + "_ms"] = round(statistics.median(times[a]), 4)
                line[a + "_range_ms"] = [round(min(times[a]), 4), round(max(times[a]), 4)]
            print(json.dumps(line), flush=True)
            pkg.set_profiling(True); pkg.prof_reset()
            oindex_arm()
            torch.cuda.synchronize()
            prof = pkg.prof_get(); pkg.set_profiling(False)
            print(json.dumps({"data": kind, "residency": where, "sel": name, "arm": "oindex",
                              "kernels_ms": {n: [round(v[0], 4), v[1]] for n, v in prof.items() if v[1]}}), flush=True)
            del outs
        del d_full


if __name__ == "__main__":
    main()

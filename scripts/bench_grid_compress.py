#!/usr/bin/env python
"""bench_grid_compress.py -- float32 arrays written as a regular grid of chunks (zarr v2 / HDF5 blosc layout; bench.c
words made on the device, lz4, shuffle, typesize 4, clevel 5), four ways:

  grid      one blosc_b200_grid_compress call, with BLOSC_B200_FRAME_WORKERS at 1 (grid_w1) and at its default (grid)
  loop      today's loop: per chunk a torch slice, padded into a zeroed chunk at the edge, made contiguous,
            compress_ctx into a scratch buffer and a clone of the chunk's bytes
  frame     a ceiling, not a way to write the grid: frame_compress of the array's bytes at chunksize = chunk bytes, which
            compresses as many equal-sized chunks (fewer at the edge grid) with no packing and one header and index

The grids: 16384^2 in 1024^2 chunks (4 MiB, 256 chunks), 512^3 in 64^3 chunks (1 MiB, 512 chunks), 16000^2 in 1024^2
chunks (edge padding), the 512^3 grid with 7/8 of its chunks all zero, written with and without skip_fill (loop_skip
tests each chunk for a non-zero item first), and 8192^2 in 1024^2 chunks from a pinned host array (to device dest).  The
grid and loop results are checked byte-identical first.  The arms are then alternated --reps times, each call host-timed
up to a device synchronise, after --warmup untimed calls of each; medians and ranges are printed as one JSON line per
grid, after a line with the GPU's name and power limit read in the same run, and followed by the CUDA-event kernel
times of one grid call.
    python scripts/bench_grid_compress.py [--reps R] [--warmup W]"""
import argparse
import itertools
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

TS = 4
# (name, shape, chunkshape, sparse, host src)
GRIDS = (("2d_1024", (16384, 16384), (1024, 1024), False, False),
         ("3d_64", (512, 512, 512), (64, 64, 64), False, False),
         ("2d_1024_edge", (16000, 16000), (1024, 1024), False, False),
         ("3d_64_sparse", (512, 512, 512), (64, 64, 64), True, False),
         ("2d_1024_pinned", (8192, 8192), (1024, 1024), False, True))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_grid_compress.py measures on a GPU"
    pkg = g.load_package()
    default_workers = os.environ.get("BLOSC_B200_FRAME_WORKERS")
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit(),
                      "workload": "float32 grids, lz4-shuffle-ts4-cl5 chunks", "reps": args.reps,
                      "warmup": args.warmup}), flush=True)
    for gname, shape, cs, sparse, host in GRIDS:
        nitems = 1
        for s in shape:
            nitems *= s
        src = bench_words_dev(nitems * TS).view(torch.float32).view(*shape)
        ngrid = [-(-s // c) for s, c in zip(shape, cs)]
        if sparse:                                             # keep the chunks whose coordinates are all even
            keep = torch.zeros(ngrid, dtype=torch.bool, device="cuda")
            keep[tuple(slice(0, None, 2) for _ in ngrid)] = True
            for k, c in enumerate(cs):
                keep = keep.repeat_interleave(c, dim=k)
            src = src * keep
            del keep
        if host:
            src = src.cpu().pin_memory()
        cbytes = TS
        for c in cs:
            cbytes *= c
        coords = list(itertools.product(*(range(n) for n in ngrid)))
        bound = pkg.grid_bound(shape, cs, TS)
        dest = torch.empty(bound, dtype=torch.uint8, device="cuda")
        scratch = torch.empty(cbytes + 16, dtype=torch.uint8, device="cuda")
        nbytes = nitems * TS
        fdest = torch.empty(pkg.frame_bound(nbytes, TS, cbytes), dtype=torch.uint8, device="cuda")

        def grid_arm(workers, skip=False):
            if workers:
                os.environ["BLOSC_B200_FRAME_WORKERS"] = workers
            elif default_workers is None:
                os.environ.pop("BLOSC_B200_FRAME_WORKERS", None)
            else:
                os.environ["BLOSC_B200_FRAME_WORKERS"] = default_workers
            r, off = pkg.grid_compress(src, shape, cs, TS, 5, 1, "lz4", dest, skip_fill=skip)
            assert r > 0
            return r, off

        def loop_arm(skip=False):
            out = []
            for co in coords:
                part = src[tuple(slice(c * k, (c + 1) * k) for c, k in zip(co, cs))]
                if skip and not bool(part.any()):
                    out.append(None)
                    continue
                if tuple(part.shape) != cs:
                    buf = torch.zeros(cs, dtype=torch.float32, device=part.device)
                    buf[tuple(slice(0, e) for e in part.shape)] = part
                    part = buf
                part = part.contiguous()
                cb = pkg.compress_ctx(5, 1, TS, cbytes, part, scratch, cbytes + 16, "lz4")
                assert cb > 0
                out.append(scratch[:cb].clone())
            return out

        def frame_arm():
            assert pkg.frame_compress(5, 1, TS, nbytes, src, fdest, fdest.numel(), "lz4", chunksize=cbytes) > 0

        fns = {"grid_w1": lambda: grid_arm("1"), "grid": lambda: grid_arm(None), "loop": loop_arm, "frame": frame_arm}
        if sparse:
            fns["grid_skip"] = lambda: grid_arm(None, True)
            fns["loop_skip"] = lambda: loop_arm(True)
        # the same bytes from every way of writing the grid
        want = torch.cat([c.cpu() for c in loop_arm()])
        for a in ("grid_w1", "grid"):
            dest.fill_(0xAA)
            r, off = fns[a]()
            assert r == want.numel() and torch.equal(dest[:r].cpu(), want), (gname, a)
        if sparse:
            kept = [c for c in loop_arm(True) if c is not None]
            r, off = fns["grid_skip"]()
            assert r == sum(c.numel() for c in kept) and torch.equal(dest[:r].cpu(), torch.cat([c.cpu() for c in kept]))
            nskipped = int(sum(off[1:] == off[:-1]))
        del want
        for a in fns:
            for _ in range(args.warmup):
                fns[a]()
        torch.cuda.synchronize()
        times = {a: [] for a in fns}
        for _ in range(args.reps):
            for a in fns:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fns[a]()
                torch.cuda.synchronize()
                times[a].append((time.perf_counter() - t0) * 1e3)
        line = {"grid": gname, "shape": shape, "chunkshape": cs, "src": "pinned host" if host else "device",
                "chunks": len(coords), "array_bytes": nbytes, "grid_bytes": r if not sparse else int(off[-1])}
        if sparse:
            line["skipped"] = nskipped
        for a in fns:
            line[a + "_ms"] = round(statistics.median(times[a]), 3)
            line[a + "_range_ms"] = [round(min(times[a]), 3), round(max(times[a]), 3)]
        print(json.dumps(line), flush=True)
        pkg.set_profiling(True); pkg.prof_reset()
        fns["grid"]()
        torch.cuda.synchronize()
        prof = pkg.prof_get(); pkg.set_profiling(False)
        print(json.dumps({"grid": gname, "arm": "grid",
                          "kernels_ms": {n: [round(v[0], 4), v[1]] for n, v in prof.items() if v[1]}}), flush=True)
        del src, dest, scratch, fdest
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

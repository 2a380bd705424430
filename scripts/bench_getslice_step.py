#!/usr/bin/env python
"""bench_getslice_step.py -- strided selections a[start:stop:step] read from a 256 MiB chunk and from an 8 GiB frame of
32 such chunks (bench.c words made on the device, lz4, shuffle, typesize 4, clevel 5), read up to three ways:

  step       one blosc_b200_getslice_step / blosc_b200_frame_getslice_step call with the box and its steps
  getslices  one blosc_b200_getslices / blosc_b200_frame_getslices call with one corner per selected row, the corners
             a CUDA tensor; only where the step is on outer dimensions alone (a row is then one box)
  full       a full blosc_decompress_ctx / frame_decompress, then a torch strided slice made contiguous

The selections, on the chunk read as 8192 x 8192 float32 (the frame: 32 times the rows): [::2, ::2] (every block
touched, one-item runs), [::16, 3::16], every 1024th row, the column [::4, 17], and the 1-d [::2**20], which skips
most blocks.  The data is in device memory, then in pinned host memory; dest is device memory.  All results are
checked equal first.  The arms are then alternated --reps times in the same process, each call host-timed up to a
device synchronise, after --warmup untimed calls of each; medians and ranges are printed as one JSON line per (data,
residency, selection), after a line with the GPU's name and power limit read in the same run, and followed by the
CUDA-event kernel times of one stepped call.
    python scripts/bench_getslice_step.py [--reps R] [--warmup W] [--no-frame]"""
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


def selections(rows):
    """(name, shape, start, stop, step, rows_only) over `rows` x SIDE items; rows_only: the step is on the rows alone"""
    n = rows * SIDE
    return (("half", (rows, SIDE), (0, 0), (rows, SIDE), (2, 2), False),
            ("sixteenth", (rows, SIDE), (0, 3), (rows, SIDE), (16, 16), False),
            ("rows_1024", (rows, SIDE), (0, 0), (rows, SIDE), (1024, 1), True),
            ("column_4", (rows, SIDE), (0, 17), (rows, 18), (4, 1), True),
            ("flat_2^20", (n,), (0,), (n,), (1 << 20,), True))


def row_corners(shape, start, stop, step):
    """one corner per selected row (the last dimension's box whole in each): corners and the extent"""
    lead = [torch.arange(s, e, t, dtype=torch.int64, device="cuda") for s, e, t in zip(start[:-1], stop[:-1], step[:-1])]
    if len(shape) == 1:                                 # a 1-d selection: one one-item box per selected item
        c = torch.arange(start[0], stop[0], step[0], dtype=torch.int64, device="cuda")
        return c.view(-1, 1).contiguous(), (1,)
    grid = torch.cartesian_prod(*lead) if len(lead) > 1 else lead[0]
    corners = torch.cat([grid.view(grid.shape[0], -1), torch.full((grid.shape[0], 1), start[-1], dtype=torch.int64,
                                                                   device="cuda")], 1).contiguous()
    return corners, [1] * (len(shape) - 1) + [stop[-1] - start[-1]]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-frame", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_getslice_step.py measures on a GPU"
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
        for name, shape, start, stop, step, rows_only in selections(SIDE if kind == "chunk" else NCHUNKS * SIDE):
            nout = TS
            for s, e, t in zip(start, stop, step):
                nout *= (e - s - 1) // t + 1
            sl = tuple(slice(s, e, t) for s, e, t in zip(start, stop, step))
            arms = ["step"] + (["getslices"] if rows_only else []) + ["full"]
            outs = {a: torch.empty(nout, dtype=torch.uint8, device="cuda") for a in arms[:-1]}
            corners, extent = row_corners(shape, start, stop, step) if rows_only else (None, None)

            def step_arm():
                if kind == "chunk":
                    assert pkg.getslice(data, shape, start, stop, outs["step"], step=step) == nout
                else:
                    assert pkg.frame_getslice(data, size, shape, start, stop, outs["step"], step=step) == nout

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
                return d_full.view(torch.int32).view(*shape)[sl].contiguous().view(torch.uint8).reshape(-1)

            fns = {"step": step_arm, "getslices": getslices_arm, "full": full_arm}
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
            line = {"data": kind, "residency": where, "sel": name, "shape": shape, "start": start, "stop": stop,
                    "step": step, "out_bytes": nout}
            for a in arms:
                line[a + "_ms"] = round(statistics.median(times[a]), 4)
                line[a + "_range_ms"] = [round(min(times[a]), 4), round(max(times[a]), 4)]
            print(json.dumps(line), flush=True)
            pkg.set_profiling(True); pkg.prof_reset()
            step_arm()
            torch.cuda.synchronize()
            prof = pkg.prof_get(); pkg.set_profiling(False)
            print(json.dumps({"data": kind, "residency": where, "sel": name, "arm": "step",
                              "kernels_ms": {n: [round(v[0], 4), v[1]] for n, v in prof.items() if v[1]}}), flush=True)
            del outs, corners
        del d_full


if __name__ == "__main__":
    main()

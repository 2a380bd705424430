#!/usr/bin/env python
"""bench_grid_getslice.py -- boxes of float32 arrays stored as a regular grid of chunks (zarr v2 / HDF5 blosc layout;
bench.c words made on the device, lz4, shuffle, typesize 4, clevel 5, chunks in device memory), read three ways:

  grid      one blosc_b200_grid_getslice call, with BLOSC_B200_FRAME_WORKERS at 1 (grid_w1) and at its default (grid)
  loop      a Python loop of getslice_step per touched chunk into a temporary, then a torch copy into place
  full      decompress_ctx of every touched chunk into a staging array, then a torch slice made contiguous

The grids: 16384 x 16384 in 1024 x 1024 chunks (4 MiB, 256 chunks) and 512^3 in 64^3 chunks (1 MiB, 512 chunks).  The
selections on each: an unaligned tile touching 5 x 5 (x 5) chunks, a 10-column band across every chunk row, [::8] in
every dimension, and the tile again with a quarter of its chunks missing (read as zeros).  All results are checked
equal first.  The arms are then alternated --reps times in the same process, each call host-timed up to a device
synchronise, after --warmup untimed calls of each; medians and ranges are printed as one JSON line per (grid,
selection), after a line with the GPU's name and power limit read in the same run, and followed by the CUDA-event
kernel times of one grid call.
    python scripts/bench_grid_getslice.py [--reps R] [--warmup W]"""
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
GRIDS = (("2d_1024", (16384, 16384), (1024, 1024)), ("3d_64", (512, 512, 512), (64, 64, 64)))


def selections(shape, cs):
    """(name, start, stop, step, missing): missing drops every 4th touched chunk of the tile"""
    nd = len(shape)
    tile = ([c // 2 + 3 for c in cs], [c // 2 + 3 + 4 * c + 1 for c in cs])          # unaligned, 5 chunks a side
    band = ([0] * nd, list(shape[:-1]) + [shape[-1]])
    band[0][-1], band[1][-1] = cs[-1] - 5, cs[-1] + 5                              # 10 columns, across a chunk edge
    return (("tile", tile[0], tile[1], [1] * nd, False),
            ("band_10", band[0], band[1], [1] * nd, False),
            ("step_8", [0] * nd, list(shape), [8] * nd, False),
            ("tile_quarter_missing", tile[0], tile[1], [1] * nd, True))


def touched(shape, cs, start, stop, step):
    """grid C-order indices of the chunks holding a selected item, and the grid's extents"""
    grid = [-(-s // c) for s, c in zip(shape, cs)]
    per = [sorted({x // c for x in range(a, b, t)}) for a, b, t, c in zip(start, stop, step, cs)]
    out = []
    for coords in itertools.product(*per):
        gi = 0
        for k, c in enumerate(coords):
            gi = gi * grid[k] + c
        out.append((gi, coords))
    return out, grid


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_grid_getslice.py measures on a GPU"
    pkg = g.load_package()
    default_workers = os.environ.get("BLOSC_B200_FRAME_WORKERS")
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit(),
                      "workload": "float32 grids, lz4-shuffle-ts4-cl5 chunks in device memory", "reps": args.reps,
                      "warmup": args.warmup}), flush=True)
    for gname, shape, cs in GRIDS:
        nitems = 1
        for s in shape:
            nitems *= s
        src = bench_words_dev(nitems * TS).view(torch.float32).view(*shape)
        cbytes = TS
        for c in cs:
            cbytes *= c
        ngrid = [s // c for s, c in zip(shape, cs)]                 # the shapes are multiples of the chunk shapes
        chunks = []
        for coords in itertools.product(*(range(n) for n in ngrid)):
            part = src[tuple(slice(c * k, (c + 1) * k) for c, k in zip(coords, cs))].contiguous().view(torch.uint8)
            d = torch.empty(cbytes + 16, dtype=torch.uint8, device="cuda")
            cb = pkg.compress_ctx(5, 1, TS, cbytes, part.view(-1), d, cbytes + 16, "lz4")
            assert cb > 0
            chunks.append(d[:cb].clone())
        stage = torch.empty(cbytes, dtype=torch.uint8, device="cuda")
        for name, start, stop, step, drop in selections(shape, cs):
            tl, grid = touched(shape, cs, start, stop, step)
            table = list(chunks)
            if drop:
                for gi, _ in tl[::4]:
                    table[gi] = None
            sl = tuple(slice(a, b, t) for a, b, t in zip(start, stop, step))
            ref = src.clone()
            for gi, coords in tl:
                if table[gi] is None:
                    ref[tuple(slice(c * k, (c + 1) * k) for c, k in zip(coords, cs))] = 0
            ref = ref[sl].contiguous().view(torch.uint8).view(-1)
            nout = ref.numel()
            outs = {a: torch.empty(nout, dtype=torch.uint8, device="cuda") for a in ("grid", "loop", "full")}
            oshape = [(b - a - 1) // t + 1 for a, b, t in zip(start, stop, step)]

            def grid_arm(workers, out=None):
                if workers:
                    os.environ["BLOSC_B200_FRAME_WORKERS"] = workers
                elif default_workers is None:
                    os.environ.pop("BLOSC_B200_FRAME_WORKERS", None)
                else:
                    os.environ["BLOSC_B200_FRAME_WORKERS"] = default_workers
                assert pkg.grid_getslice(table, shape, cs, TS, start, stop, outs["grid"] if out is None else out,
                                         step=step) == nout

            def part_of(coords):
                """the chunk-local selection of the chunk at coords, and its place in the output"""
                lst, lsp, osl = [], [], []
                for c, k, a, b, t, s in zip(coords, cs, start, stop, step, shape):
                    org = c * k
                    f = a if a >= org else a + -(-(org - a) // t) * t
                    last = a + ((b - a - 1) // t) * t
                    hi = min(last, org + k - 1)
                    ln = f + (hi - f) // t * t
                    lst.append(f - org), lsp.append(ln - org + 1)
                    o = (f - a) // t
                    osl.append(slice(o, o + (ln - f) // t + 1))
                return lst, lsp, tuple(osl)

            parts = {gi: part_of(coords) for gi, coords in tl}

            def loop_arm():
                out = outs["loop"].view(torch.float32).view(*oshape)
                for gi, coords in tl:
                    lst, lsp, osl = parts[gi]
                    dst = out[osl]
                    if table[gi] is None:
                        dst.zero_()
                        continue
                    tmp = torch.empty(dst.numel() * TS, dtype=torch.uint8, device="cuda")
                    assert pkg.getslice(table[gi], cs, lst, lsp, tmp, step=step) == tmp.numel()
                    dst.copy_(tmp.view(torch.float32).view(dst.shape))

            def full_arm():
                out = outs["full"].view(torch.float32).view(*oshape)
                for gi, coords in tl:
                    lst, lsp, osl = parts[gi]
                    dst = out[osl]
                    if table[gi] is None:
                        dst.zero_()
                        continue
                    assert pkg.decompress_ctx(table[gi], stage, cbytes) == cbytes
                    blk = stage.view(torch.float32).view(*cs)
                    dst.copy_(blk[tuple(slice(a, b, t) for a, b, t in zip(lst, lsp, step))])

            fns = {"grid_w1": lambda: grid_arm("1"), "grid": lambda: grid_arm(None), "loop": loop_arm, "full": full_arm}
            grid_arm("1")
            torch.cuda.synchronize()
            assert torch.equal(outs["grid"], ref), (gname, name, "grid_w1")
            outs["grid"].fill_(0xAA)
            for a in ("grid", "loop", "full"):
                fns[a]()
            torch.cuda.synchronize()
            for a in ("grid", "loop", "full"):
                assert torch.equal(outs[a], ref), (gname, name, a)
            del ref
            for a in fns:
                for _ in range(args.warmup):
                    fns[a]()
            times = {a: [] for a in fns}
            for _ in range(args.reps):
                for a in fns:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fns[a]()
                    torch.cuda.synchronize()
                    times[a].append((time.perf_counter() - t0) * 1e3)
            line = {"grid": gname, "shape": shape, "chunkshape": cs, "sel": name, "start": start, "stop": stop,
                    "step": step, "touched": len(tl), "missing": sum(table[gi] is None for gi, _ in tl),
                    "out_bytes": nout}
            for a in fns:
                line[a + "_ms"] = round(statistics.median(times[a]), 4)
                line[a + "_range_ms"] = [round(min(times[a]), 4), round(max(times[a]), 4)]
            print(json.dumps(line), flush=True)
            pkg.set_profiling(True); pkg.prof_reset()
            fns["grid"]()
            torch.cuda.synchronize()
            prof = pkg.prof_get(); pkg.set_profiling(False)
            print(json.dumps({"grid": gname, "sel": name, "arm": "grid",
                              "kernels_ms": {n: [round(v[0], 4), v[1]] for n, v in prof.items() if v[1]}}), flush=True)
            del outs
        del src, chunks, stage


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Workload for the AddressSanitizer build of the emulated library (make -C tests/emu asan), for grid_compress:
  LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python scripts/asan_grid_compress.py
Edge-chunk geometries (1-d to 4-d, chunk shapes larger than the shape, chunk shape 1), with the array, the fill pattern,
dest and offsets each in an exactly sized allocation, read as device memory (the pack kernel) and as host memory (the
host gather), with and without skip_fill; every chunk is decompressed back and checked against the padded sub-array."""
import ctypes as C
import itertools
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = C.CDLL(os.path.join(ROOT, "tests", "emu", "_build", "libblosc_b200_emu_asan.so"))
vp, sz, ci, ll = C.c_void_p, C.c_size_t, C.c_int, C.c_longlong
lib.blosc_b200_grid_bound.restype = sz
lib.blosc_b200_grid_bound.argtypes = [ci, vp, vp, sz]
lib.blosc_b200_grid_compress.restype = ll
lib.blosc_b200_grid_compress.argtypes = [ci, ci, sz, C.c_char_p, sz, ci, ci, vp, vp, sz, vp, vp, ci, vp, sz, vp]
lib.blosc_decompress_ctx.restype = ci
lib.blosc_decompress_ctx.argtypes = [vp, vp, sz, ci]
lib.emu_set_all_device.argtypes = [ci]
lib.blosc_set_splitmode.argtypes = [ci]
lib.blosc_set_splitmode(2)

rng = np.random.default_rng(7)
cases = 0
for shape, chunkshape in (((37,), (8,)), ((13, 11), (4, 5)), ((5, 9), (8, 1)), ((7, 6, 5), (3, 8, 2)),
                          ((3, 5, 4, 6), (2, 2, 3, 4)), ((2, 3), (5, 5))):
    for itemsize in (1, 4, 12):
        grid = [-(-s // c) for s, c in zip(shape, chunkshape)]
        nchunks = int(np.prod(grid))
        n = int(np.prod(shape)) * itemsize
        src = (np.arange(n) // 5 % 7).astype(np.uint8)           # exactly n bytes: a read past the array shows
        src[: n // 4] = 0
        fill = rng.integers(0, 256, itemsize, dtype=np.uint8)
        sh, cs = np.array(shape, np.int64), np.array(chunkshape, np.int64)
        bound = int(lib.blosc_b200_grid_bound(len(shape), sh.ctypes.data, cs.ctypes.data, itemsize))
        cb = int(np.prod(chunkshape)) * itemsize
        for dev, skip, f, comp in itertools.product((0, 1), (0, 1), (None, fill), (b"lz4", b"blosclz")):
            dest = np.full(bound, 0xAA, np.uint8)
            off = np.zeros(nchunks + 1, np.int64)
            lib.emu_set_all_device(dev)
            r = lib.blosc_b200_grid_compress(5, 1, itemsize, comp, 0, 1, len(shape), sh.ctypes.data, cs.ctypes.data,
                                             itemsize, src.ctypes.data, None if f is None else f.ctypes.data, skip,
                                             dest.ctypes.data, bound, off.ctypes.data)
            lib.emu_set_all_device(0)
            assert r > 0 and r == off[-1], (shape, chunkshape, itemsize, r)
            pat = np.zeros(itemsize, np.uint8) if f is None else f
            arr = src.reshape(*shape, itemsize)
            for i, g in enumerate(itertools.product(*(range(k) for k in grid))):
                want = np.empty(tuple(chunkshape) + (itemsize,), np.uint8)
                want[...] = pat
                sl = tuple(slice(c * k, min((c + 1) * k, s)) for c, k, s in zip(g, chunkshape, shape))
                part = arr[sl]
                want[tuple(slice(0, e) for e in part.shape[:-1])] = part
                if off[i + 1] == off[i]:
                    assert skip and (part.reshape(-1, itemsize) == pat).all(), (shape, g)
                    continue
                chunk = dest[off[i]:off[i + 1]].copy()
                out = np.zeros(cb, np.uint8)
                assert lib.blosc_decompress_ctx(chunk.ctypes.data, out.ctypes.data, cb, 1) == cb
                assert (out == want.reshape(-1)).all(), (shape, chunkshape, itemsize, g)
            cases += 1
print(f"grid_compress asan ok: {cases} cases")

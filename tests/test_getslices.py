"""blosc_b200_getslices / blosc_b200_frame_getslices: a batch of equal-sized boxes of an N-d C-order array, box i at
its own corner, written as the stack of the boxes.

Every result is checked against np.stack (or torch.stack) of numpy (torch) slices of the source, and for small
batches also against one blosc_b200_getslice call per box.  CPU: the product's host code and kernels inside the SIMT
emulator (tests/emu/getslice_stage.cpp, which counts every launch and shows the decode launch's listed blocks).  GPU:
the CUDA library through the C ABI with torch tensors."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from datagen import bench_words, ci, compress, gen, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ll = C.c_longlong
CODECS = (("blosclz", None), ("lz4", None), ("lz4hc", None), ("zstd", "BLOSC_B200_ZSTD"),
          ("zlib", "BLOSC_B200_ZLIB"), ("snappy", "BLOSC_B200_SNAPPY"))
TYPESIZES = (1, 2, 3, 4, 8, 16)
NITEMS = 5040                                                   # 2^4 * 3^2 * 5 * 7
NEVER_SPLIT, FORWARD_COMPAT_SPLIT = 2, 4
SHAPES = {1: (5040,), 2: (72, 70), 3: (14, 18, 20), 4: (7, 8, 9, 10), 8: (2, 3, 2, 2, 5, 3, 7, 2)}
PLAN_TILE = 2048


def _bind(lib):
    vp = C.c_void_p
    lib.blosc_b200_getslices.restype = ll
    lib.blosc_b200_getslices.argtypes = [vp, ci, vp, vp, ll, vp, vp]
    lib.blosc_b200_frame_getslices.restype = ll
    lib.blosc_b200_frame_getslices.argtypes = [vp, sz, ci, vp, vp, ll, vp, vp]
    lib.blosc_b200_getslice.restype = ll
    lib.blosc_b200_getslice.argtypes = [vp, ci, vp, vp, vp, vp]
    lib.blosc_b200_frame_compress.restype = ll
    lib.blosc_b200_frame_compress.argtypes = [ci, ci, sz, sz, vp, vp, sz, C.c_char_p, sz, sz, ci]
    lib.blosc_b200_frame_bound.restype = sz
    lib.blosc_b200_frame_bound.argtypes = [sz, sz, sz]
    lib.blosc_b200_frame_chunk.restype = ll
    lib.blosc_b200_frame_chunk.argtypes = [vp, sz, sz, C.POINTER(sz)]
    lib.blosc_getitem.restype = ci
    lib.blosc_compress_ctx.restype = ci
    return lib


@pytest.fixture(scope="session")
def slib(tmp_path_factory):
    """the emulated library with the launch counters of tests/emu/getslice_stage.cpp, built into a temporary
    directory; small forced blocks, never split, so that a chunk has many blocks"""
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("getslices_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "c-blosc_b200", "csrc", "blosc_b200.c"), "-o",
                    str(d / "host.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "getslice_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    path = str(d / "libgetslices_stage.so")
    subprocess.run(["g++", "-shared", "-o", path, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    lib = _bind(C.CDLL(path))
    lib.emu_last_decode_blocks.restype = ci
    lib.emu_all_launches.restype = ll
    lib.emu_set_device_ptrs.argtypes = [C.c_void_p, C.c_void_p]
    lib.blosc_set_splitmode.argtypes = [ci]
    lib.blosc_set_splitmode(NEVER_SPLIT)
    return lib


# ---------------------------------------------------------------------------------------------------------------
# expected results, from the geometry alone
# ---------------------------------------------------------------------------------------------------------------
def _want(src, ts, shape, extent, starts):
    a = src.reshape(*shape, ts)
    if len(starts) == 0:
        return np.zeros(0, np.uint8)
    return np.stack([a[tuple(slice(s, s + e) for s, e in zip(c, extent))] for c in starts]).reshape(-1)


def _touched(shape, extent, starts, ts, bs):
    """the blocks of a chunk that hold a byte of some box"""
    blocks = set()
    for c in starts:
        idx = np.indices(extent).reshape(len(extent), -1) + np.asarray(c).reshape(-1, 1)
        flat = np.ravel_multi_index(tuple(idx), shape)
        blocks.update(((flat * ts) // bs).tolist())
        blocks.update(((flat * ts + ts - 1) // bs).tolist())
    return len(blocks)


def _arr(v):
    return np.ascontiguousarray(v, dtype=np.int64)


def _corners(shape, extent, rng, k):
    """k seeded corners of boxes of `extent`"""
    return np.stack([rng.integers(0, s - e + 1, k) for s, e in zip(shape, extent)], axis=1).astype(np.int64) if k else \
        np.zeros((0, len(shape)), np.int64)


def _extent(shape, rng):
    """a seeded extent, none empty; a third of the dimensions whole, so that they merge"""
    return [s if rng.integers(0, 3) == 0 else int(rng.integers(1, s + 1)) for s in shape]


def _getslices(lib, src_p, shape, extent, starts, dest_p):
    sh, ex, st = _arr(shape), _arr(extent), _arr(starts)
    return lib.blosc_b200_getslices(src_p, len(shape), sh.ctypes.data, ex.ctypes.data, len(starts), st.ctypes.data,
                                    dest_p)


def _check(lib, chunk, src, ts, shape, extent, starts, loop=True):
    want = _want(src, ts, shape, extent, starts)
    out = np.full(want.size + 16, 0xAA, np.uint8)
    st = _arr(starts)
    sh, ex = _arr(shape), _arr(extent)
    r = lib.blosc_b200_getslices(ptr(chunk), len(shape), sh.ctypes.data, ex.ctypes.data, len(st), st.ctypes.data,
                                 ptr(out))
    assert r == want.size, (shape, extent, r, want.size)
    assert (out[:r] == want).all() and (out[r:] == 0xAA).all(), (shape, extent)
    if loop and len(st) <= 8:                                      # the same bytes as one getslice call per box
        b = want.size // max(len(st), 1)
        for i, c in enumerate(st):
            one = np.full(b, 0xAA, np.uint8)
            stop = _arr(c + ex)
            assert lib.blosc_b200_getslice(ptr(chunk), len(shape), sh.ctypes.data, _arr(c).ctypes.data,
                                           stop.ctypes.data, ptr(one)) == b
            assert (one == out[i * b:(i + 1) * b]).all()
    return r


def _compress(lib, comp, clevel, shuf, ts, src, bs, monkeypatch=None, switch=None):
    if switch:
        monkeypatch.setenv(switch, "1")
    r, c = compress(lib, "blosc_compress_ctx", clevel, shuf, ts, src, len(src) + 16, comp, bs)
    assert r > 0, (comp, ts, shuf, r)
    return c[:r].copy()


# ---------------------------------------------------------------------------------------------------------------
# CPU: the emulator
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("comp,switch", CODECS)
@pytest.mark.parametrize("shuf", [0, 1, 2])
def test_getslices_matrix_emu(slib, monkeypatch, comp, switch, shuf):
    """every codec, filter, typesize and ndim, split and unsplit blocks: seeded batches against np.stack and against
    getslice per box"""
    for ts, split in [(ts, NEVER_SPLIT) for ts in TYPESIZES] + [(16, FORWARD_COMPAT_SPLIT), (4, FORWARD_COMPAT_SPLIT)]:
        src = gen("mixed" if ts % 2 else "i32", NITEMS * ts, seed=ts)
        slib.blosc_set_splitmode(split)
        try:
            chunk = _compress(slib, comp, 5, shuf, ts, src, 1024, monkeypatch, switch)
        finally:
            slib.blosc_set_splitmode(NEVER_SPLIT)
        for ndim, shape in SHAPES.items():
            rng = np.random.default_rng(100 * ts + ndim + shuf)
            extent = _extent(shape, rng)
            _check(slib, chunk, src, ts, shape, extent, _corners(shape, extent, rng, 3))


def test_getslices_layouts_emu(slib):
    """overlapping and repeated boxes, boxes on block edges and in the short last block, whole dimensions that merge,
    one box equal to the whole array; on a compressed and a memcpyed chunk, typesizes 4 and 3"""
    for ts in (4, 3):
        src = gen("i32" if ts == 4 else "mixed", NITEMS * ts, seed=ts)
        for clevel in (5, 0):
            chunk = _compress(slib, "lz4", clevel, 1, ts, src, 1024)
            bs = int(chunk[8:12].view(np.int32)[0])
            assert bool(chunk[2] & 0x2) == (clevel == 0) and (NITEMS * ts) % bs
            shape = (72, 70)
            row = bs // ts // 70 + 1                                # a row that holds a block edge
            for extent, starts in (([3, 5], [[2, 2], [3, 4], [2, 2], [2, 2], [69, 65], [0, 0]]),   # overlap, repeat
                                   ([2, 70], [[row - 1, 0], [row, 0], [70, 0], [0, 0]]),         # rows merge
                                   ([1, 3], [[row, 0], [row - 1, 67], [71, 67], [71, 0]]),       # edges, short block
                                   ([72, 70], [[0, 0], [0, 0]]),                                  # the whole array
                                   ([72, 1], [[0, 69], [0, 0], [0, 35]])):                        # columns
                _check(slib, chunk, src, ts, shape, extent, starts)
            for extent, starts in (([2, 8, 9, 10], [[1, 0, 0, 0], [5, 0, 0, 0]]), ([1, 2, 9, 10], [[6, 6, 0, 0], [0, 0, 0, 0]]),
                                   ([7, 8, 9, 10], [[0, 0, 0, 0]]), ([1, 1, 1, 10], [[6, 7, 8, 0], [0, 0, 0, 0]])):
                _check(slib, chunk, src, ts, (7, 8, 9, 10), extent, starts)


@pytest.mark.parametrize("k", [1, 2, PLAN_TILE - 1, PLAN_TILE, PLAN_TILE + 1])
def test_getslices_batch_sizes_emu(slib, k):
    """batches around the scan tile"""
    ts, shape = 4, (14, 18, 20)
    src = gen("i32", NITEMS * ts, seed=11)
    chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
    rng = np.random.default_rng(k)
    for extent in ([2, 3, 4], [1, 18, 20]):
        _check(slib, chunk, src, ts, shape, extent, _corners(shape, extent, rng, k))


@pytest.mark.parametrize("clevel", [5, 0])
@pytest.mark.parametrize("src_dev,dest_dev,starts_dev", [(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)])
def test_getslices_placements_emu(slib, clevel, src_dev, dest_dev, starts_dev):
    """src, dest and the corners in host and device memory (a memcpyed device chunk is read in place, with no touch)"""
    ts, shape, extent = 4, (14, 18, 20), [3, 18, 7]
    src = gen("i32", NITEMS * ts, seed=7)
    chunk = _compress(slib, "lz4", clevel, 1, ts, src, 1024)
    starts = _corners(shape, extent, np.random.default_rng(clevel + 2 * src_dev + 4 * dest_dev + 8 * starts_dev), 5)
    want = _want(src, ts, shape, extent, starts)
    out = np.full(want.size + 16, 0xAA, np.uint8)
    marked = [p for p, on in ((chunk.ctypes.data, src_dev), (out.ctypes.data, dest_dev), (starts.ctypes.data, starts_dev))
              if on]
    if len(marked) == 3:
        slib.emu_set_all_device(1)
    else:
        slib.emu_set_device_ptrs(*(marked + [None, None])[:2])
    try:
        before = slib.emu_all_launches()
        r = _getslices(slib, ptr(chunk), shape, extent, starts, out.ctypes.data)
        launches = slib.emu_all_launches() - before
    finally:
        slib.emu_set_device_ptrs(None, None)
        slib.emu_set_all_device(0)
    assert r == want.size and (out[:r] == want).all() and (out[r:] == 0xAA).all()
    # check, touch, slot scan, decode, unfilter, gather; a memcpyed chunk: no decode; in place: no touch either
    assert launches == (6 if clevel else 2 if src_dev else 4), launches


def test_getslices_launches_emu(slib):
    """one box and 4096 boxes of one chunk make the same launches"""
    src = bench_words(80000)
    chunk = _compress(slib, "lz4", 5, 1, 4, src, 4096)
    assert not chunk[2] & 0x2
    shape, extent = (100, 200), [4, 7]
    counts = []
    for k in (1, 4096):
        before = slib.emu_all_launches()
        _check(slib, chunk, src, 4, shape, extent, _corners(shape, extent, np.random.default_rng(k), k), loop=False)
        counts.append(slib.emu_all_launches() - before)
    assert counts == [6, 6], counts                               # check, touch, slot scan, decode, unfilter, gather


def test_getslices_decodes_touched_blocks_emu(slib):
    """the decode launch lists exactly the union of the blocks the boxes touch, each once"""
    for ts, shape in ((4, (72, 70)), (3, (7, 8, 9, 10)), (16, (14, 18, 20))):
        src = gen("mixed" if ts == 3 else "i32", NITEMS * ts, seed=ts)
        chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
        bs = int(chunk[8:12].view(np.int32)[0])
        assert not chunk[2] & 0x2
        rng = np.random.default_rng(ts)
        for _ in range(4):
            extent = _extent(shape, rng)
            starts = _corners(shape, extent, rng, int(rng.integers(1, 6)))
            _check(slib, chunk, src, ts, shape, extent, starts, loop=False)
            assert slib.emu_last_decode_blocks() == _touched(shape, extent, starts, ts, bs), (extent, starts)


def test_getslices_rejects_emu(slib, capfd):
    """every host-side geometry error, and a bad corner first, in the middle and last: -1, one message, dest untouched,
    nothing decoded; an empty batch or an empty extent returns 0 with nothing launched and the corners never read"""
    ts = 4
    src = gen("i32", NITEMS * ts, seed=2)
    chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
    out = np.full(256, 0xAA, np.uint8)
    good = _arr([[0, 0]])
    capfd.readouterr()
    for shape, extent, k in (((), (), 1), ((1,) * 8 + (5040,), (1,) * 9, 1), ((-72, -70), (1, 1), 1),
                             ((72, 70), (1, -1), 1), ((72, 70), (73, 1), 1), ((72, 71), (1, 1), 1),
                             ((1 << 40, 1 << 40), (1, 1), 1), ((72, 70), (1, 1), -1), ((72, 70), (72, 70), 1 << 50),
                             ((72, 70), (1, 1), 1 << 59)):              # 4-byte boxes whose corners overflow
        before = slib.emu_all_launches()
        sh, ex = (_arr(v) if len(v) else np.zeros(1, np.int64) for v in (shape, extent))
        r = slib.blosc_b200_getslices(ptr(chunk), len(shape), sh.ctypes.data, ex.ctypes.data, k, good.ctypes.data,
                                      ptr(out))
        assert r == -1 and (out == 0xAA).all() and slib.emu_all_launches() == before, (shape, extent, k, r)
        assert "blosc_b200" in capfd.readouterr().err, (shape, extent, k)
    for extent, k in (((2, 3), 0), ((0, 3), 5)):
        before = slib.emu_all_launches()
        sh, ex = _arr((72, 70)), _arr(extent)
        assert slib.blosc_b200_getslices(ptr(chunk), 2, sh.ctypes.data, ex.ctypes.data, k, None, ptr(out)) == 0
        assert slib.emu_all_launches() == before and (out == 0xAA).all()
    shape, extent = (72, 70), (3, 5)
    for bad_at in (0, 1000, 2047):
        for dim, v in ((0, -1), (1, 66), (0, 70), (1, -(1 << 62))):
            starts = _corners(shape, extent, np.random.default_rng(bad_at), 2048)
            starts[bad_at, dim] = v
            starts[bad_at + 1:, 1 - dim] = -5                       # later boxes fail too: the first one is named
            dest = np.full(2048 * 60 + 16, 0xAA, np.uint8)
            before = slib.emu_all_launches()
            r = _getslices(slib, ptr(chunk), shape, extent, starts, dest.ctypes.data)
            err = capfd.readouterr().err
            assert r == -1 and (dest == 0xAA).all(), (bad_at, dim, r)
            assert slib.emu_all_launches() - before == 3                # check, touch, slot scan: no decode, no gather
            assert err.count("blosc_b200") == 1 and f"box {bad_at} " in err and f"dimension {dim}" in err, err
    for patch, code in ((lambda h: h.__setitem__(0, 3), -9), (lambda h: h.__setitem__(2, (h[2] & 0x1f) | (6 << 5)), -5),
                        (lambda h: h[8:12].view(np.int32).__setitem__(0, 0), -1)):
        h = chunk.copy()
        patch(h)
        assert _getslices(slib, ptr(h), shape, extent, [[0, 0], [1, 1]], out.ctypes.data) == code and (out == 0xAA).all()


def test_getslices_damaged_block_emu(slib):
    """a damaged block that no box touches is not read; one that a box touches gives blosc_d's code, dest untouched"""
    ts, shape = 4, (72, 70)
    src = gen("i32", NITEMS * ts, seed=3)
    chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
    bs = int(chunk[8:12].view(np.int32)[0])
    h = chunk.copy()
    h[16 + 4 * 5:16 + 4 * 6].view(np.int32)[0] = 0x7fff0000      # block 5's bstarts entry
    r5 = 5 * bs // ts // 70                                        # a row with an item of block 5
    for src_dev in (0, 1):
        slib.emu_set_device_ptrs(h.ctypes.data if src_dev else None, None)
        try:
            code = slib.blosc_getitem(ptr(h), ci(5 * bs // ts), ci(1), ptr(np.zeros(64, np.uint8)))
            assert code < 0
            _check(slib, h, src, ts, shape, [2, 70], [[0, 0], [r5 - 3, 0], [r5 + 6, 0]], loop=False)
            out = np.full(3 * 2 * 70 * ts, 0xAA, np.uint8)
            assert _getslices(slib, ptr(h), shape, [2, 70], [[0, 0], [r5, 0], [60, 0]], out.ctypes.data) == code
            assert (out == 0xAA).all()
        finally:
            slib.emu_set_device_ptrs(None, None)


def _frame(lib, src, ts, chunksize, clevel=5):
    fb = lib.blosc_b200_frame_bound(len(src), ts, chunksize)
    frame = np.zeros(fb, np.uint8)
    r = lib.blosc_b200_frame_compress(clevel, 1, ts, len(src), ptr(src), ptr(frame), fb, b"lz4", 1024, chunksize, 1)
    assert r > 0
    return frame[:r].copy()


def _frame_getslices(lib, frame_p, fb, shape, extent, starts, dest_p):
    sh, ex, st = _arr(shape), _arr(extent), _arr(starts)
    return lib.blosc_b200_frame_getslices(frame_p, fb, len(shape), sh.ctypes.data, ex.ctypes.data, len(starts),
                                          st.ctypes.data, dest_p)


def _check_frame(lib, frame, src, ts, shape, extent, starts):
    want = _want(src, ts, shape, extent, starts)
    out = np.full(want.size + 16, 0xAA, np.uint8)
    r = _frame_getslices(lib, frame.ctypes.data, len(frame), shape, extent, starts, out.ctypes.data)
    assert r == want.size and (out[:r] == want).all() and (out[r:] == 0xAA).all(), (shape, extent, r)


@pytest.mark.parametrize("frame_dev,dest_dev,starts_dev", [(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)])
def test_frame_getslices_emu(slib, frame_dev, dest_dev, starts_dev):
    """boxes inside one chunk and across chunk edges, a chunksize that is no multiple of the row, a short last chunk;
    frame, dest and corners in host and device memory"""
    ts, shape = 4, (50, 37)
    src = gen("i32", 50 * 37 * ts, seed=5)
    frame = _frame(slib, src, ts, 1000)                           # 250 items a chunk, 8 chunks, the last of 100
    rng = np.random.default_rng(frame_dev + 2 * dest_dev + 4 * starts_dev)
    cases = [([2, 5], [[0, 0], [1, 20], [7, 30], [48, 32]]),      # inside one chunk each
             ([3, 37], [[5, 0], [12, 0], [47, 0], [5, 0]]),       # across edges, repeated
             ([50, 1], [[0, 36], [0, 0]]), ([50, 37], [[0, 0]]), ([1, 1], [[6, 28], [49, 36]])]
    for _ in range(3):
        extent = _extent(shape, rng)
        cases.append((extent, _corners(shape, extent, rng, 4)))
    for extent, starts in cases:
        starts = _arr(starts)
        want = _want(src, ts, shape, extent, starts)
        out = np.full(want.size + 16, 0xAA, np.uint8)
        marked = [p for p, on in ((frame.ctypes.data, frame_dev), (out.ctypes.data, dest_dev),
                                  (starts.ctypes.data, starts_dev)) if on]
        if len(marked) == 3:
            slib.emu_set_all_device(1)
        else:
            slib.emu_set_device_ptrs(*(marked + [None, None])[:2])
        try:
            r = _frame_getslices(slib, frame.ctypes.data, len(frame), shape, extent, starts, out.ctypes.data)
        finally:
            slib.emu_set_device_ptrs(None, None)
            slib.emu_set_all_device(0)
        assert r == want.size and (out[:r] == want).all() and (out[r:] == 0xAA).all(), (extent, starts, r)


def test_frame_getslices_edges_emu(slib, capfd):
    """damaged touched and untouched chunks, a chunk whose typesize differs from chunk 0's, a bad corner, an empty
    frame"""
    fb = slib.blosc_b200_frame_bound(0, 4, 1000)
    buf = np.zeros(fb, np.uint8)
    n = slib.blosc_b200_frame_compress(5, 1, 4, 0, ptr(buf), ptr(buf), fb, b"lz4", 0, 1000, 1)
    assert n > 0
    empty = buf[:n].copy()
    out = np.full(64, 0xAA, np.uint8)
    assert _frame_getslices(slib, empty.ctypes.data, len(empty), (0,), (0,), [[0]], out.ctypes.data) == 0
    assert _frame_getslices(slib, empty.ctypes.data, len(empty), (4,), (1,), [[0]], out.ctypes.data) == -1
    assert (out == 0xAA).all()

    ts, shape = 4, (50, 37)
    src = gen("i32", 50 * 37 * ts, seed=6)
    frame = _frame(slib, src, ts, 1000)
    off = [slib.blosc_b200_frame_chunk(frame.ctypes.data, len(frame), i, None) for i in range(8)]
    for patch, code in ((lambda f: f.__setitem__(off[2] + 3, 2), -1), (lambda f: f.__setitem__(off[2], 3), -9),
                        (lambda f: f[off[2] + 16:off[2] + 20].view(np.int32).__setitem__(0, 0x7fff0000), None)):
        f = frame.copy()
        patch(f)
        for dev in (0, 1):
            slib.emu_set_all_device(dev)
            try:
                out = np.full(3 * 10 * 37 * ts + 16, 0xAA, np.uint8)
                capfd.readouterr()
                r = _frame_getslices(slib, f.ctypes.data, len(f), shape, (10, 37), [[0, 0], [10, 0], [40, 0]],
                                     out.ctypes.data)                 # box 1 holds items of chunk 2
                assert r < 0 and (code is None or r == code) and (dev or (out == 0xAA).all()), (code, r)
                if code == -1:
                    assert "blosc_b200" in capfd.readouterr().err
                _check_frame(slib, f, src, ts, shape, [6, 37], [[0, 0], [21, 0], [44, 0]])   # chunks 0, 1, 3 to 7
            finally:
                slib.emu_set_all_device(0)
    out = np.full(3 * 60 + 16, 0xAA, np.uint8)
    capfd.readouterr()
    assert _frame_getslices(slib, frame.ctypes.data, len(frame), shape, (3, 5), [[0, 0], [47, 32], [48, 0]],
                            out.ctypes.data) == -1
    err = capfd.readouterr().err
    assert (out == 0xAA).all() and err.count("blosc_b200") == 1 and "box 2 " in err


# ---------------------------------------------------------------------------------------------------------------
# GPU: the CUDA library
# ---------------------------------------------------------------------------------------------------------------
def _torch_want(torch, d_src, dtype, shape, extent, starts):
    a = d_src.view(dtype).view(*shape)
    return torch.stack([a[tuple(slice(s, s + e) for s, e in zip(c, extent))] for c in starts.tolist()]).reshape(-1)


def _big_chunk(torch, pkg, nbytes):
    src = bench_words(nbytes)
    d_src = torch.from_numpy(src).cuda()
    d_chunk = torch.zeros(nbytes + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(5, 1, 4, nbytes, d_src, d_chunk, nbytes + 16, "lz4")
    assert cb > 0
    return d_src, d_chunk[:cb]


@pytest.mark.gpu
def test_getslices_big_chunk_gpu(pkg, cuda):
    """a 256 MiB LZ4 + shuffle chunk read as (256, 512, 512) int32: torch.randint corners on the device against
    torch.stack of torch slices; host corners give the same bytes"""
    torch = cuda
    d_src, d_chunk = _big_chunk(torch, pkg, 256 << 20)
    shape = (256, 512, 512)
    g = torch.Generator(device="cuda").manual_seed(5)
    for extent, k in (([64, 64, 64], 256), ([1, 512, 512], 16), ([7, 3, 200], 4096), ([256, 512, 512], 1)):
        starts = torch.stack([torch.randint(0, s - e + 1, (k,), device="cuda", generator=g)
                              for s, e in zip(shape, extent)], dim=1)
        want = _torch_want(torch, d_src, torch.int32, shape, extent, starts).view(torch.uint8)
        out = torch.full((want.numel() + 16,), 0xAA, dtype=torch.uint8, device="cuda")
        assert pkg.getslices(d_chunk, shape, extent, starts, out) == want.numel()
        assert torch.equal(out[:want.numel()], want) and bool((out[want.numel():] == 0xAA).all())
        host = torch.full_like(out, 0x55)
        assert pkg.getslices(d_chunk, shape, extent, starts.cpu().numpy(), host) == want.numel()
        assert torch.equal(host[:want.numel()], want)


@pytest.mark.gpu
@pytest.mark.parametrize("dest_dev", [False, True])
def test_frame_getslices_1gib_gpu(pkg, cuda, dest_dev):
    """a 1 GiB frame of 4 chunks read as (1024, 512, 512) int32: device corners, boxes across chunk edges; host dest
    and host corners"""
    torch = cuda
    n = 1 << 30
    src = bench_words(n)
    d_src = torch.from_numpy(src).cuda()
    fb = pkg.frame_bound(n, 4, 0)
    d_frame = torch.zeros(fb, dtype=torch.uint8, device="cuda")
    fs = pkg.frame_compress(5, 1, 4, n, d_src, d_frame, fb, "lz4")
    assert fs > 0
    shape = (1024, 512, 512)
    g = torch.Generator(device="cuda").manual_seed(7)
    for extent, k in (([64, 64, 64], 64), ([300, 1, 512], 8), ([2, 512, 512], 3)):
        starts = torch.stack([torch.randint(0, s - e + 1, (k,), device="cuda", generator=g)
                              for s, e in zip(shape, extent)], dim=1)
        want = _torch_want(torch, d_src, torch.int32, shape, extent, starts).view(torch.uint8)
        for st in (starts, starts.cpu()):
            out = torch.full((want.numel() + 16,), 0xAA, dtype=torch.uint8, device="cuda" if dest_dev else "cpu")
            assert pkg.frame_getslices(d_frame[:fs], fs, shape, extent, st if st.is_cuda else st.numpy(), out) == \
                want.numel()
            assert torch.equal(out[:want.numel()].cuda(), want) and bool((out[want.numel():] == 0xAA).all())


@pytest.mark.gpu
def test_getslices_emu_and_gpu_agree(pkg, slib, cuda):
    """the emulator and the GPU give byte-identical output on one shared case"""
    torch = cuda
    ts, shape, extent = 4, (14, 18, 20), [3, 18, 7]
    src = gen("i32", NITEMS * ts, seed=7)
    chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
    starts = _corners(shape, extent, np.random.default_rng(1), 9)
    want = _want(src, ts, shape, extent, starts)
    emu_out = np.full(want.size, 0xAA, np.uint8)
    assert _getslices(slib, ptr(chunk), shape, extent, starts, emu_out.ctypes.data) == want.size
    out = torch.full((want.size,), 0xAA, dtype=torch.uint8, device="cuda")
    assert pkg.getslices(torch.from_numpy(chunk).cuda(), shape, extent, torch.from_numpy(starts).cuda(), out) == want.size
    assert (out.cpu().numpy() == emu_out).all() and (emu_out == want).all()


@pytest.mark.gpu
def test_getslices_launches_gpu(pkg, cuda):
    """the launches of a batch do not grow with the number of boxes, by the profiler's count per kind"""
    torch = cuda
    src = bench_words(8 << 20)
    d_chunk = torch.from_numpy(_compress(pkg.lib, "lz4", 5, 1, 4, src, 0)).cuda()
    shape, extent = (1 << 16, 32), [10, 5]
    counts = []
    pkg.set_profiling(True)
    try:
        for k in (1, 16, 4096):
            starts = _corners(shape, extent, np.random.default_rng(k), k)
            want = _want(src, 4, shape, extent, starts)
            out = torch.zeros(want.size, dtype=torch.uint8, device="cuda")
            pkg.prof_reset()
            before = pkg.launch_count()
            assert pkg.getslices(d_chunk, shape, extent, torch.from_numpy(starts).cuda(), out) == want.size
            kinds = {kd: n for kd, (_, n) in pkg.prof_get().items() if n}
            counts.append((pkg.launch_count() - before, kinds))
            assert (out.cpu().numpy() == want).all()
    finally:
        pkg.set_profiling(False)
    assert counts[0] == counts[1] == counts[2], counts
    assert counts[0][1]["plan"] == 3 and counts[0][1]["gather"] == 1, counts   # check, touch, slot scan; one gather


@pytest.mark.gpu
def test_getslices_corners_on_another_device_gpu(pkg, cuda):
    torch = cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    src = bench_words(1 << 20)
    d_chunk = torch.from_numpy(_compress(pkg.lib, "lz4", 5, 1, 4, src, 0)).to("cuda:0")
    out = torch.full((64 * 4 * 2,), 0xAA, dtype=torch.uint8, device="cuda:0")
    starts = torch.tensor([[0, 0], [5, 3]], dtype=torch.int64, device="cuda:1")
    assert pkg.getslices(d_chunk, (1024, 256), (8, 8), starts, out) == -1
    assert bool((out == 0xAA).all())


@pytest.mark.gpu
def test_getslices_arguments_gpu(pkg, cuda):
    """corners as a CUDA tensor of another dtype raise TypeError, the wrong second dimension ValueError"""
    torch = cuda
    for call in (lambda st: pkg.getslices(np.zeros(32, np.uint8), (4, 4), (2, 2), st, np.zeros(64, np.uint8)),
                 lambda st: pkg.frame_getslices(np.zeros(32, np.uint8), 32, (4, 4), (2, 2), st, np.zeros(64, np.uint8))):
        with pytest.raises(ValueError):
            call(np.zeros((3, 3), np.int64))
        with pytest.raises(ValueError):
            call(torch.zeros((3, 1), dtype=torch.int64, device="cuda"))
    src = np.arange(16, dtype=np.uint8)
    chunk = np.zeros(64, np.uint8)
    cb = pkg.compress_ctx(5, 1, 1, 16, src, chunk, 64, "lz4")
    assert cb > 0
    for st in ([], np.zeros((0, 2), np.int64)):                         # no boxes: 0, nothing written
        out = np.full(8, 0xAA, np.uint8)
        assert pkg.getslices(chunk[:cb], (4, 4), (2, 2), st, out) == 0 and (out == 0xAA).all()
    with pytest.raises(TypeError):
        pkg.getslices(torch.zeros(64, dtype=torch.uint8, device="cuda"), (4, 4), (2, 2),
                      torch.zeros((3, 2), dtype=torch.int32, device="cuda"), torch.zeros(64, dtype=torch.uint8,
                                                                                         device="cuda"))


@pytest.mark.gpu
def test_getslices_two_threads_gpu(pkg, cuda):
    """two host threads reading batches of the same chunk and frame at once"""
    torch = cuda
    ts, shape = 4, (1024, 1536)
    src = bench_words(1024 * 1536 * ts)
    d_chunk = torch.from_numpy(_compress(pkg.lib, "lz4", 5, 1, ts, src, 0)).cuda()
    fb = pkg.frame_bound(len(src), ts, 1 << 20)
    frame = np.zeros(fb, np.uint8)
    fs = pkg.frame_compress(5, 1, ts, len(src), src, frame, fb, "lz4", 0, 1 << 20)
    assert fs > 0
    d_frame = torch.from_numpy(frame[:fs].copy()).cuda()
    errors = []

    def reader(seed):
        try:
            rng = np.random.default_rng(seed)
            for rep in range(6):
                extent = _extent(shape, rng)
                starts = _corners(shape, extent, rng, 20)
                want = _want(src, ts, shape, extent, starts)
                out = torch.full((want.size + 8,), 0xAA, dtype=torch.uint8, device="cuda")
                d_st = torch.from_numpy(starts).cuda()
                r = pkg.getslices(d_chunk, shape, extent, d_st, out) if rep % 2 else \
                    pkg.frame_getslices(d_frame, fs, shape, extent, d_st, out)
                got = out.cpu().numpy()
                if r != want.size or not (got[:r] == want).all() or not (got[r:] == 0xAA).all():
                    errors.append((seed, rep, r, want.size))
        except Exception as e:                                      # noqa: BLE001 -- reported below
            errors.append((seed, repr(e)))

    threads = [threading.Thread(target=reader, args=(s,)) for s in (1, 2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors

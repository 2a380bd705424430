"""blosc_b200_getslice / blosc_b200_frame_getslice: a box of an N-d C-order array, planned and gathered from the box.

Every result is checked against numpy (or torch) slicing of the source array, and, where the number of innermost runs
fits in an int, against blosc_b200_getitems (frame_getitems) over the list of those runs.  CPU: the product's host
code and kernels inside the SIMT emulator (tests/emu/getslice_stage.cpp, which also counts launches and shows the
decode launch's listed blocks).  GPU: the CUDA library through the C ABI with torch tensors."""
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


def _bind(lib):
    lib.blosc_b200_getslice.restype = ll
    lib.blosc_b200_getslice.argtypes = [C.c_void_p, ci, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.blosc_b200_frame_getslice.restype = ll
    lib.blosc_b200_frame_getslice.argtypes = [C.c_void_p, sz, ci, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.blosc_b200_getitems.restype = ll
    lib.blosc_b200_getitems.argtypes = [C.c_void_p, ci, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.blosc_b200_frame_getitems.restype = ll
    lib.blosc_b200_frame_getitems.argtypes = [C.c_void_p, sz, sz, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.blosc_b200_frame_compress.restype = ll
    lib.blosc_b200_frame_compress.argtypes = [ci, ci, sz, sz, C.c_void_p, C.c_void_p, sz, C.c_char_p, sz, sz, ci]
    lib.blosc_b200_frame_bound.restype = sz
    lib.blosc_b200_frame_bound.argtypes = [sz, sz, sz]
    lib.blosc_b200_frame_chunk.restype = ll
    lib.blosc_b200_frame_chunk.argtypes = [C.c_void_p, sz, sz, C.POINTER(sz)]
    lib.blosc_getitem.restype = ci
    lib.blosc_compress_ctx.restype = ci
    return lib


@pytest.fixture(scope="session")
def slib(tmp_path_factory):
    """the emulated library with the launch counters of tests/emu/getslice_stage.cpp, built into a temporary
    directory"""
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("getslice_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "c-blosc_b200", "csrc", "blosc_b200.c"), "-o",
                    str(d / "host.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "getslice_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    path = str(d / "libgetslice_stage.so")
    subprocess.run(["g++", "-shared", "-o", path, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    lib = _bind(C.CDLL(path))
    lib.emu_last_decode_blocks.restype = ci
    lib.emu_all_launches.restype = ll
    lib.emu_set_device_ptrs.argtypes = [C.c_void_p, C.c_void_p]
    lib.blosc_set_splitmode.argtypes = [ci]
    lib.blosc_set_splitmode(NEVER_SPLIT)                          # small forced blocks: many of them per chunk
    return lib


# ---------------------------------------------------------------------------------------------------------------
# expected results, from the geometry alone
# ---------------------------------------------------------------------------------------------------------------
def _want(src, ts, shape, start, stop):
    a = src.reshape(*shape, ts)
    return np.ascontiguousarray(a[tuple(slice(s, e) for s, e in zip(start, stop))]).reshape(-1)


def _runs(shape, start, stop):
    """the box as one range per innermost run (not merged): flat starts and counts"""
    ext = [e - s for s, e in zip(start, stop)]
    if 0 in ext:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    outer = np.indices(ext[:-1]).reshape(len(ext) - 1, -1) if len(ext) > 1 else np.zeros((0, 1), np.int64)
    coords = [outer[k] + start[k] for k in range(len(ext) - 1)] + [np.full(outer.shape[1], start[-1])]
    st = np.ravel_multi_index(coords, shape).astype(np.int64)
    return st, np.full(st.size, ext[-1], np.int64)


def _touched(shape, start, stop, ts, bs, nbytes):
    """blocks of a chunk of nbytes that hold a byte of the box"""
    st, n = _runs(shape, start, stop)
    lo, hi = st * ts, (st + n) * ts - 1
    blocks = set()
    for a, b in zip(lo // bs, hi // bs):
        blocks.update(range(int(a), int(b) + 1))
    assert all(b * bs < nbytes for b in blocks)
    return len(blocks)


def _arr(v):
    return np.ascontiguousarray(v, dtype=np.int64)


def _getslice(lib, src_p, shape, start, stop, dest):
    sh, st, sp = _arr(shape), _arr(start), _arr(stop)
    return lib.blosc_b200_getslice(src_p, len(shape), sh.ctypes.data, st.ctypes.data, sp.ctypes.data, dest.ctypes.data)


def _frame_getslice(lib, frame_p, fb, shape, start, stop, dest_p):
    sh, st, sp = _arr(shape), _arr(start), _arr(stop)
    return lib.blosc_b200_frame_getslice(frame_p, fb, len(shape), sh.ctypes.data, st.ctypes.data, sp.ctypes.data, dest_p)


def _boxes(shape, rng, k):
    """k seeded boxes, none empty; a third of the dimensions whole, so that they merge"""
    out = []
    for _ in range(k):
        start, stop = [], []
        for s in shape:
            if rng.integers(0, 3) == 0:
                a, b = 0, s
            else:
                a = int(rng.integers(0, s))
                b = int(rng.integers(a + 1, s + 1))
            start.append(a)
            stop.append(b)
        out.append((start, stop))
    return out


def _check(lib, chunk, src, ts, shape, start, stop, getitems=True):
    want = _want(src, ts, shape, start, stop)
    out = np.full(want.size + 16, 0xAA, np.uint8)
    r = _getslice(lib, ptr(chunk), shape, start, stop, out)
    assert r == want.size, (shape, start, stop, r, want.size)
    assert (out[:r] == want).all() and (out[r:] == 0xAA).all(), (shape, start, stop)
    if getitems:
        st, nn = _runs(shape, start, stop)
        if 0 < st.size and st.max() < 2 ** 31:
            g = np.full(want.size + 16, 0xAA, np.uint8)
            st32, nn32 = st.astype(np.int32), nn.astype(np.int32)
            assert lib.blosc_b200_getitems(ptr(chunk), st.size, st32.ctypes.data, nn32.ctypes.data, ptr(g)) == want.size
            assert (g == out).all()
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
def test_getslice_matrix_emu(slib, monkeypatch, comp, switch, shuf):
    """every codec, filter, typesize and ndim: seeded boxes against numpy and against getitems over the runs"""
    for i, (ts, split) in enumerate([(ts, NEVER_SPLIT) for ts in TYPESIZES] + [(16, FORWARD_COMPAT_SPLIT)]):
        src = gen("mixed" if ts % 2 else "i32", NITEMS * ts, seed=ts)   # odd typesizes: i32 would not compress
        slib.blosc_set_splitmode(split)                           # blocks of 64 KiB, split into streams
        try:
            chunk = _compress(slib, comp, 5, shuf, ts, src, 1024, monkeypatch, switch)
        finally:
            slib.blosc_set_splitmode(NEVER_SPLIT)
        for ndim, shape in SHAPES.items():
            for start, stop in _boxes(shape, np.random.default_rng(100 * ts + ndim + shuf), 2):
                _check(slib, chunk, src, ts, shape, start, stop)


def test_getslice_special_boxes_emu(slib):
    """the whole array, one item, an empty box, a box inside one block, rows across block edges, whole trailing
    dimensions and the short last block, on a compressed and on a memcpyed chunk, for typesizes 4 and 3"""
    for ts in (4, 3):
        src = gen("i32" if ts == 4 else "mixed", NITEMS * ts, seed=ts)
        for clevel in (5, 0):
            chunk = _compress(slib, "lz4", clevel, 1, ts, src, 1024)
            bs = int(chunk[8:12].view(np.int32)[0])
            assert bool(chunk[2] & 0x2) == (clevel == 0) and (NITEMS * ts) % bs
            shape = (72, 70)
            row = bs // ts // 70 + 1                                # a row that holds a block edge
            for start, stop in (([0, 0], [72, 70]), ([5, 7], [6, 8]), ([0, 1], [1, 3]), ([row, 0], [row + 2, 70]),
                                ([row - 1, 3], [row + 3, 69]), ([71, 69], [72, 70]), ([60, 0], [72, 70]),
                                ([0, 69], [72, 70])):
                _check(slib, chunk, src, ts, shape, start, stop)
            for start, stop in (([1, 0, 0, 0], [3, 8, 9, 10]), ([1, 2, 0, 0], [3, 4, 9, 10]), ([0, 0, 0, 0], [7, 8, 9, 10]),
                                ([6, 7, 8, 0], [7, 8, 9, 10])):
                _check(slib, chunk, src, ts, (7, 8, 9, 10), start, stop)
            out = np.full(64, 0xAA, np.uint8)
            before = slib.emu_all_launches()
            assert _getslice(slib, ptr(chunk), shape, [3, 5], [3, 9], out) == 0
            assert slib.emu_all_launches() == before and (out == 0xAA).all()


@pytest.mark.parametrize("clevel", [5, 0])
@pytest.mark.parametrize("src_dev,dest_dev", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_getslice_placements_emu(slib, clevel, src_dev, dest_dev):
    """src and dest in host and device memory (a memcpyed chunk in device memory is read in place, with no plan)"""
    ts, shape = 4, (14, 18, 20)
    src = gen("i32", NITEMS * ts, seed=7)
    chunk = _compress(slib, "lz4", clevel, 1, ts, src, 1024)
    rng = np.random.default_rng(clevel + 10 * src_dev + 20 * dest_dev)
    for start, stop in _boxes(shape, rng, 4) + [([0, 0, 0], list(shape))]:
        want = _want(src, ts, shape, start, stop)
        out = np.full(want.size + 16, 0xAA, np.uint8)
        slib.emu_set_device_ptrs(chunk.ctypes.data if src_dev else None, out.ctypes.data if dest_dev else None)
        try:
            r = _getslice(slib, ptr(chunk), shape, start, stop, out)
        finally:
            slib.emu_set_device_ptrs(None, None)
        assert r == want.size and (out[:r] == want).all() and (out[r:] == 0xAA).all()


def test_getslice_decodes_touched_blocks_emu(slib):
    """the decode launch lists exactly the blocks that hold a byte of the box"""
    for ts, shape in ((4, (72, 70)), (3, (7, 8, 9, 10)), (16, (14, 18, 20))):
        src = gen("mixed" if ts == 3 else "i32", NITEMS * ts, seed=ts)
        chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
        bs = int(chunk[8:12].view(np.int32)[0])
        assert not chunk[2] & 0x2
        for start, stop in _boxes(shape, np.random.default_rng(ts), 6):
            _check(slib, chunk, src, ts, shape, start, stop, getitems=False)
            assert slib.emu_last_decode_blocks() == _touched(shape, start, stop, ts, bs, NITEMS * ts), (start, stop)


def test_getslice_damaged_block_emu(slib):
    """a damaged block that the box does not touch is not read; one it touches gives blosc_d's code, dest untouched"""
    ts, shape = 4, (72, 70)
    src = gen("i32", NITEMS * ts, seed=3)
    chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
    bs = int(chunk[8:12].view(np.int32)[0])
    h = chunk.copy()
    h[16 + 4 * 5:16 + 4 * 6].view(np.int32)[0] = 0x7fff0000      # block 5's bstarts entry
    item5 = 5 * bs // ts                                           # an item of block 5
    for src_dev in (0, 1):
        slib.emu_set_device_ptrs(h.ctypes.data if src_dev else None, None)
        try:
            code = slib.blosc_getitem(ptr(h), ci(item5), ci(1), ptr(np.zeros(64, np.uint8)))
            assert code < 0
            _check(slib, h, src, ts, shape, [0, 0], [item5 // 70 - 1, 70], getitems=False)
            r5, c5 = divmod(item5, 70)
            out = np.full(4096, 0xAA, np.uint8)
            assert _getslice(slib, ptr(h), shape, [r5, 0], [r5 + 1, 70], out) == code and (out == 0xAA).all()
            assert _getslice(slib, ptr(h), shape, [0, c5], [72, c5 + 1], out) == code and (out == 0xAA).all()
        finally:
            slib.emu_set_device_ptrs(None, None)


def test_getslice_launches_emu(slib):
    """a box of one run and one of 10^4 runs in the same chunk make the same launches"""
    src = bench_words(80000)
    chunk = _compress(slib, "lz4", 5, 1, 4, src, 4096)
    assert not chunk[2] & 0x2
    counts = []
    for start, stop in (([5, 0], [6, 2]), ([0, 1], [10000, 2])):
        before = slib.emu_all_launches()
        _check(slib, chunk, src, 4, (10000, 2), start, stop, getitems=False)
        counts.append(slib.emu_all_launches() - before)
    assert counts[0] == counts[1] == 5, counts                    # touch, slot scan, decode, unfilter, gather


def test_getslice_rejects_emu(slib, capfd):
    ts = 4
    src = gen("i32", NITEMS * ts, seed=2)
    chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
    out = np.full(64, 0xAA, np.uint8)
    capfd.readouterr()
    for shape, start, stop in (((), (), ()), ((1,) * 8 + (5040,), (0,) * 9, (1,) * 9), ((-72, -70), (0, 0), (1, 1)),
                               ((72, 71), (0, 0), (1, 1)), ((1 << 40, 1 << 40), (0, 0), (1, 1)),
                               ((72, 70), (3, 0), (2, 1)), ((72, 70), (0, 0), (1, 71)), ((72, 70), (-1, 0), (1, 1))):
        before = slib.emu_all_launches()
        sh, st, sp = (_arr(v) if len(v) else np.zeros(1, np.int64) for v in (shape, start, stop))
        r = slib.blosc_b200_getslice(ptr(chunk), len(shape), sh.ctypes.data, st.ctypes.data, sp.ctypes.data, ptr(out))
        assert r == -1 and (out == 0xAA).all() and slib.emu_all_launches() == before, (shape, r)
        assert "blosc_b200" in capfd.readouterr().err, shape
    for patch, code in ((lambda h: h.__setitem__(0, 3), -9), (lambda h: h.__setitem__(1, 9), -9),
                        (lambda h: h.__setitem__(2, (h[2] & 0x1f) | (6 << 5)), -5),
                        (lambda h: h[8:12].view(np.int32).__setitem__(0, 0), -1)):
        h = chunk.copy()
        patch(h)
        assert slib.blosc_getitem(ptr(h), ci(0), ci(4), ptr(np.zeros(64, np.uint8))) == code
        assert _getslice(slib, ptr(h), (72, 70), (0, 0), (2, 3), out) == code and (out == 0xAA).all()


def _frame(lib, src, ts, chunksize, clevel=5):
    fb = lib.blosc_b200_frame_bound(len(src), ts, chunksize)
    frame = np.zeros(fb, np.uint8)
    r = lib.blosc_b200_frame_compress(clevel, 1, ts, len(src), ptr(src), ptr(frame), fb, b"lz4", 1024, chunksize, 1)
    assert r > 0
    return frame[:r].copy()


def _check_frame(lib, frame, src, ts, shape, start, stop, getitems=True):
    want = _want(src, ts, shape, start, stop)
    out = np.full(want.size + 16, 0xAA, np.uint8)
    r = _frame_getslice(lib, frame.ctypes.data, len(frame), shape, start, stop, out.ctypes.data)
    assert r == want.size and (out[:r] == want).all() and (out[r:] == 0xAA).all(), (shape, start, stop, r)
    if getitems:
        st, nn = _runs(shape, start, stop)
        g = np.full(want.size + 16, 0xAA, np.uint8)
        st64, nn64 = st.astype(np.uint64), nn.astype(np.uint64)
        assert lib.blosc_b200_frame_getitems(frame.ctypes.data, len(frame), st.size, st64.ctypes.data, nn64.ctypes.data,
                                             g.ctypes.data) == want.size
        assert (g == out).all()


@pytest.mark.parametrize("dev", [0, 1])
def test_frame_getslice_emu(slib, dev):
    """boxes across chunk boundaries, a chunksize that is no multiple of the row, a short last chunk"""
    ts, shape = 4, (50, 37)
    src = gen("i32", 50 * 37 * ts, seed=5)
    frame = _frame(slib, src, ts, 1000)                           # 250 items a chunk, 8 chunks, the last of 100
    slib.emu_set_all_device(dev)
    try:
        boxes = _boxes(shape, np.random.default_rng(dev), 5) + [([0, 0], [50, 37]), ([6, 36], [7, 37]),
                                                               ([47, 2], [50, 30]), ([0, 9], [50, 10])]
        for start, stop in boxes:
            _check_frame(slib, frame, src, ts, shape, start, stop)
        for start, stop in _boxes((10, 5, 37), np.random.default_rng(9), 3):
            _check_frame(slib, frame, src, ts, (10, 5, 37), start, stop)
    finally:
        slib.emu_set_all_device(0)


def test_frame_getslice_edges_emu(slib, capfd):
    """an empty frame, a chunk whose typesize differs from chunk 0's, a damaged chunk"""
    fb = slib.blosc_b200_frame_bound(0, 4, 1000)
    buf = np.zeros(fb, np.uint8)
    n = slib.blosc_b200_frame_compress(5, 1, 4, 0, ptr(buf), ptr(buf), fb, b"lz4", 0, 1000, 1)
    assert n > 0
    empty = buf[:n].copy()
    out = np.full(64, 0xAA, np.uint8)
    assert _frame_getslice(slib, empty.ctypes.data, len(empty), (0,), (0,), (0,), out.ctypes.data) == 0
    assert _frame_getslice(slib, empty.ctypes.data, len(empty), (0, 5), (0, 1), (0, 3), out.ctypes.data) == 0
    assert _frame_getslice(slib, empty.ctypes.data, len(empty), (4,), (0,), (1,), out.ctypes.data) == -1
    assert (out == 0xAA).all()

    ts, shape = 4, (50, 37)
    src = gen("i32", 50 * 37 * ts, seed=6)
    frame = _frame(slib, src, ts, 1000)
    off = [slib.blosc_b200_frame_chunk(frame.ctypes.data, len(frame), i, None) for i in range(8)]
    for patch, code in ((lambda f: f.__setitem__(off[2] + 3, 2), -1), (lambda f: f.__setitem__(off[2], 3), -9)):
        f = frame.copy()
        patch(f)
        for dev in (0, 1):
            slib.emu_set_all_device(dev)
            try:
                out = np.full(50 * 37 * ts + 16, 0xAA, np.uint8)
                capfd.readouterr()
                r = _frame_getslice(slib, f.ctypes.data, len(f), shape, (0, 0), (50, 37), out.ctypes.data)
                assert r == code and (dev or (out == 0xAA).all()), (code, r)
                if code == -1:
                    assert "blosc_b200" in capfd.readouterr().err
                _check_frame(slib, f, src, ts, shape, [0, 0], [6, 37], getitems=False)      # chunks 0 and 1 only
                _check_frame(slib, f, src, ts, shape, [21, 0], [50, 37], getitems=False)    # chunks 3 to 7
            finally:
                slib.emu_set_all_device(0)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the CUDA library
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def glib(pkg):
    return _bind(pkg.lib)


def _gpu_check(pkg, torch, chunk_h, chunk_d, src, ts, shape, start, stop):
    want = _want(src, ts, shape, start, stop)
    for s_buf in (chunk_h, chunk_d):
        for dest_dev in (False, True):
            out = torch.full((want.size + 16,), 0xAA, dtype=torch.uint8, device="cuda") if dest_dev else \
                np.full(want.size + 16, 0xAA, np.uint8)
            r = pkg.getslice(s_buf, shape, start, stop, out)
            got = out.cpu().numpy() if dest_dev else out
            assert r == want.size and (got[:r] == want).all() and (got[r:] == 0xAA).all(), (shape, start, stop, r)


@pytest.mark.gpu
@pytest.mark.parametrize("comp,switch", (("blosclz", None), ("lz4", None), ("zstd", "BLOSC_B200_ZSTD")))
@pytest.mark.parametrize("shuf", [0, 1, 2])
def test_getslice_matrix_gpu(pkg, glib, cuda, monkeypatch, comp, switch, shuf):
    n = 1 << 18                                                   # items: shapes below multiply to it
    shapes = {2: (512, 512), 3: (64, 64, 64), 8: (4, 4, 4, 4, 4, 4, 8, 8)}
    for i, ts in enumerate((1, 4, 3, 16)):
        src = (gen("mixed", n * ts, seed=ts) if i % 2 else bench_words(n * ts))
        for bs in (0, 16384):
            chunk = _compress(glib, comp, 5, shuf, ts, src, bs, monkeypatch, switch)
            d_chunk = cuda.from_numpy(chunk).cuda()
            for ndim, shape in shapes.items():
                for start, stop in _boxes(shape, np.random.default_rng(ts + ndim + bs), 2) + [([0] * ndim, list(shape))]:
                    _gpu_check(pkg, cuda, chunk, d_chunk, src, ts, shape, start, stop)
            _gpu_check(pkg, cuda, chunk, d_chunk, src, ts, (512, 512), [3, 0], [5, 512])
            _gpu_check(pkg, cuda, chunk, d_chunk, src, ts, (512, 512), [0, 7], [512, 8])


@pytest.mark.gpu
def test_getslice_rows_of_big_chunk_gpu(pkg, cuda):
    """a 256 MiB LZ4 + shuffle chunk, typesize 4, read as (2^24, 4): 2^22 rows of 8 bytes; equal to getitems with
    device lists and to the torch slice"""
    torch = cuda
    src = bench_words(256 << 20)
    d_src = torch.from_numpy(src).cuda()
    d_chunk = torch.zeros((256 << 20) + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(5, 1, 4, 256 << 20, d_src, d_chunk, (256 << 20) + 16, "lz4")
    assert cb > 0
    shape, start, stop = (1 << 24, 4), (1 << 20, 1), ((1 << 20) + (1 << 22), 3)
    want = d_src.view(torch.int32).view(1 << 24, 4)[start[0]:stop[0], 1:3].contiguous().view(torch.uint8).reshape(-1)
    out = torch.full((want.numel(),), 0xAA, dtype=torch.uint8, device="cuda")
    assert pkg.getslice(d_chunk, shape, start, stop, out) == want.numel() == 1 << 25
    assert torch.equal(out, want)
    st = torch.arange(start[0], stop[0], dtype=torch.int32, device="cuda") * 4 + 1
    g = torch.zeros_like(out)
    assert pkg.getitems(d_chunk, st, torch.full_like(st, 2), g) == want.numel()
    assert torch.equal(g, out)


@pytest.mark.gpu
def test_getslice_column_of_1gib_chunk_gpu(pkg, cuda):
    """a 1 GiB typesize-1 chunk shaped (2^29, 2), column 1: 2^29 one-byte runs"""
    torch = cuda
    n = 1 << 30
    i = torch.arange(n // 4, dtype=torch.int64, device="cuda")
    w = ((i << 26) ^ (i << 18) ^ (i << 11) ^ (i << 3) ^ i) & ((1 << 19) - 1)
    d_src = w.to(torch.int32).view(torch.uint8)
    del i, w
    d_chunk = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(5, 1, 1, n, d_src, d_chunk, n + 16, "lz4")
    assert cb > 0
    out = torch.full((n // 2,), 0xAA, dtype=torch.uint8, device="cuda")
    assert pkg.getslice(d_chunk[:cb], (1 << 29, 2), (0, 1), (1 << 29, 2), out) == n // 2
    assert torch.equal(out, d_src.view(1 << 29, 2)[:, 1])


@pytest.mark.gpu
def test_getslice_launches_gpu(pkg, cuda):
    """the launches of a box read do not grow with its runs"""
    torch = cuda
    src = bench_words(8 << 20)
    d_chunk = torch.from_numpy(_compress(pkg.lib, "lz4", 5, 1, 4, src, 0)).cuda()
    shape = (1 << 16, 32)
    grown = []
    for start, stop in (((5, 0), (6, 3)), ((0, 2), (10000, 5)), ((100, 1), (60000, 31))):
        want = _want(src, 4, shape, start, stop)
        out = torch.zeros(want.size, dtype=torch.uint8, device="cuda")
        before = pkg.launch_count()
        assert pkg.getslice(d_chunk, shape, start, stop, out) == want.size
        grown.append(pkg.launch_count() - before)
        assert (out.cpu().numpy() == want).all()
    assert grown == [5, 5, 5], grown


@pytest.mark.gpu
@pytest.mark.parametrize("frame_dev", [False, True])
def test_frame_getslice_gpu(pkg, glib, cuda, frame_dev):
    torch = cuda
    ts, shape = 4, (3000, 1001)
    src = bench_words(3000 * 1001 * ts)
    frame = _frame(glib, src, ts, 1 << 20)                        # 262144 items a chunk: 12 chunks, the last one short
    f_buf = torch.from_numpy(frame).cuda() if frame_dev else frame
    for start, stop in _boxes(shape, np.random.default_rng(3), 4) + [([0, 0], list(shape)), ([0, 500], [3000, 501]),
                                                                   ([261, 0], [1310, 1001])]:
        want = _want(src, ts, shape, start, stop)
        for dest_dev in (False, True):
            out = torch.full((want.size + 16,), 0xAA, dtype=torch.uint8, device="cuda") if dest_dev else \
                np.full(want.size + 16, 0xAA, np.uint8)
            assert pkg.frame_getslice(f_buf, len(frame), shape, start, stop, out) == want.size
            got = out.cpu().numpy() if dest_dev else out
            assert (got[:want.size] == want).all() and (got[want.size:] == 0xAA).all(), (start, stop)


@pytest.mark.gpu
def test_getslice_two_threads_gpu(pkg, cuda):
    """two host threads reading boxes of the same chunk and frame at once"""
    torch = cuda
    ts, shape = 4, (1024, 1536)
    src = bench_words(1024 * 1536 * ts)
    d_chunk = torch.from_numpy(_compress(pkg.lib, "lz4", 5, 1, ts, src, 0)).cuda()
    frame = _frame(pkg.lib, src, ts, 1 << 20)
    d_frame = torch.from_numpy(frame).cuda()
    errors = []

    def reader(seed):
        try:
            for rep, (start, stop) in enumerate(_boxes(shape, np.random.default_rng(seed), 6)):
                want = _want(src, ts, shape, start, stop)
                out = torch.full((want.size + 8,), 0xAA, dtype=torch.uint8, device="cuda")
                r = pkg.getslice(d_chunk, shape, start, stop, out) if rep % 2 else \
                    pkg.frame_getslice(d_frame, len(frame), shape, start, stop, out)
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

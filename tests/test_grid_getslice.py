"""blosc_b200_grid_getslice: a[start:stop:step] of an N-d C-order array stored as a regular grid of Blosc-1 chunks
(zarr v2, HDF5 blosc, PyTables), every touched chunk's part gathered straight into place.

Every result is checked against numpy slicing of the whole array, with sentinel bytes after the output left untouched.
The edge chunks' padding holds bytes (0xEE) that the array never holds.  CPU: the product's host code and kernels
inside the SIMT emulator (tests/emu/grid_stage.cpp, which counts launches by kind, keeps every decode launch's block
list and places any set of buffers in device memory).  GPU: the CUDA library through the Python API with torch
tensors."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

from datagen import bench_words, ci, compress, ptr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ll = C.c_longlong
vp = C.c_void_p
sz = C.c_size_t
CODECS = (("blosclz", None), ("lz4", None), ("lz4hc", None), ("zstd", "BLOSC_B200_ZSTD"),
          ("zlib", "BLOSC_B200_ZLIB"), ("snappy", "BLOSC_B200_SNAPPY"))
NEVER_SPLIT = 2
PAD = 0xEE


def _bind(lib):
    lib.blosc_b200_grid_getslice.restype = ll
    lib.blosc_b200_grid_getslice.argtypes = [ci, vp, vp, sz, vp, vp, vp, vp, vp, vp]
    lib.blosc_b200_getslice_step.restype = ll
    lib.blosc_b200_getslice_step.argtypes = [vp, ci, vp, vp, vp, vp, vp]
    lib.blosc_compress_ctx.restype = ci
    lib.blosc_getitem.restype = ci
    return lib


@pytest.fixture(scope="session")
def glib(tmp_path_factory):
    """the emulated library with the counters of tests/emu/grid_stage.cpp, built into a temporary directory"""
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("grid_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "c-blosc_b200", "csrc", "blosc_b200.c"), "-o",
                    str(d / "host.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "grid_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    path = str(d / "libgrid_stage.so")
    subprocess.run(["g++", "-shared", "-o", path, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    lib = _bind(C.CDLL(path))
    lib.emu_grid_set_device.argtypes = [vp, ci]
    lib.emu_grid_counts.argtypes = [vp]
    lib.emu_grid_decode_list.argtypes = [ci, vp, ci]
    lib.emu_grid_decode_list.restype = ci
    lib.blosc_set_splitmode.argtypes = [ci]
    lib.blosc_set_splitmode(NEVER_SPLIT)                          # small forced blocks: many of them per chunk
    return lib


# ---------------------------------------------------------------------------------------------------------------
# grids and expected results
# ---------------------------------------------------------------------------------------------------------------
def _array(shape, itemsize, seed):
    """a seeded array of itemsize-byte items whose bytes are all below 0xE0, as (shape + (itemsize,)) uint8"""
    rng = np.random.default_rng(seed)
    n = int(np.prod(shape)) * itemsize
    a = (np.arange(n) // 24 % 200).astype(np.uint8)               # compressible runs ...
    noise = rng.integers(0, 0xE0, n, dtype=np.uint8)
    a[n // 3:n // 2] = noise[n // 3:n // 2]                       # ... and a stretch of noise
    return a.reshape(*shape, itemsize)


def _grid(shape, chunkshape):
    return tuple(-(-s // c) for s, c in zip(shape, chunkshape))


def _chunk_data(arr, chunkshape, g):
    """the sub-array of chunk g at full chunk shape, padding bytes PAD"""
    itemsize = arr.shape[-1]
    buf = np.full(tuple(chunkshape) + (itemsize,), PAD, np.uint8)
    sl = tuple(slice(c * k, min((c + 1) * k, s)) for c, k, s in zip(g, chunkshape, arr.shape[:-1]))
    part = arr[sl]
    buf[tuple(slice(0, e) for e in part.shape[:-1])] = part
    return buf.reshape(-1)


def _compress(lib, comp, clevel, shuf, ts, data, bs, monkeypatch=None, switch=None):
    if switch:
        monkeypatch.setenv(switch, "1")
    r, c = compress(lib, "blosc_compress_ctx", clevel, shuf, ts, data, len(data) + 16, comp, bs)
    assert r > 0, (comp, ts, shuf, r)
    return c[:r].copy()


def _make_grid(lib, arr, chunkshape, comp="lz4", clevel=5, shuf=1, ts=None, bs=256, missing=(), monkeypatch=None,
               switch=None, each=None):
    """the chunks of arr, in grid C order (None at the grid indices in `missing`).  ts: the header typesize (default the
    itemsize, capped at 255).  each(i) -> (comp, clevel, shuf, ts) varies them per chunk."""
    itemsize = arr.shape[-1]
    out = []
    for i, g in enumerate(itertools.product(*(range(n) for n in _grid(arr.shape[:-1], chunkshape)))):
        if i in missing:
            out.append(None)
            continue
        c, lv, sh, t = each(i) if each else (comp, clevel, shuf, ts or min(itemsize, 255))
        out.append(_compress(lib, c, lv, sh, t, _chunk_data(arr, chunkshape, g), bs, monkeypatch, switch))
    return out


def _want(arr, start, stop, step, fill=None, chunkshape=None, missing=()):
    a = arr.copy()
    if missing:
        fb = np.zeros(arr.shape[-1], np.uint8) if fill is None else np.frombuffer(bytes(fill), np.uint8)
        grid = _grid(arr.shape[:-1], chunkshape)
        for i, g in enumerate(itertools.product(*(range(n) for n in grid))):
            if i in missing:
                a[tuple(slice(c * k, (c + 1) * k) for c, k in zip(g, chunkshape))] = fb
    sl = tuple(slice(s, e, t) for s, e, t in zip(start, stop, step or [1] * len(start)))
    return np.ascontiguousarray(a[sl]).reshape(-1)


def _i64(v):
    return np.ascontiguousarray(v, dtype=np.int64)


def _call(lib, chunks, shape, chunkshape, itemsize, start, stop, step, dest, fill=None, table=None):
    """blosc_b200_grid_getslice; `table` overrides the chunk table built from `chunks` (a ctypes array, or None)"""
    if table is None and chunks is not None:
        table = (vp * max(len(chunks), 1))(*[None if c is None else c.ctypes.data for c in chunks])
    sh, cs, st, sp = _i64(shape), _i64(chunkshape), _i64(start), _i64(stop)
    t = None if step is None else _i64(step)
    f = None if fill is None else np.frombuffer(bytes(fill), np.uint8)
    return lib.blosc_b200_grid_getslice(len(shape), sh.ctypes.data, cs.ctypes.data, itemsize, table,
                                        None if f is None else f.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                        None if t is None else t.ctypes.data, dest.ctypes.data)


def _check(lib, chunks, arr, chunkshape, start, stop, step=None, fill=None, missing=()):
    itemsize = arr.shape[-1]
    want = _want(arr, start, stop, step, fill, chunkshape, missing)
    out = np.full(want.size + 16, 0xAA, np.uint8)
    r = _call(lib, chunks, arr.shape[:-1], chunkshape, itemsize, start, stop, step, out, fill)
    assert r == want.size, (arr.shape, chunkshape, start, stop, step, r, want.size)
    assert (out[:r] == want).all() and (out[r:] == 0xAA).all(), (arr.shape, chunkshape, start, stop, step)
    return out[:r]


def _counts(lib):
    c = np.zeros(6, np.int64)
    lib.emu_grid_counts(c.ctypes.data)
    return dict(zip(("decode", "unfilter", "plan", "gather", "fill", "all"), c.tolist()))


def _sels(shape, chunkshape, rng, k):
    """k seeded selections: whole, inside one chunk, crossing chunks, with steps below, at and above the chunk shape"""
    out = []
    for _ in range(k):
        start, stop, step = [], [], []
        for s, c in zip(shape, chunkshape):
            a = int(rng.integers(0, s))
            b = int(rng.integers(a + 1, s + 1))
            t = int(rng.choice([1, 1, 2, 3, c, c + 1, 2 * c + 1]))
            start.append(a), stop.append(b), step.append(t)
        out.append((start, stop, step))
    return out


# ---------------------------------------------------------------------------------------------------------------
# CPU: the emulator
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("comp,switch", CODECS)
@pytest.mark.parametrize("shuf", [0, 1, 2])
def test_grid_codecs_emu(glib, monkeypatch, comp, switch, shuf):
    """every codec and filter, typesizes 1, 2, 3, 4, 8, 16, on a 2-d grid whose shape is no multiple of the chunk's"""
    for itemsize in (1, 2, 3, 4, 8, 16):
        shape, chunkshape = (23, 19), (8, 7)
        arr = _array(shape, itemsize, seed=itemsize + shuf)
        chunks = _make_grid(glib, arr, chunkshape, comp, 5, shuf, monkeypatch=monkeypatch, switch=switch)
        rng = np.random.default_rng(itemsize * 10 + shuf)
        for start, stop, step in [([0, 0], list(shape), None)] + _sels(shape, chunkshape, rng, 2):
            out = _check(glib, chunks, arr, chunkshape, start, stop, step)
            assert (out != PAD).all()


@pytest.mark.parametrize("shape,chunkshape", [((100,), (17,)), ((23, 19), (8, 7)), ((9, 11, 10), (4, 5, 3)),
                                              ((5, 6, 7, 4), (2, 4, 3, 3)),
                                              ((3, 2, 3, 2, 3, 2, 3, 4), (2, 1, 2, 2, 2, 1, 2, 3))])
def test_grid_ndim_emu(glib, shape, chunkshape):
    """ndim 1, 2, 3, 4 and 8: the whole array, one chunk exactly, aligned and unaligned boxes, one item, a line across
    every chunk, boxes inside one chunk, steps below, at and above the chunk shape"""
    itemsize = 4
    arr = _array(shape, itemsize, seed=len(shape))
    chunks = _make_grid(glib, arr, chunkshape)
    nd = len(shape)
    sels = [([0] * nd, list(shape), None),
            ([c for c in chunkshape], [min(2 * c, s) for c, s in zip(chunkshape, shape)], None),     # chunk 1,1,..
            ([0] * nd, [min(2 * c, s) for c, s in zip(chunkshape, shape)], None),                    # aligned
            ([1] * nd, [s - 1 if s > 2 else s for s in shape], None),                                # unaligned
            ([s // 2 for s in shape], [s // 2 + 1 for s in shape], None),                            # one item
            ([0] * (nd - 1) + [0], [1] * (nd - 1) + [shape[-1]], None),                              # a row
            ([0] * nd, list(shape[:1]) + [1] * (nd - 1), None),                                      # a column
            ([0] * nd, [min(c - 1, s) or 1 for c, s in zip(chunkshape, shape)], None),               # inside chunk 0
            ([0] * nd, list(shape), [max(c - 1, 1) for c in chunkshape]),
            ([0] * nd, list(shape), list(chunkshape)),
            ([1] * nd, list(shape), [c + 1 for c in chunkshape])]
    for start, stop, step in sels + _sels(shape, chunkshape, np.random.default_rng(nd), 4):
        out = _check(glib, chunks, arr, chunkshape, start, stop, step)
        assert (out != PAD).all()


def test_grid_untouched_never_read_emu(glib):
    """the table entries of untouched chunks point at 0xFF bytes, which fail any header check; the call succeeds"""
    shape, chunkshape, itemsize = (30, 28), (6, 7), 4
    arr = _array(shape, itemsize, seed=3)
    chunks = _make_grid(glib, arr, chunkshape)
    junk = np.full(64, 0xFF, np.uint8)
    grid = _grid(shape, chunkshape)
    for start, stop, step in (([7, 8], [17, 20], None), ([0, 3], [30, 4], None), ([0, 0], [30, 28], [13, 15]),
                              ([2, 1], [30, 28], [19, 22])):
        t = step or [1, 1]
        rows, cols = {r // 6 for r in range(start[0], stop[0], t[0])}, {q // 7 for q in range(start[1], stop[1], t[1])}
        bad = [c if (g // grid[1] in rows and g % grid[1] in cols) else junk for g, c in enumerate(chunks)]
        assert any(b is junk for b in bad)
        _check(glib, bad, arr, chunkshape, start, stop, step)


def test_grid_one_chunk_is_getslice_step_emu(glib, monkeypatch):
    """a grid of one chunk gives getslice_step's bytes and launches"""
    monkeypatch.setenv("BLOSC_B200_FRAME_WORKERS", "1")
    shape, itemsize = (40, 30), 4
    arr = _array(shape, itemsize, seed=5)
    chunks = _make_grid(glib, arr, shape)
    for start, stop, step in (([0, 0], [40, 30], None), ([3, 4], [37, 29], [2, 3]), ([0, 5], [40, 6], [1, 1]),
                              ([1, 0], [40, 30], [13, 1])):
        want = _want(arr, start, stop, step)
        a, b = np.full(want.size + 8, 0xAA, np.uint8), np.full(want.size + 8, 0xAA, np.uint8)
        glib.emu_grid_reset()
        assert _call(glib, chunks, shape, shape, itemsize, start, stop, step, a) == want.size
        ca = _counts(glib)
        glib.emu_grid_reset()
        t = None if step is None else _i64(step)
        assert glib.blosc_b200_getslice_step(ptr(chunks[0]), 2, _i64(shape).ctypes.data, _i64(start).ctypes.data,
                                             _i64(stop).ctypes.data, None if t is None else t.ctypes.data,
                                             b.ctypes.data) == want.size
        cb = _counts(glib)
        assert (a == b).all() and (a[:want.size] == want).all()
        assert ca == cb and ca["all"] == 5, (ca, cb)


@pytest.mark.parametrize("itemsize,fill", [(4, None), (4, b"\x01\x02\x03\x04"), (3, b"\xab\xcd\xef"), (1, b"\x7f")])
def test_grid_missing_chunks_emu(glib, monkeypatch, itemsize, fill):
    """missing chunks read as the fill value (zeros for NULL): one launch each, no decode"""
    monkeypatch.setenv("BLOSC_B200_FRAME_WORKERS", "1")
    shape, chunkshape = (25, 44), (8, 20)                        # a grid of 4 x 3 chunks
    arr = _array(shape, itemsize, seed=itemsize)
    grid = _grid(shape, chunkshape)
    missing = {0, 4, 7, 11}
    chunks = _make_grid(glib, arr, chunkshape, missing=missing)
    assert all(not c[2] & 0x2 for c in chunks if c is not None)    # compressed: each makes a decode launch
    for start, stop, step in (([0, 0], [25, 44], None), ([4, 3], [20, 41], None), ([0, 0], [25, 44], [4, 3])):
        glib.emu_grid_reset()
        _check(glib, chunks, arr, chunkshape, start, stop, step, fill=fill, missing=missing)
        c = _counts(glib)
        sel_rows = set(range(start[0], stop[0], (step or [1, 1])[0]))
        sel_cols = set(range(start[1], stop[1], (step or [1, 1])[1]))
        touched = {r // 8 * grid[1] + q // 20 for r in sel_rows for q in sel_cols}
        nmiss = len(touched & missing)
        assert c["fill"] == nmiss and c["decode"] == len(touched) - nmiss, (c, nmiss, len(touched))
        per = 5 if itemsize > 1 else 4                              # shuffle at typesize 1 has no unfilter launch
        assert c["all"] == per * (len(touched) - nmiss) + nmiss, c


def test_grid_itemsize_differs_from_typesize_emu(glib):
    """itemsize 4 over typesize-1 chunks, itemsize 300 over typesize-1 chunks, memcpyed chunks (in place on the
    device), and one grid mixing codecs, filters and typesizes"""
    shape, chunkshape = (19, 17), (5, 6)
    arr = _array(shape, 4, seed=8)
    sels = [([0, 0], [19, 17], None), ([2, 3], [18, 16], [2, 1]), ([1, 0], [19, 17], [1, 5])]
    for clevel in (5, 0):
        chunks = _make_grid(glib, arr, chunkshape, clevel=clevel, ts=1)
        for dev in (0, 1):
            glib.emu_grid_set_device((vp * len(chunks))(*[c.ctypes.data for c in chunks]) if dev else None,
                                     len(chunks) if dev else 0)
            try:
                for start, stop, step in sels:
                    _check(glib, chunks, arr, chunkshape, start, stop, step)
            finally:
                glib.emu_grid_set_device(None, 0)
    big = _array((7, 6), 300, seed=9)
    chunks = _make_grid(glib, big, (3, 4), ts=1, bs=512)
    for start, stop, step in (([0, 0], [7, 6], None), ([1, 1], [7, 5], [2, 3]), ([3, 2], [4, 3], None)):
        _check(glib, chunks, big, (3, 4), start, stop, step)
    kinds = [("lz4", 5, 1, 4), ("blosclz", 5, 2, 2), ("lz4", 0, 0, 1), ("lz4hc", 3, 0, 4), ("blosclz", 9, 1, 1)]
    chunks = _make_grid(glib, arr, chunkshape, each=lambda i: kinds[i % len(kinds)])
    for start, stop, step in sels:
        _check(glib, chunks, arr, chunkshape, start, stop, step)


@pytest.mark.parametrize("place", ["host", "device", "mixed"])
@pytest.mark.parametrize("dest_dev", [0, 1])
def test_grid_placements_emu(glib, place, dest_dev):
    """chunks in host memory, device memory or both, and dest in either"""
    shape, chunkshape = (21, 26), (5, 8)
    arr = _array(shape, 4, seed=11)
    chunks = _make_grid(glib, arr, chunkshape, each=lambda i: ("lz4", 0 if i % 3 == 0 else 5, 1, 4))
    rng = np.random.default_rng(len(place) + dest_dev)
    for start, stop, step in [([0, 0], [21, 26], None)] + _sels(shape, chunkshape, rng, 3):
        want = _want(arr, start, stop, step)
        out = np.full(want.size + 16, 0xAA, np.uint8)
        devs = [c.ctypes.data for i, c in enumerate(chunks) if place == "device" or (place == "mixed" and i % 2)]
        devs += [out.ctypes.data] if dest_dev else []
        glib.emu_grid_set_device((vp * max(len(devs), 1))(*devs), len(devs))
        try:
            r = _call(glib, chunks, shape, chunkshape, 4, start, stop, step, out)
        finally:
            glib.emu_grid_set_device(None, 0)
        assert r == want.size and (out[:r] == want).all() and (out[r:] == 0xAA).all()


def test_grid_launches_and_blocks_emu(glib, monkeypatch):
    """five launches per present touched chunk, none for untouched ones, and each chunk's decode lists exactly the
    blocks that hold a byte of a selected item"""
    monkeypatch.setenv("BLOSC_B200_FRAME_WORKERS", "1")
    for itemsize, shape, chunkshape in ((4, (40, 36), (16, 12)), (3, (30, 33), (11, 14)), (16, (12, 20), (5, 9))):
        arr = _array(shape, itemsize, seed=itemsize)
        chunks = _make_grid(glib, arr, chunkshape, bs=128)
        grid = _grid(shape, chunkshape)
        for start, stop, step in _sels(shape, chunkshape, np.random.default_rng(itemsize), 6):
            glib.emu_grid_reset()
            _check(glib, chunks, arr, chunkshape, start, stop, step)
            c = _counts(glib)
            rows, cols = range(start[0], stop[0], step[0]), range(start[1], stop[1], step[1])
            touched = sorted({r // chunkshape[0] * grid[1] + q // chunkshape[1] for r in rows for q in cols})
            assert c["decode"] == len(touched) and c["all"] == 5 * len(touched), (c, touched)
            for i, g in enumerate(touched):
                g0, g1 = divmod(g, grid[1])
                fl = [((r - g0 * chunkshape[0]) * chunkshape[1] + (q - g1 * chunkshape[1]))
                      for r in rows if r // chunkshape[0] == g0 for q in cols if q // chunkshape[1] == g1]
                fl = np.array(fl, np.int64) * itemsize
                want = np.unique(np.concatenate([fl // 128, (fl + itemsize - 1) // 128]))
                got = np.zeros(4096, np.int32)
                n = glib.emu_grid_decode_list(i, got.ctypes.data, 4096)
                assert n == want.size and (got[:n] == want).all(), (start, stop, step, g, got[:n], want)


@pytest.mark.parametrize("workers", ["1", "2", "8"])
def test_grid_workers_emu(glib, monkeypatch, workers):
    """1, 2 and 8 workers give identical bytes"""
    monkeypatch.setenv("BLOSC_B200_FRAME_WORKERS", workers)
    shape, chunkshape = (33, 29), (6, 5)
    arr = _array(shape, 4, seed=13)
    chunks = _make_grid(glib, arr, chunkshape, missing={4, 9})
    for start, stop, step in [([0, 0], [33, 29], None)] + _sels(shape, chunkshape, np.random.default_rng(1), 4):
        _check(glib, chunks, arr, chunkshape, start, stop, step, fill=b"\x05\x06\x07\x08", missing={4, 9})


def test_grid_damaged_chunks_emu(glib, monkeypatch):
    """two failing chunks, one with a damaged block and one with a bad header: the lower chunk's code, whatever the
    worker count and the placement; a host dest untouched"""
    shape, chunkshape = (24, 24), (6, 8)                          # a grid of 4 x 3 chunks
    arr = _array(shape, 4, seed=17)
    chunks = _make_grid(glib, arr, chunkshape, bs=128)
    out = np.full(24 * 24 * 4 + 16, 0xAA, np.uint8)

    def damaged(c):
        d = c.copy()
        d[16:20].view(np.int32)[0] = 0x7fff0000                    # block 0's bstarts entry
        return d

    def header(c, code):
        h = c.copy()
        if code == -5:
            h[2] = (h[2] & 0x1f) | (6 << 5)                        # an unknown codec
        else:
            h[0] = 3                                               # an unknown version
        return h

    for dev in (0, 1):
        glib.emu_set_all_device(dev)
        try:
            block = list(chunks)
            block[5] = damaged(chunks[5])
            code = _call(glib, block, shape, chunkshape, 4, [6, 16], [12, 24], None, out)   # chunk (1, 2) alone
            assert code < 0 and code not in (-5, -9) and (dev or (out == 0xAA).all())
            for lo, hi, want in ((header(chunks[5], -5), damaged(chunks[9]), -5),
                                 (damaged(chunks[5]), header(chunks[9], -9), code)):
                bad = list(chunks)
                bad[5], bad[9] = lo, hi
                for workers in ("1", "2", "8"):
                    monkeypatch.setenv("BLOSC_B200_FRAME_WORKERS", workers)
                    out[:] = 0xAA
                    assert _call(glib, bad, shape, chunkshape, 4, [0, 0], [24, 24], None, out) == want, (dev, workers)
                    assert dev or (out == 0xAA).all()
                    assert _call(glib, bad, shape, chunkshape, 4, [12, 0], [24, 24], None, out) not in (0, want)
                    _check(glib, bad, arr, chunkshape, [0, 0], [6, 24])                   # neither touched
        finally:
            glib.emu_set_all_device(0)


def test_grid_rejects_emu(glib, capfd):
    """every rejection returns -1 with one message before any launch; an empty selection with chunks NULL returns 0"""
    shape, chunkshape = (12, 10), (4, 5)
    arr = _array(shape, 4, seed=19)
    chunks = _make_grid(glib, arr, chunkshape)
    out = np.full(64, 0xAA, np.uint8)
    capfd.readouterr()
    big = 1 << 40
    for sh, cs, isz, st, sp, t, msg in (
            ((12, 10), (4, 5), 4, (0, 0), (2, 3), (1, 0), "step[1] = 0"),
            ((12, 10), (4, 5), 4, (0, 0), (13, 3), None, "inside"),
            ((-12, 10), (4, 5), 4, (0, 0), (1, 1), None, "negative"),
            ((12, 10), (0, 5), 4, (0, 0), (1, 1), None, "chunkshape[0] = 0"),
            ((12, 10), (4, -5), 4, (0, 0), (1, 1), None, "chunkshape[1] = -5"),
            ((12, 10), (4, 5), 0, (0, 0), (1, 1), None, "itemsize"),
            ((12, 10), (1 << 20, 1 << 20), 4, (0, 0), (1, 1), None, "larger"),
            ((12, 10), (big, big), 4, (0, 0), (1, 1), None, "larger"),
            ((12, 10), (4, 5), 1 << 62, (0, 0), (1, 1), None, "larger"),
            ((1 << 31, 1 << 31), (1, 1), 4, (0, 0), (1 << 31, 1 << 31), None, "output")):
        glib.emu_grid_reset()
        r = _call(glib, chunks, sh, cs, isz, st, sp, t, out)
        assert r == -1 and (out == 0xAA).all() and _counts(glib)["all"] == 0, (sh, cs, isz, r)
        err = capfd.readouterr().err
        assert err.count("blosc_b200") == 1 and msg in err, (sh, cs, isz, err)
    glib.emu_grid_reset()
    nul = C.cast(None, vp)
    assert _call(glib, None, shape, chunkshape, 4, (0, 0), (12, 10), None, out, table=nul) == -1
    assert "chunks is NULL" in capfd.readouterr().err
    assert _call(glib, None, shape, chunkshape, 4, (3, 0), (3, 10), None, out, table=nul) == 0
    assert _call(glib, None, shape, chunkshape, 4, (0, 0), (12, 10), (1, 1), out, table=nul) == -1
    assert _counts(glib)["all"] == 0 and (out == 0xAA).all()
    capfd.readouterr()
    h = list(chunks)                                               # a touched chunk of the wrong nbytes
    h[3] = _compress(glib, "lz4", 5, 1, 4, _chunk_data(arr, (4, 5), (1, 1))[:64], 256)
    assert _call(glib, h, shape, chunkshape, 4, (0, 0), (12, 10), None, out) == -1 and (out == 0xAA).all()
    assert "chunk (1, 1)" in capfd.readouterr().err
    h[3] = chunks[3].copy()
    h[3][0] = 3                                                    # a bad version: blosc_getitem's -9
    assert _call(glib, h, shape, chunkshape, 4, (0, 0), (12, 10), None, out) == -9 and (out == 0xAA).all()


# ---------------------------------------------------------------------------------------------------------------
# GPU: the CUDA library
# ---------------------------------------------------------------------------------------------------------------
def _gpu_grid(pkg, torch, src, chunkshape, comp, shuf, missing=()):
    """the chunks of the CUDA uint8 array src (shape + (itemsize,)) compressed on the device, in grid C order"""
    shape, itemsize = tuple(src.shape[:-1]), src.shape[-1]
    out = []
    for i, g in enumerate(itertools.product(*(range(n) for n in _grid(shape, chunkshape)))):
        if i in missing:
            out.append(None)
            continue
        buf = torch.full(tuple(chunkshape) + (itemsize,), PAD, dtype=torch.uint8, device="cuda")
        sl = tuple(slice(c * k, min((c + 1) * k, s)) for c, k, s in zip(g, chunkshape, shape))
        part = src[sl]
        buf[tuple(slice(0, e) for e in part.shape[:-1])] = part
        n = buf.numel()
        d = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
        cb = pkg.compress_ctx(5, shuf, min(itemsize, 255), n, buf, d, n + 16, comp)
        assert cb > 0
        out.append(d[:cb].clone())
    return out


def _gpu_want(torch, src, start, stop, step, chunkshape=None, missing=(), fill=None):
    a = src.clone()
    if missing:
        fb = torch.zeros(src.shape[-1], dtype=torch.uint8) if fill is None else torch.tensor(list(fill), dtype=torch.uint8)
        for i, g in enumerate(itertools.product(*(range(n) for n in _grid(src.shape[:-1], chunkshape)))):
            if i in missing:
                a[tuple(slice(c * k, (c + 1) * k) for c, k in zip(g, chunkshape))] = fb.cuda()
    return a[tuple(slice(s, e, t) for s, e, t in zip(start, stop, step))].contiguous().view(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("comp,switch", CODECS)
def test_grid_random_gpu(pkg, cuda, monkeypatch, comp, switch):
    """random grids and selections against torch, with 1 worker and the default, device and host dest"""
    torch = cuda
    if switch:
        monkeypatch.setenv(switch, "1")
    rng = np.random.default_rng(len(comp))
    for ndim, itemsize in ((1, 4), (2, 4), (3, 2), (4, 8)):
        shape = tuple(int(x) for x in rng.integers(20, {1: 5000, 2: 300, 3: 60, 4: 24}[ndim], ndim))
        chunkshape = tuple(int(max(1, s // int(rng.integers(2, 5)) + int(rng.integers(0, 3)))) for s in shape)
        src = torch.from_numpy(_array(shape, itemsize, seed=ndim)).cuda()
        chunks = _gpu_grid(pkg, torch, src, chunkshape, comp, 1 + ndim % 2)
        for start, stop, step in _sels(shape, chunkshape, rng, 3) + [([0] * ndim, list(shape), [1] * ndim)]:
            want = _gpu_want(torch, src, start, stop, step)
            for workers in ("1", None):
                if workers:
                    monkeypatch.setenv("BLOSC_B200_FRAME_WORKERS", workers)
                else:
                    monkeypatch.delenv("BLOSC_B200_FRAME_WORKERS", raising=False)
                for dest_dev in (True, False):
                    out = torch.full((want.numel() + 16,), 0xAA, dtype=torch.uint8,
                                     device="cuda" if dest_dev else "cpu")
                    r = pkg.grid_getslice(chunks, shape, chunkshape, itemsize, start, stop, out, step=step)
                    assert r == want.numel(), (shape, chunkshape, start, stop, step, r)
                    assert torch.equal(out[:r].cuda(), want) and bool((out[r:] == 0xAA).all())


@pytest.mark.gpu
def test_grid_many_in_flight_gpu(pkg, cuda):
    """a 256^3 float32 grid of 32^3 chunks (512 chunks, host and device), read whole, as a tile, a band and strided"""
    torch = cuda
    n, c = 256, 32
    src = torch.from_numpy(bench_words(n ** 3 * 4)).cuda().view(n, n, n, 4)
    chunks = _gpu_grid(pkg, torch, src, (c, c, c), "lz4", 1)
    host = [ch.cpu().numpy() for ch in chunks]
    for start, stop, step in (([0, 0, 0], [n, n, n], [1, 1, 1]), ([5, 17, 40], [200, 250, 170], [1, 1, 1]),
                              ([0, 100, 0], [n, 110, n], [1, 1, 1]), ([0, 0, 0], [n, n, n], [8, 8, 8]),
                              ([3, 1, 2], [n, n, n], [33, 5, 2])):
        want = _gpu_want(torch, src, start, stop, step)
        for table in (chunks, host):
            out = torch.full((want.numel(),), 0xAA, dtype=torch.uint8, device="cuda")
            assert pkg.grid_getslice(table, (n, n, n), (c, c, c), 4, start, stop, out, step=step) == want.numel()
            assert torch.equal(out, want), (start, stop, step)


@pytest.mark.gpu
def test_grid_missing_gpu(pkg, cuda):
    """missing chunks read as the fill value, with a numpy-scalar fill and with zeros"""
    torch = cuda
    shape, chunkshape = (300, 260), (64, 50)
    src = torch.from_numpy(_array(shape, 4, seed=2)).cuda()
    missing = {0, 5, 6, 11, 29}
    chunks = _gpu_grid(pkg, torch, src, chunkshape, "lz4", 1, missing=missing)
    for fill in (None, np.float32(1.5)):
        fb = None if fill is None else fill.tobytes()
        for start, stop, step in (([0, 0], [300, 260], [1, 1]), ([10, 7], [290, 250], [3, 2])):
            want = _gpu_want(torch, src, start, stop, step, chunkshape, missing, fb)
            out = torch.full((want.numel(),), 0xAA, dtype=torch.uint8, device="cuda")
            assert pkg.grid_getslice(chunks, shape, chunkshape, 4, start, stop, out, step=step, fill=fill) == want.numel()
            assert torch.equal(out, want), (fill, start, stop, step)


@pytest.mark.gpu
def test_grid_python_args_gpu(pkg, cuda):
    """a table of the wrong length and a fill of the wrong size raise"""
    torch = cuda
    src = torch.from_numpy(_array((10, 10), 4, seed=1)).cuda()
    chunks = _gpu_grid(pkg, torch, src, (5, 5), "lz4", 1)
    out = torch.zeros(400, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        pkg.grid_getslice(chunks[:3], (10, 10), (5, 5), 4, (0, 0), (10, 10), out)
    with pytest.raises(ValueError):
        pkg.grid_getslice(chunks, (10, 10), (5, 5), 4, (0, 0), (10, 10), out, fill=b"\x00")
    assert pkg.grid_getslice(chunks, (10, 10), (5, 5), 4, (0, 0), (10, 10), out) == 400
    assert torch.equal(out, src.view(-1))

"""blosc_b200_grid_compress: an N-d C-order array written as the regular grid of Blosc-1 chunks that grid_getslice reads
(zarr v2, HDF5 blosc), each chunk packed out of the array and compressed, several in flight.

Every chunk is checked byte for byte against the same library's blosc_compress_ctx of the numpy-padded sub-array, and
the offsets against the chunks' sizes laid back to back.  CPU: the product's host code and kernels inside the SIMT
emulator (tests/emu/grid_stage.cpp, which counts launches by kind and places any set of buffers in device memory).
GPU: the CUDA library through the Python API with torch tensors."""
import ctypes as C
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

from datagen import ci
from test_grid_getslice import _array, _bind, _call, _grid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ll = C.c_longlong
vp = C.c_void_p
sz = C.c_size_t
CODECS = (("blosclz", None), ("lz4", None), ("lz4hc", None), ("zstd", "BLOSC_B200_ZSTD"),
          ("zlib", "BLOSC_B200_ZLIB"), ("snappy", "BLOSC_B200_SNAPPY"))
NEVER_SPLIT = 2


@pytest.fixture(scope="session")
def glib(tmp_path_factory):
    """the emulated library with the counters of tests/emu/grid_stage.cpp, built into a temporary directory"""
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("grid_compress_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "c-blosc_b200", "csrc", "blosc_b200.c"), "-o",
                    str(d / "host.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "grid_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    path = str(d / "libgrid_compress_stage.so")
    subprocess.run(["g++", "-shared", "-o", path, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    lib = _bind(C.CDLL(path))
    lib.blosc_compress_ctx.argtypes = [ci, ci, sz, sz, vp, vp, sz, C.c_char_p, sz, ci]
    lib.blosc_decompress_ctx.restype = ci
    lib.blosc_decompress_ctx.argtypes = [vp, vp, sz, ci]
    lib.blosc_b200_grid_bound.restype = sz
    lib.blosc_b200_grid_bound.argtypes = [ci, vp, vp, sz]
    lib.blosc_b200_grid_compress.restype = ll
    lib.blosc_b200_grid_compress.argtypes = [ci, ci, sz, C.c_char_p, sz, ci, ci, vp, vp, sz, vp, vp, ci, vp, sz, vp]
    lib.emu_grid_set_device.argtypes = [vp, ci]
    lib.emu_grid_counts.argtypes = [vp]
    lib.emu_set_all_device.argtypes = [ci]
    lib.blosc_set_splitmode.argtypes = [ci]
    lib.blosc_set_splitmode(NEVER_SPLIT)                          # small forced blocks: many of them per chunk
    return lib


# ---------------------------------------------------------------------------------------------------------------
# expected chunks
# ---------------------------------------------------------------------------------------------------------------
def _coords(shape, chunkshape):
    return list(itertools.product(*(range(n) for n in _grid(shape, chunkshape))))


def _edge(shape, chunkshape, g):
    return any((c + 1) * k > s for c, k, s in zip(g, chunkshape, shape))


def _padded(arr, chunkshape, g, fill=None):
    """chunk g's sub-array at full chunk shape, padding the fill pattern (None: zeros), as flat bytes"""
    itemsize = arr.shape[-1]
    buf = np.empty(tuple(chunkshape) + (itemsize,), np.uint8)
    buf[...] = np.zeros(itemsize, np.uint8) if fill is None else np.frombuffer(bytes(fill), np.uint8)
    sl = tuple(slice(c * k, min((c + 1) * k, s)) for c, k, s in zip(g, chunkshape, arr.shape[:-1]))
    part = arr[sl]
    buf[tuple(slice(0, e) for e in part.shape[:-1])] = part
    return buf.reshape(-1)


def _ref_chunk(lib, data, clevel, shuf, ts, comp, bs):
    d = np.full(data.size + 16, 0xAA, np.uint8)
    r = lib.blosc_compress_ctx(clevel, shuf, ts, data.size, data.ctypes.data, d.ctypes.data, data.size + 16,
                               comp.encode(), bs, 1)
    assert r > 0, (comp, clevel, shuf, ts, r)
    return d[:r].copy()


def _i64(v):
    return np.ascontiguousarray(v, dtype=np.int64)


def _bound(lib, shape, chunkshape, itemsize):
    sh, cs = _i64(shape), _i64(chunkshape)
    return int(lib.blosc_b200_grid_bound(len(shape), sh.ctypes.data, cs.ctypes.data, itemsize))


def _gc(lib, src, shape, chunkshape, itemsize, clevel=5, shuf=1, comp="lz4", ts=None, bs=256, fill=None, skip=0,
        dest=None, destsize=None, offsets=None, nchunks=None):
    """blosc_b200_grid_compress; returns (code, offsets, dest)"""
    if nchunks is None:
        nchunks = int(np.prod(_grid(shape, chunkshape))) if all(c >= 1 for c in chunkshape) else 0
    sh, cs = _i64(shape), _i64(chunkshape)                        # kept alive across the call
    if dest is None:
        dest = np.full(max(_bound(lib, shape, chunkshape, itemsize), 1), 0xAA, np.uint8)
    if offsets is None:
        offsets = np.full(nchunks + 1, -7, np.int64)
    f = None if fill is None else np.frombuffer(bytes(fill), np.uint8)
    r = lib.blosc_b200_grid_compress(clevel, shuf, itemsize if ts is None else ts, comp.encode() if comp else None, bs, 1,
                                     len(shape), sh.ctypes.data, cs.ctypes.data, itemsize,
                                     None if src is None else src.ctypes.data, None if f is None else f.ctypes.data, skip,
                                     dest.ctypes.data, dest.size if destsize is None else destsize,
                                     None if offsets is False else offsets.ctypes.data)
    return r, offsets, dest


def _check(lib, arr, chunkshape, clevel=5, shuf=1, comp="lz4", ts=None, bs=256, fill=None, dev=()):
    """the grid of arr against compress_ctx of every padded sub-array; dev: which of "src" / "dest" are device memory.
    Returns the chunks."""
    shape, itemsize = arr.shape[:-1], arr.shape[-1]
    src = np.ascontiguousarray(arr).reshape(-1)
    dest = np.full(_bound(lib, shape, chunkshape, itemsize) + 32, 0xAA, np.uint8)
    ptrs = ([src.ctypes.data] if "src" in dev else []) + ([dest.ctypes.data] if "dest" in dev else [])
    lib.emu_grid_set_device((vp * max(len(ptrs), 1))(*ptrs), len(ptrs))
    try:
        r, off, out = _gc(lib, src, shape, chunkshape, itemsize, clevel, shuf, comp, ts, bs, fill, dest=dest)
    finally:
        lib.emu_grid_set_device(None, 0)
    assert r > 0 and off[0] == 0 and off[-1] == r, (shape, chunkshape, itemsize, comp, r, off)
    assert (out[r:] == 0xAA).all()
    chunks = []
    for i, g in enumerate(_coords(shape, chunkshape)):
        want = _ref_chunk(lib, _padded(arr, chunkshape, g, fill), clevel, shuf, itemsize if ts is None else ts, comp, bs)
        got = out[off[i]:off[i + 1]]
        assert got.size == want.size and (got == want).all(), (shape, chunkshape, itemsize, comp, shuf, g)
        chunks.append(got.copy())
    return chunks


def _counts(lib):
    c = np.zeros(6, np.int64)
    lib.emu_grid_counts(c.ctypes.data)
    return dict(zip(("decode", "filter", "plan", "gather", "fill", "all"), c.tolist()))


# ---------------------------------------------------------------------------------------------------------------
# CPU: the emulator
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("comp,switch", CODECS)
@pytest.mark.parametrize("shuf", [0, 1, 2])
def test_grid_compress_codecs_emu(glib, monkeypatch, comp, switch, shuf):
    """every codec and filter at itemsizes 1, 2, 4, 8, 12 and 300 (header typesize 1), on a 2-d grid whose shape is no
    multiple of the chunk's, from a device array"""
    if switch:
        monkeypatch.setenv(switch, "1")
    for itemsize in (1, 2, 4, 8, 12, 300):
        shape, chunkshape = ((11, 9), (4, 5)) if itemsize < 300 else ((5, 3), (2, 2))
        arr = _array(shape, itemsize, seed=itemsize + shuf)
        _check(glib, arr, chunkshape, 5, shuf, comp, bs=256 if itemsize < 300 else 1200, dev=("src",))


@pytest.mark.parametrize("shape,chunkshape", [((100,), (17,)), ((64,), (16,)), ((23, 19), (8, 7)), ((24, 21), (8, 7)),
                                              ((9, 11, 10), (4, 12, 3)), ((5, 6, 7, 4), (2, 1, 3, 4)),
                                              ((6, 5), (1, 9))])
@pytest.mark.parametrize("itemsize,fill", [(4, None), (4, b"\x01\x02\x03\x04"), (12, bytes(range(7, 19))),
                                           (2, b"\xff\x7f")])
def test_grid_compress_ndim_emu(glib, shape, chunkshape, itemsize, fill):
    """1-d to 4-d, shapes that are and are not multiples of the chunk shape, a chunk shape larger than the shape or 1
    along a dimension, zero and non-zero fill patterns: host and device src"""
    arr = _array(shape, itemsize, seed=len(shape) + itemsize)
    for dev in ((), ("src",)):
        _check(glib, arr, chunkshape, 5, 1, "lz4", fill=fill, dev=dev)


@pytest.mark.parametrize("dev", [(), ("src",), ("dest",), ("src", "dest")])
def test_grid_compress_placements_emu(glib, monkeypatch, dev):
    """device and host src and dest give identical bytes; a device src packs with one gather launch per chunk plus one
    fill per edge chunk, a host src with none"""
    monkeypatch.setenv("BLOSC_B200_FRAME_WORKERS", "1")
    shape, chunkshape = (21, 26), (5, 8)
    arr = _array(shape, 4, seed=11)
    coords = _coords(shape, chunkshape)
    nedge = sum(_edge(shape, chunkshape, g) for g in coords)
    glib.emu_grid_reset()
    _check(glib, arr, chunkshape, 5, 1, "lz4", fill=b"\x09\x08\x07\x06", dev=dev)
    c = _counts(glib)
    if "src" in dev:
        assert c["gather"] == len(coords) + nedge and c["fill"] == nedge, c
    else:
        assert c["gather"] == 0 and c["fill"] == 0, c


@pytest.mark.parametrize("comp,switch", [("lz4", None), ("zstd", "BLOSC_B200_ZSTD"), ("blosclz", None)])
@pytest.mark.parametrize("dev", [("src",), ("src", "dest"), ()])
def test_grid_compress_memcpyed_emu(glib, monkeypatch, comp, switch, dev):
    """memcpyed chunks come from the packed bytes: incompressible noise, clevel 0, and chunks below 128 bytes"""
    if switch:
        monkeypatch.setenv(switch, "1")
    rng = np.random.default_rng(5)
    noise = rng.integers(0, 256, (12, 18, 4), dtype=np.uint8)          # no edge chunk: no compressible padding
    chunks = _check(glib, noise, (6, 6), 5, 1, comp, dev=dev)
    assert all(c[2] & 0x2 for c in chunks)                           # every chunk is memcpyed
    arr = _array((13, 14), 4, seed=3)
    chunks = _check(glib, arr, (6, 6), 0, 1, comp, dev=dev)
    assert all(c[2] & 0x2 for c in chunks)
    chunks = _check(glib, arr, (3, 4), 5, 1, comp, fill=b"\x01\x00\x00\x00", dev=dev)    # 48-byte chunks
    assert all(c[2] & 0x2 for c in chunks) and all(c.size == 48 + 16 for c in chunks)


def test_grid_compress_round_trip_emu(glib, ref_if_built):
    """each chunk decompresses to its padded sub-array (and so in the reference, where it is built); grid_getslice over
    the chunks reproduces numpy slicing, steps included"""
    shape, chunkshape, fill = (25, 31, 6), (8, 10, 4), b"\x05\x06\x07\x08"
    arr = _array(shape, 4, seed=21)
    for comp in ("lz4", "blosclz", "lz4hc"):
        chunks = _check(glib, arr, chunkshape, 5, 1, comp, fill=fill, dev=("src",))
        for g, c in zip(_coords(shape, chunkshape), chunks):
            want = _padded(arr, chunkshape, g, fill)
            out = np.zeros(want.size, np.uint8)
            assert glib.blosc_decompress_ctx(c.ctypes.data, out.ctypes.data, out.size, 1) == want.size
            assert (out == want).all()
            if ref_if_built is not None:
                out[:] = 0
                assert ref_if_built.blosc_decompress_ctx(C.c_void_p(c.ctypes.data), C.c_void_p(out.ctypes.data),
                                                         C.c_size_t(out.size), C.c_int(1)) == want.size
                assert (out == want).all()
        for start, stop, step in (([0, 0, 0], list(shape), None), ([3, 2, 1], [24, 30, 6], [2, 3, 1]),
                                  ([1, 0, 5], [25, 31, 6], [7, 11, 1])):
            sl = tuple(slice(s, e, t) for s, e, t in zip(start, stop, step or [1] * 3))
            want = np.ascontiguousarray(arr[sl]).reshape(-1)
            out = np.full(want.size + 8, 0xAA, np.uint8)
            assert _call(glib, chunks, shape, chunkshape, 4, start, stop, step, out) == want.size
            assert (out[:want.size] == want).all() and (out[want.size:] == 0xAA).all()


@pytest.mark.parametrize("dev", [(), ("src",)])
@pytest.mark.parametrize("fill", [None, b"\x00\x00\x80\x3f"])
def test_grid_compress_skip_fill_emu(glib, dev, fill):
    """chunks holding only the fill pattern inside the array are left out (an edge chunk included), a chunk with one
    differing byte is kept, and grid_getslice over the result reproduces the array"""
    shape, chunkshape = (20, 23), (6, 8)                          # a grid of 4 x 3 chunks; the last row and column edge
    coords = _coords(shape, chunkshape)
    fb = np.zeros(4, np.uint8) if fill is None else np.frombuffer(fill, np.uint8)
    arr = _array(shape, 4, seed=2)
    empty = {0, 5, 11}                                            # 5 and 11 are edge chunks
    for i in empty:
        g = coords[i]
        arr[g[0] * 6:(g[0] + 1) * 6, g[1] * 8:(g[1] + 1) * 8] = fb
    g = coords[7]                                                 # all fill but one byte
    arr[g[0] * 6:(g[0] + 1) * 6, g[1] * 8:(g[1] + 1) * 8] = fb
    arr[g[0] * 6 + 2, g[1] * 8 + 3, 1] ^= 0x10
    src = np.ascontiguousarray(arr).reshape(-1)
    lib = glib
    lib.emu_grid_set_device((vp * 1)(src.ctypes.data) if dev else None, 1 if dev else 0)
    try:
        r, off, out = _gc(lib, src, shape, chunkshape, 4, fill=fill, skip=1)
        r0, off0, out0 = _gc(lib, src, shape, chunkshape, 4, fill=fill, skip=0)
    finally:
        lib.emu_grid_set_device(None, 0)
    sizes = np.diff(off)
    assert r == off[-1] and [i for i in range(len(coords)) if sizes[i] == 0] == sorted(empty), sizes
    kept = [i for i in range(len(coords)) if i not in empty]
    assert (np.concatenate([out0[off0[i]:off0[i + 1]] for i in kept]) == out[:r]).all()
    chunks = [None if sizes[i] == 0 else out[off[i]:off[i + 1]].copy() for i in range(len(coords))]
    want = np.ascontiguousarray(arr).reshape(-1)
    got = np.full(want.size, 0xAA, np.uint8)
    assert _call(lib, chunks, shape, chunkshape, 4, [0, 0], list(shape), None, got, fill=fill) == want.size
    assert (got == want).all()


def test_grid_compress_budget_emu(glib):
    """destsize equal to the total fits, one byte less returns 0, and the bound always fits"""
    shape, chunkshape = (17, 19), (5, 6)
    arr = _array(shape, 4, seed=4)
    src = np.ascontiguousarray(arr).reshape(-1)
    r, off, out = _gc(glib, src, shape, chunkshape, 4)
    assert r > 0
    nb = _bound(glib, shape, chunkshape, 4)
    assert nb == len(_coords(shape, chunkshape)) * (30 * 4 + 16)
    r2, off2, out2 = _gc(glib, src, shape, chunkshape, 4, dest=np.full(r, 0xAA, np.uint8))
    assert r2 == r and (off2 == off).all() and (out2 == out[:r]).all()
    assert _gc(glib, src, shape, chunkshape, 4, dest=np.full(r - 1, 0xAA, np.uint8))[0] == 0
    noise = np.random.default_rng(1).integers(0, 256, src.size, dtype=np.uint8)
    r3, _, _ = _gc(glib, noise, shape, chunkshape, 4, dest=np.zeros(nb, np.uint8))
    assert r3 == nb                                               # every chunk memcpyed: the bound exactly
    big = 1 << 40
    assert _bound(glib, (big, big), (1, 1), 1 << 20) == 0 and _bound(glib, (4, 4), (0, 1), 4) == 0


@pytest.mark.parametrize("comp,switch", [("lz4", None), ("snappy", "BLOSC_B200_SNAPPY")])
def test_grid_compress_workers_emu(glib, monkeypatch, comp, switch):
    """1 and 4 workers give identical bytes and offsets"""
    if switch:
        monkeypatch.setenv(switch, "1")
    shape, chunkshape = (33, 29), (6, 5)
    arr = _array(shape, 4, seed=13)
    src = np.ascontiguousarray(arr).reshape(-1)
    res = []
    for workers in ("1", "4"):
        monkeypatch.setenv("BLOSC_B200_FRAME_WORKERS", workers)
        for dev in (0, 1):
            glib.emu_grid_set_device((vp * 1)(src.ctypes.data) if dev else None, dev)
            try:
                r, off, out = _gc(glib, src, shape, chunkshape, 4, comp=comp)
            finally:
                glib.emu_grid_set_device(None, 0)
            res.append((r, off.copy(), out[:r].copy()))
    for r, off, out in res[1:]:
        assert r == res[0][0] and (off == res[0][1]).all() and (out == res[0][2]).all()


def test_grid_compress_rejects_emu(glib, capfd):
    """every -1, -10 and -5 returns before anything is launched, -1 with one message; an empty grid returns 0 with
    offsets[0] == 0"""
    shape, chunkshape = (12, 10), (4, 5)
    src = np.ascontiguousarray(_array(shape, 4, seed=19)).reshape(-1)
    dest = np.full(4096, 0xAA, np.uint8)
    capfd.readouterr()
    big = 1 << 40
    for sh, cs, isz, msg in (((-12, 10), (4, 5), 4, "negative"), ((12, 10), (0, 5), 4, "chunkshape[0] = 0"),
                             ((12, 10), (4, -5), 4, "chunkshape[1] = -5"), ((12, 10), (4, 5), 0, "itemsize"),
                             ((12, 10), (1 << 20, 1 << 20), 4, "larger"), ((12, 10), (big, big), 4, "larger"),
                             ((1 << 31, 1 << 31), (1, 1), 1, "chunks"), ((1 << 20, 1 << 20), (1, 1), 1, "chunks"),
                             ((1,) * 9, (1,) * 9, 4, "ndim")):
        glib.emu_grid_reset()
        r, _, _ = _gc(glib, src, sh, cs, isz, ts=4, dest=dest, offsets=np.zeros(4, np.int64), nchunks=3)
        assert r == -1 and (dest == 0xAA).all() and _counts(glib)["all"] == 0, (sh, cs, isz, r)
        err = capfd.readouterr().err
        assert err.count("blosc_b200") == 1 and msg in err, (sh, cs, isz, err)
    for kw, code in (({"clevel": 10}, -10), ({"clevel": -1}, -10), ({"shuf": 3}, -10), ({"ts": 0}, -10),
                     ({"comp": "nope"}, -5), ({"comp": "zstd"}, -5), ({"comp": None}, -5)):
        glib.emu_grid_reset()
        assert _gc(glib, src, shape, chunkshape, 4, dest=dest, **kw)[0] == code, kw
        assert _counts(glib)["all"] == 0 and (dest == 0xAA).all()
    glib.emu_grid_reset()
    assert _gc(glib, None, shape, chunkshape, 4, dest=dest)[0] == -1
    assert "src is NULL" in capfd.readouterr().err
    assert _gc(glib, src, shape, chunkshape, 4, dest=dest, offsets=False)[0] == -1
    assert "offsets is NULL" in capfd.readouterr().err
    assert _counts(glib)["all"] == 0 and (dest == 0xAA).all()
    off = np.full(1, -7, np.int64)
    assert _gc(glib, None, (12, 0), chunkshape, 4, dest=dest, offsets=off, nchunks=0)[0] == 0 and off[0] == 0
    assert _gc(glib, None, (0, 10), chunkshape, 4, dest=dest, offsets=False, nchunks=0)[0] == 0
    assert _counts(glib)["all"] == 0 and (dest == 0xAA).all()


def test_grid_compress_asan_emu(tmp_path):
    """the AddressSanitizer build of the emulated library over edge-chunk geometries, the array in an exactly sized
    allocation: no read outside it"""
    libasan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(libasan) or not os.path.exists(libasan):
        pytest.skip("no libasan")
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "tests", "emu"), "asan"], check=True)
    env = dict(os.environ, LD_PRELOAD=libasan, ASAN_OPTIONS="detect_leaks=0")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "asan_grid_compress.py")], env=env,
                       capture_output=True, text=True)
    assert p.returncode == 0 and "ERROR: AddressSanitizer" not in p.stderr, p.stderr[-4000:]
    assert "grid_compress asan ok" in p.stdout


# ---------------------------------------------------------------------------------------------------------------
# GPU: the CUDA library
# ---------------------------------------------------------------------------------------------------------------
def _gpu_ref(pkg, torch, src, chunkshape, comp, shuf, clevel=5, fill=None):
    """compress_ctx on the GPU of every padded sub-array of the CUDA uint8 array src (shape + (itemsize,))"""
    shape, itemsize = tuple(src.shape[:-1]), src.shape[-1]
    fb = torch.zeros(itemsize, dtype=torch.uint8) if fill is None else torch.tensor(list(fill), dtype=torch.uint8)
    out = []
    for g in _coords(shape, chunkshape):
        buf = fb.cuda().expand(tuple(chunkshape) + (itemsize,)).contiguous()
        sl = tuple(slice(c * k, min((c + 1) * k, s)) for c, k, s in zip(g, chunkshape, shape))
        part = src[sl]
        buf[tuple(slice(0, e) for e in part.shape[:-1])] = part
        n = buf.numel()
        d = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
        cb = pkg.compress_ctx(clevel, shuf, itemsize, n, buf, d, n + 16, comp)
        assert cb > 0
        out.append(d[:cb].cpu())
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("comp,switch", CODECS)
def test_grid_compress_gpu(pkg, cuda, monkeypatch, comp, switch):
    """byte identity against per-chunk compress_ctx for a CUDA src with CUDA or host dest and for a numpy src, with 1
    worker and the default, and the round trip through grid_getslice"""
    torch = cuda
    if switch:
        monkeypatch.setenv(switch, "1")
    for shape, chunkshape, itemsize, shuf, fill in (((1000, 37), (128, 16), 4, 1, None),
                                                    ((50, 60, 70), (16, 32, 20), 2, 2, b"\x01\x02"),
                                                    ((3000,), (512,), 8, 1, bytes(range(8))),
                                                    ((40, 30), (64, 7), 12, 0, None)):
        host = _array(shape, itemsize, seed=len(shape))
        src = torch.from_numpy(host).cuda()
        want = _gpu_ref(pkg, torch, src, chunkshape, comp, shuf, fill=fill)
        bound = pkg.grid_bound(shape, chunkshape, itemsize)
        for workers in ("1", None):
            if workers:
                monkeypatch.setenv("BLOSC_B200_FRAME_WORKERS", workers)
            else:
                monkeypatch.delenv("BLOSC_B200_FRAME_WORKERS", raising=False)
            for s, dest_dev in ((src, True), (src, False), (host, True), (host, False)):
                dest = torch.full((bound,), 0xAA, dtype=torch.uint8, device="cuda" if dest_dev else "cpu")
                r, off = pkg.grid_compress(s, shape, chunkshape, itemsize, 5, shuf, comp, dest, fill=fill)
                assert r == off[-1] > 0 and off[0] == 0, (shape, r)
                chunks = pkg.grid_chunks(dest, off)
                for g, c, w in zip(_coords(shape, chunkshape), chunks, want):
                    assert torch.equal(c.cpu(), w), (shape, chunkshape, g, dest_dev)
        nd = len(shape)
        for start, stop, step in (([0] * nd, list(shape), [1] * nd), ([1] * nd, list(shape), [3] * nd)):
            sel = src[tuple(slice(a, b, t) for a, b, t in zip(start, stop, step))].contiguous().view(-1)
            out = torch.full((sel.numel(),), 0xAA, dtype=torch.uint8, device="cuda")
            assert pkg.grid_getslice(chunks, shape, chunkshape, itemsize, start, stop, out, step=step) == sel.numel()
            assert torch.equal(out, sel)


@pytest.mark.gpu
def test_grid_compress_skip_fill_gpu(pkg, cuda):
    """a 256^3 float32 grid of 32^3 chunks with most chunks all fill: those are left out, and the round trip holds"""
    torch = cuda
    n, c = 256, 32
    for fill in (None, np.float32(-1.0)):
        f = 0.0 if fill is None else float(fill)
        src = torch.full((n, n, n), f, dtype=torch.float32, device="cuda")
        src[:64, :, :96] = torch.rand(64, n, 96, device="cuda")
        src[200, 17, 250] = 3.0                                    # one item in an otherwise empty chunk
        dest = torch.empty(pkg.grid_bound((n, n, n), (c, c, c), 4), dtype=torch.uint8, device="cuda")
        r, off = pkg.grid_compress(src, (n, n, n), (c, c, c), 4, 5, 1, "lz4", dest, fill=fill, skip_fill=True)
        chunks = pkg.grid_chunks(dest, off)
        kept = [i for i, ch in enumerate(chunks) if ch is not None]
        assert r == off[-1] and len(kept) == 2 * 8 * 3 + 1, len(kept)
        out = torch.empty(n ** 3 * 4, dtype=torch.uint8, device="cuda")
        assert pkg.grid_getslice(chunks, (n, n, n), (c, c, c), 4, (0, 0, 0), (n, n, n), out, fill=fill) == n ** 3 * 4
        assert torch.equal(out.view(torch.float32).view(n, n, n), src)


@pytest.mark.gpu
def test_grid_compress_other_device_gpu(pkg, cuda):
    """a CUDA src on another device than dest's is refused"""
    torch = cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    src = torch.zeros(64, 64, dtype=torch.float32, device="cuda:1")
    dest = torch.empty(pkg.grid_bound((64, 64), (16, 16), 4), dtype=torch.uint8, device="cuda:0")
    assert pkg.grid_compress(src, (64, 64), (16, 16), 4, 5, 1, "lz4", dest)[0] == -1

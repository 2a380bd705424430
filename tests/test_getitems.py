"""blosc_b200_getitems / blosc_b200_frame_getitems: many item ranges in one call, each touched block decoded once.

Every result is checked against the concatenation of per-range blosc_getitem (frame_getitem) calls on the same library,
and, where oracle/_ref was built, against the reference's blosc_getitem on a chunk the reference wrote.  CPU: the
product's host code and kernels inside the SIMT emulator (tests/emu).  GPU: the same matrix through the CUDA library,
plus host / device pointer combinations, launch counts and the profiler's decode count."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

from datagen import bench_words, ci, compress, gen, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "compat", "*.cdata")))
ll = C.c_longlong
NEVER_SPLIT, FORWARD_COMPAT_SPLIT = 2, 4
# (codec, switch that makes the library write it)
CODECS = (("blosclz", None), ("lz4", None), ("lz4hc", None), ("snappy", "BLOSC_B200_SNAPPY"),
          ("zlib", "BLOSC_B200_ZLIB"), ("zstd", "BLOSC_B200_ZSTD"))
TYPESIZES = (1, 2, 4, 8, 3, 16)


def _bind(lib):
    lib.blosc_getitem.restype = C.c_int
    lib.blosc_b200_getitems.restype = ll
    lib.blosc_b200_getitems.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.blosc_b200_frame_getitem.restype = ll
    lib.blosc_b200_frame_getitem.argtypes = [C.c_void_p, sz, sz, sz, C.c_void_p]
    lib.blosc_b200_frame_getitems.restype = ll
    lib.blosc_b200_frame_getitems.argtypes = [C.c_void_p, sz, sz, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.blosc_b200_frame_compress.restype = ll
    lib.blosc_b200_frame_compress.argtypes = [ci, ci, sz, sz, C.c_void_p, C.c_void_p, sz, C.c_char_p, sz, sz, ci]
    lib.blosc_b200_frame_bound.restype = sz
    lib.blosc_b200_frame_bound.argtypes = [sz, sz, sz]
    lib.blosc_set_splitmode.argtypes = [ci]
    return lib


@pytest.fixture(scope="session")
def elib(tmp_path_factory):
    """the emulated library with the decode-launch counters of tests/emu/getitems_stage.cpp (which includes
    backend_emu.cpp whole), built into a temporary directory"""
    import subprocess
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("getitems_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "c-blosc_b200", "csrc", "blosc_b200.c"), "-o",
                    str(d / "host.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "getitems_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    path = str(d / "libgetitems_stage.so")
    subprocess.run(["g++", "-shared", "-o", path, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    lib = _bind(C.CDLL(path))
    lib.blosc_compress_ctx.restype = C.c_int
    lib.emu_last_decode_streams.restype = ci
    lib.emu_last_decode_blocks.restype = ci
    lib.emu_launches_with_gather.restype = ll
    return lib


def _ranges(nit, bs_items, ts, rng, k=14):
    """unsorted, overlapping, repeated, empty, single-item and whole-chunk ranges; some cross a block or a split
    boundary and one ends in the last (short) block"""
    out = [(0, 0), (nit // 2, 1), (0, nit), (max(bs_items - 3, 0), min(7, nit - max(bs_items - 3, 0))),
           (max(nit - 5, 0), min(5, nit)), (nit, 0)]
    split_items = max(bs_items // max(ts, 1), 1)                # a split boundary inside block 0 (split 1 starts there)
    if split_items + 2 <= nit:
        out.append((split_items - 2, 4))
    for _ in range(k):
        s = int(rng.integers(0, nit))
        out.append((s, int(rng.integers(0, min(nit - s, 2 * bs_items) + 1))))
    out.append(out[3])                                          # repeated
    out.append((out[-3][0], out[-3][1] // 2))                   # overlaps a random one
    order = rng.permutation(len(out))
    return [out[i] for i in order]


def _per_range(lib, src, ranges, ts, fn="blosc_getitem"):
    parts = []
    for s, n in ranges:
        buf = np.zeros(n * ts + 1, np.uint8)
        r = getattr(lib, fn)(ptr(src), ci(s), ci(n), ptr(buf))
        assert r == n * ts, (s, n, r)
        parts.append(buf[:n * ts])
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


def _getitems(lib, src, ranges, dest_len):
    st = np.array([s for s, _ in ranges], np.int32)
    nn = np.array([n for _, n in ranges], np.int32)
    out = np.full(dest_len + 8, 0xAA, np.uint8)
    r = lib.blosc_b200_getitems(ptr(src), len(ranges), st.ctypes.data, nn.ctypes.data, ptr(out))
    return r, out


def _check_chunk(lib, chunk, ts, nbytes, bs_items, seed, ref=None, refchunk=None, k=14):
    rng = np.random.default_rng(seed)
    ranges = _ranges(nbytes // ts, bs_items, ts, rng, k)
    want = _per_range(lib, chunk, ranges, ts)
    r, out = _getitems(lib, chunk, ranges, len(want))
    assert r == len(want), (r, len(want))
    assert (out[:r] == want).all() and (out[r:] == 0xAA).all()
    if ref is not None:
        assert (_per_range(ref, refchunk, ranges, ts) == want).all()
    return ranges


def _compress(lib, comp, clevel, shuf, ts, src, bs, monkeypatch, switch):
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
def test_getitems_equals_getitem_emu(elib, ref_if_built, monkeypatch, comp, switch, shuf):
    n = 65536 + 4816              # split: blocks of at least 64 KiB (blosc.c:1050); unsplit: 8 KiB; a short last one
    for i, ts in enumerate(TYPESIZES):
        src = gen("mixed" if i % 2 else "i32", n - n % ts, seed=ts)
        for split in (FORWARD_COMPAT_SPLIT, NEVER_SPLIT):
            elib.blosc_set_splitmode(split)
            try:
                chunk = _compress(elib, comp, 5, shuf, ts, src, 8192, monkeypatch, switch)
            finally:
                elib.blosc_set_splitmode(FORWARD_COMPAT_SPLIT)
            bs = int(chunk[8:12].view(np.int32)[0])
            refchunk = None
            if ref_if_built is not None and comp in ("blosclz", "lz4", "lz4hc") and split == FORWARD_COMPAT_SPLIT:
                r, rc = compress(ref_if_built, "blosc_compress_ctx", 5, shuf, ts, src, len(src) + 16, comp, 8192)
                refchunk = rc[:r].copy()
            _check_chunk(elib, chunk, ts, len(src), bs // ts, seed=ts * 7 + shuf, ref=ref_if_built if refchunk is not None
                         else None, refchunk=refchunk, k=6)


def test_getitems_memcpyed_emu(elib):
    for ts, n, clevel in ((4, 100, 5), (4, 40000, 0), (3, 999, 0), (1, 127, 9)):
        src = gen("rand", n, seed=n)
        r, c = compress(elib, "blosc_compress_ctx", clevel, 1, ts, src, n + 16, "lz4")
        assert r == n + 16 and c[2] & 0x2                        # BLOSC_MEMCPYED
        for dev in (0, 1):
            elib.emu_set_all_device(dev)
            try:
                _check_chunk(elib, c[:r].copy(), ts, n, max(n // ts // 3, 1), seed=n + dev)
            finally:
                elib.emu_set_all_device(0)


@pytest.mark.parametrize("dev", [0, 1])
def test_getitems_device_pointers_emu(elib, dev):
    """dev=1: the emulated backend treats every pointer as device memory (no staging, the gather writes dest)"""
    src = bench_words(70000)
    c = compress(elib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4", 16384)[1]
    elib.emu_set_all_device(dev)
    try:
        _check_chunk(elib, c, 4, len(src), 4096, seed=11)
    finally:
        elib.emu_set_all_device(0)


def test_getitems_one_pass_emu(elib):
    """One decode, one unfilter and one gather launch per call whatever the number of ranges, and the decode covers
    the touched blocks times their splits, not the ranges"""
    src = bench_words(8 * 65536 + 1000)
    r, c = compress(elib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4", 16384)
    assert r > 0 and not c[2] & 0x10 and int(c[8:12].view(np.int32)[0]) == 65536   # 4 streams per full block
    nit = len(src) // 4
    counts = []
    for ranges, blocks in (([(20000, 64)], 1),
                           ([(16384 * b + 7, 64) for b in (1, 3, 3, 1, 5)] * 3, 3),
                           ([(int(s), 64) for s in np.random.default_rng(1).integers(0, nit - 64, 4096)], 9)):
        before = elib.emu_launches_with_gather()
        got, out = _getitems(elib, c, ranges, 64 * 4 * len(ranges))
        counts.append(elib.emu_launches_with_gather() - before)
        assert got == 64 * 4 * len(ranges)
        want = np.concatenate([src[4 * s:4 * (s + n)] for s, n in ranges])
        assert (out[:got] == want).all()
        assert elib.emu_last_decode_blocks() == blocks
        assert elib.emu_last_decode_streams() == 4 * blocks - (1 if blocks == 9 else 0) * 3   # the short block: 1 stream
    assert counts == [3, 3, 3]


def test_getitems_rejects_emu(elib):
    src = gen("i32", 40000)
    elib.blosc_set_splitmode(NEVER_SPLIT)                        # blocks of 8 KiB: 2048 items, 5 of them
    try:
        c = compress(elib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4", 8192)[1]
    finally:
        elib.blosc_set_splitmode(FORWARD_COMPAT_SPLIT)
    assert int(c[8:12].view(np.int32)[0]) == 8192
    nit = 10000
    good = [(0, 10), (500, 20)]
    for bad, code in (((-1, 5), -1), ((nit + 1, 0), -1), ((nit - 2, 5), -1), ((10, -20), -1)):
        for where in (0, 1, 2):
            ranges = good[:where] + [bad] + good[where:]
            assert elib.blosc_getitem(ptr(c), ci(bad[0]), ci(bad[1]), ptr(np.zeros(64, np.uint8))) == code
            r, out = _getitems(elib, c, ranges, 256)
            assert r == code and (out == 0xAA).all(), (bad, where, r)
    assert _getitems(elib, c, [], 16)[0] == 0
    for patch, code in ((lambda h: h.__setitem__(0, 3), -9), (lambda h: h.__setitem__(1, 9), -9),
                        (lambda h: h[8:12].view(np.int32).__setitem__(0, 0), -1)):
        h = c.copy()
        patch(h)
        assert elib.blosc_getitem(ptr(h), ci(0), ci(4), ptr(np.zeros(64, np.uint8))) == code
        r, out = _getitems(elib, h, good, 256)
        assert r == code and (out == 0xAA).all()
    # a damaged bstarts entry: refused when a range touches that block, not read when none does
    h = c.copy()
    h[16 + 4 * 2:16 + 4 * 3].view(np.int32)[0] = 0x7fff0000
    for dev in (0, 1):
        elib.emu_set_all_device(dev)
        try:
            r, out = _getitems(elib, h, good + [(2 * 2048 + 5, 3)], 256)
            assert r == elib.blosc_getitem(ptr(h), ci(2 * 2048 + 5), ci(3), ptr(np.zeros(64, np.uint8))) < 0
            assert (out == 0xAA).all()
            assert _check_chunk(elib, h, 4, 2 * 8192, 2048, seed=5) is not None        # blocks 0 and 1 only
        finally:
            elib.emu_set_all_device(0)


def _frame(lib, src, ts, chunksize, dev=False):
    fb = lib.blosc_b200_frame_bound(len(src), ts, chunksize)
    frame = np.zeros(fb, np.uint8)
    r = lib.blosc_b200_frame_compress(5, 1, ts, len(src), ptr(src), ptr(frame), fb, b"lz4", 4096, chunksize, 1)
    assert r > 0
    return frame[:r].copy(), r


def _frame_ranges(nit, per_chunk, rng):
    out = [(per_chunk - 3, 10), (0, nit), (nit - 1, 1), (5, 0), (2 * per_chunk - 1, per_chunk + 2)]
    for _ in range(10):
        s = int(rng.integers(0, nit))
        out.append((s, int(rng.integers(0, min(nit - s, per_chunk + 500) + 1))))
    return [out[i] for i in rng.permutation(len(out))]


def _check_frame(lib, frame, fb, ts, nit, per_chunk, seed):
    ranges = _frame_ranges(nit, per_chunk, np.random.default_rng(seed))
    parts = []
    for s, n in ranges:
        buf = np.zeros(n * ts + 1, np.uint8)
        assert lib.blosc_b200_frame_getitem(ptr(frame), fb, s, n, ptr(buf)) == n * ts
        parts.append(buf[:n * ts])
    want = np.concatenate(parts)
    st = np.array([s for s, _ in ranges], np.uint64)
    nn = np.array([n for _, n in ranges], np.uint64)
    out = np.full(len(want) + 8, 0xAA, np.uint8)
    r = lib.blosc_b200_frame_getitems(ptr(frame), fb, len(ranges), st.ctypes.data, nn.ctypes.data, ptr(out))
    assert r == len(want) and (out[:r] == want).all() and (out[r:] == 0xAA).all()
    bad = st.copy()
    bad[len(bad) // 2] = nit + 1
    out[:] = 0xAA
    assert lib.blosc_b200_frame_getitems(ptr(frame), fb, len(ranges), bad.ctypes.data, nn.ctypes.data, ptr(out)) == -1
    assert (out == 0xAA).all()


@pytest.mark.parametrize("dev", [0, 1])
def test_frame_getitems_emu(elib, dev):
    src = gen("i32", 3 * 24000 + 400)
    frame, fb = _frame(elib, src, 4, 24000)
    elib.emu_set_all_device(dev)
    try:
        _check_frame(elib, frame, fb, 4, len(src) // 4, 6000, seed=dev)
    finally:
        elib.emu_set_all_device(0)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the CUDA library
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def glib(pkg):
    return _bind(pkg.lib)


@pytest.mark.gpu
@pytest.mark.parametrize("comp,switch", CODECS)
@pytest.mark.parametrize("shuf", [0, 1, 2])
def test_getitems_equals_getitem_gpu(glib, cuda, ref_if_built, monkeypatch, comp, switch, shuf):
    n = 3 * 262144 + 4800                                         # default blocksizes: several blocks, a short one
    for i, ts in enumerate(TYPESIZES):
        src = (gen("mixed", n, seed=ts) if i % 2 else bench_words(n))[:n - n % ts].copy()
        for split in (FORWARD_COMPAT_SPLIT, NEVER_SPLIT):
            for bs in (0, 16384):
                glib.blosc_set_splitmode(split)
                try:
                    chunk = _compress(glib, comp, 5, shuf, ts, src, bs, monkeypatch, switch)
                finally:
                    glib.blosc_set_splitmode(FORWARD_COMPAT_SPLIT)
                cbs = int(chunk[8:12].view(np.int32)[0])
                refchunk = None
                if ref_if_built is not None and comp in ("blosclz", "lz4", "lz4hc") and split == FORWARD_COMPAT_SPLIT:
                    r, rc = compress(ref_if_built, "blosc_compress_ctx", 5, shuf, ts, src, len(src) + 16, comp, bs)
                    refchunk = rc[:r].copy()
                _check_chunk(glib, chunk, ts, len(src), cbs // ts, seed=ts + 100 * shuf + bs,
                             ref=ref_if_built if refchunk is not None else None, refchunk=refchunk)


@pytest.mark.gpu
def test_getitems_goldens_gpu(glib, cuda, monkeypatch):
    monkeypatch.setenv("BLOSC_B200_SNAPPY", "1")
    want = np.arange(1000000, dtype=np.int32).view(np.uint8)
    for f in GOLDENS:
        chunk = np.fromfile(f, np.uint8)
        ranges = _check_chunk(glib, chunk, 4, 4000000, int(chunk[8:12].view(np.int32)[0]) // 4, seed=len(f))
        r, out = _getitems(glib, chunk, ranges, sum(n for _, n in ranges) * 4)
        assert (out[:r] == np.concatenate([want[4 * s:4 * (s + n)] for s, n in ranges])).all(), f


@pytest.mark.gpu
def test_getitems_memcpyed_gpu(glib, cuda):
    for ts, n, clevel in ((4, 100, 5), (4, 400000, 0), (3, 999, 0)):
        src = gen("rand", n, seed=n)
        r, c = compress(glib, "blosc_compress_ctx", clevel, 1, ts, src, n + 16, "lz4")
        assert r == n + 16 and c[2] & 0x2
        _check_chunk(glib, c[:r].copy(), ts, n, max(n // ts // 3, 1), seed=n)


@pytest.mark.gpu
@pytest.mark.parametrize("clevel", [0, 5])
def test_getitems_pointer_kinds_gpu(pkg, cuda, clevel):
    """src / dest in every combination of host and device memory"""
    torch = cuda
    src = bench_words(3 << 20)
    r, c = compress(pkg.lib, "blosc_compress_ctx", clevel, 1, 4, src, len(src) + 16, "lz4")
    chunk = c[:r].copy()
    rng = np.random.default_rng(clevel)
    nit = len(src) // 4
    ranges = _ranges(nit, 65536, 4, rng, k=300)
    want = np.concatenate([src[4 * s:4 * (s + n)] for s, n in ranges])
    st = [s for s, _ in ranges]
    nn = [n for _, n in ranges]
    for src_dev in (False, True):
        s_buf = torch.from_numpy(chunk).cuda() if src_dev else chunk
        for dest_dev in (False, True):
            d_buf = torch.full((len(want) + 8,), 0xAA, dtype=torch.uint8, device="cuda") if dest_dev else \
                np.full(len(want) + 8, 0xAA, np.uint8)
            assert pkg.getitems(s_buf, st, np.array(nn), d_buf) == len(want)
            got = d_buf.cpu().numpy() if dest_dev else d_buf
            assert (got[:len(want)] == want).all() and (got[len(want):] == 0xAA).all(), (src_dev, dest_dev)


@pytest.mark.gpu
def test_getitems_one_pass_gpu(pkg, cuda):
    src = bench_words(32 << 20)
    r, c = compress(pkg.lib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4")
    chunk = cuda.from_numpy(c[:r].copy()).cuda()
    nit = len(src) // 4
    grown = []
    pkg.set_profiling(True)
    try:
        for k in (1, 16, 4096):
            st = np.random.default_rng(k).integers(0, nit - 64, k)
            out = cuda.zeros(64 * 4 * k, dtype=cuda.uint8, device="cuda")
            pkg.prof_reset()
            before = pkg.launch_count()
            assert pkg.getitems(chunk, st, np.full(k, 64), out) == 64 * 4 * k
            grown.append(pkg.launch_count() - before)
            prof = pkg.prof_get()
            assert prof["decode"][1] == 1 and prof["gather"][1] == 1 and prof["unfilter"][1] == 1, prof
            want = np.concatenate([src[4 * s:4 * (s + 64)] for s in st])
            assert (out.cpu().numpy() == want).all()
    finally:
        pkg.set_profiling(False)
    assert grown == [3, 3, 3]


@pytest.mark.gpu
def test_getitems_rejects_gpu(glib, cuda):
    torch = cuda
    src = gen("i32", 400000)
    c = compress(glib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4", 16384)[1]
    assert int(c[8:12].view(np.int32)[0]) == 65536              # 16384 items per block
    nit = 100000
    good = [(0, 10), (500, 20)]
    for bad in ((-1, 5), (nit + 1, 0), (nit - 2, 5), (10, -20)):
        for where in (0, 2):
            r, out = _getitems(glib, c, good[:where] + [bad] + good[where:], 256)
            assert r == -1 and (out == 0xAA).all()
    h = c.copy()
    h[0] = 3
    assert _getitems(glib, h, good, 256)[0] == -9
    h = c.copy()
    h[16 + 4 * 2:16 + 4 * 3].view(np.int32)[0] = 0x7fff0000      # block 2's bstarts entry
    for src_dev in (False, True):
        s_buf = torch.from_numpy(h).cuda() if src_dev else h
        out = torch.full((256,), 0xAA, dtype=torch.uint8, device="cuda")
        one = glib.blosc_getitem(C.c_void_p(s_buf.data_ptr() if src_dev else h.ctypes.data), 2 * 16384 + 5, 3,
                                 C.c_void_p(out.data_ptr()))
        assert one < 0
        st = np.array([0, 2 * 16384 + 5], np.int32)
        nn = np.array([10, 3], np.int32)
        r = glib.blosc_b200_getitems(s_buf.data_ptr() if src_dev else h.ctypes.data, 2, st.ctypes.data, nn.ctypes.data,
                                     out.data_ptr())
        assert r == one and (out.cpu().numpy() == 0xAA).all(), (src_dev, r, one)
        st = np.array([0, 16384 + 5], np.int32)                   # blocks 0 and 1 only: block 2 is not read
        r = glib.blosc_b200_getitems(s_buf.data_ptr() if src_dev else h.ctypes.data, 2, st.ctypes.data, nn.ctypes.data,
                                     out.data_ptr())
        assert r == 52 and (out[:52].cpu().numpy() == np.concatenate([src[:40], src[4 * 16389:4 * 16392]])).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dev", [False, True])
def test_frame_getitems_gpu(glib, pkg, cuda, dev):
    src = bench_words(3 * 1000000 + 4000)
    frame, fb = _frame(glib, src, 4, 1000000)
    if dev:
        d_frame = cuda.from_numpy(frame).cuda()
        ranges = _frame_ranges(len(src) // 4, 250000, np.random.default_rng(3))
        want = np.concatenate([src[4 * s:4 * (s + n)] for s, n in ranges])
        out = cuda.full((len(want),), 0xAA, dtype=cuda.uint8, device="cuda")
        assert pkg.frame_getitems(d_frame, fb, [s for s, _ in ranges], [n for _, n in ranges], out) == len(want)
        assert (out.cpu().numpy() == want).all()
        h_out = np.zeros(len(want), np.uint8)
        assert pkg.frame_getitems(d_frame, fb, [s for s, _ in ranges], [n for _, n in ranges], h_out) == len(want)
        assert (h_out == want).all()
    else:
        _check_frame(glib, frame, fb, 4, len(src) // 4, 250000, seed=4)

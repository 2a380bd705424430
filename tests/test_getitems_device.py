"""blosc_b200_getitems with starts / nitems in device memory: the read is planned on the GPU (dev_chunk.cuh
plan_check_kernel / plan_scan_kernel) and must give exactly what the host plan gives for the same lists in host memory:
the return value, the stderr message, the bytes in dest, and an untouched dest on failure.

CPU: the emulated library runs each request twice, in all-device mode (every pointer is device memory, so the GPU plan
runs) and in all-host mode (the host plan runs).  GPU: the CUDA library with every mix of chunk, dest and list memory,
2^20 ranges on a 256 MiB chunk, launch counts, lists on another device, and frames."""
import ctypes as C

import numpy as np
import pytest

from datagen import bench_words, ci, compress, gen, ptr, sz

ll = C.c_longlong
NEVER_SPLIT, FORWARD_COMPAT_SPLIT = 2, 4
CODECS = (("blosclz", None), ("lz4", None), ("lz4hc", None), ("snappy", "BLOSC_B200_SNAPPY"),
          ("zlib", "BLOSC_B200_ZLIB"), ("zstd", "BLOSC_B200_ZSTD"))
TYPESIZES = (1, 2, 4, 8, 3, 16)
TILE = 2048                                          # PLAN_TILE (b2_args.h): items per CTA of a plan scan


def _bind(lib):
    lib.blosc_getitem.restype = C.c_int
    lib.blosc_b200_getitems.restype = ll
    lib.blosc_b200_getitems.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.blosc_b200_frame_getitems.restype = ll
    lib.blosc_b200_frame_getitems.argtypes = [C.c_void_p, sz, sz, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.blosc_b200_frame_compress.restype = ll
    lib.blosc_b200_frame_compress.argtypes = [ci, ci, sz, sz, C.c_void_p, C.c_void_p, sz, C.c_char_p, sz, sz, ci]
    lib.blosc_b200_frame_bound.restype = sz
    lib.blosc_b200_frame_bound.argtypes = [sz, sz, sz]
    lib.blosc_set_splitmode.argtypes = [ci]
    return lib


@pytest.fixture(scope="module")
def dlib(emu):
    """the emulated library (tests/emu), with getitems' signatures"""
    return _bind(emu)


def _rand_ranges(nit, span, k, rng, empty=0.3):
    """k random ranges of up to `span` items; a share of them empty (nitems 0, or a negative count that stops at or
    after 0), some starting at the very end"""
    st = rng.integers(0, nit + 1, k)
    nn = rng.integers(0, span + 1, k)
    nn = np.minimum(nn, nit - st)
    e = rng.random(k) < empty
    nn[e] = 0
    neg = e & (rng.random(k) < 0.3)
    nn[neg] = -rng.integers(0, 3, int(neg.sum())) * (st[neg] > 3)
    return st.astype(np.int32), nn.astype(np.int32)


def _want(src, ts, st, nn):
    parts = [src[ts * s:ts * (s + n)] for s, n in zip(st.tolist(), nn.tolist()) if n > 0]
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


def _call(lib, chunk, st, nn, dest_len, capfd):
    out = np.full(dest_len + 16, 0xAA, np.uint8)
    capfd.readouterr()
    r = lib.blosc_b200_getitems(ptr(chunk), len(st), st.ctypes.data, nn.ctypes.data, ptr(out))
    return r, out, capfd.readouterr().err


def _both(lib, chunk, st, nn, dest_len, capfd):
    """the same request through the GPU plan (all-device) and the host plan (all-host): equal in every respect"""
    lib.emu_set_all_device(1)
    try:
        dev = _call(lib, chunk, st, nn, dest_len, capfd)
    finally:
        lib.emu_set_all_device(0)
    host = _call(lib, chunk, st, nn, dest_len, capfd)
    assert dev[0] == host[0] and dev[2] == host[2], (dev[0], host[0], dev[2], host[2])
    assert (dev[1] == host[1]).all()
    return dev


def _check(lib, chunk, src, ts, st, nn, capfd):
    want = _want(src, ts, st, nn)
    r, out, err = _both(lib, chunk, st, nn, len(want), capfd)
    assert r == len(want) and err == ""
    assert (out[:r] == want).all() and (out[r:] == 0xAA).all()


def _compress(lib, comp, clevel, shuf, ts, src, bs, monkeypatch, switch, split=FORWARD_COMPAT_SPLIT):
    if switch:
        monkeypatch.setenv(switch, "1")
    lib.blosc_set_splitmode(split)
    try:
        r, c = compress(lib, "blosc_compress_ctx", clevel, shuf, ts, src, len(src) + 16, comp, bs)
    finally:
        lib.blosc_set_splitmode(FORWARD_COMPAT_SPLIT)
    assert r > 0, (comp, ts, shuf, r)
    return c[:r].copy()


# ---------------------------------------------------------------------------------------------------------------
# CPU: the emulator
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("comp,switch", CODECS)
def test_plans_agree_emu(dlib, monkeypatch, capfd, comp, switch):
    n = 65536 + 4816                         # split: blocks of 64 KiB; unsplit: 8 KiB; and a short last block
    for i, ts in enumerate(TYPESIZES):
        src = gen("mixed" if i % 2 else "i32", n - n % ts, seed=ts)
        for split in (FORWARD_COMPAT_SPLIT, NEVER_SPLIT):
            chunk = _compress(dlib, comp, 5, i % 3, ts, src, 8192, monkeypatch, switch, split)
            nit = len(src) // ts
            bs_items = int(chunk[8:12].view(np.int32)[0]) // ts
            st, nn = _rand_ranges(nit, 2 * bs_items, 40, np.random.default_rng(ts * 10 + split))
            st[:3], nn[:3] = (0, nit - 5, nit // 2), (nit, 5, 1)    # the whole chunk, the short last block, one item
            _check(dlib, chunk, src, ts, st, nn, capfd)


def test_plans_agree_memcpyed_emu(dlib, capfd):
    for ts, n, clevel in ((4, 100, 5), (4, 40000, 0), (3, 999, 0), (1, 127, 9), (16, 40000, 0)):
        src = gen("rand", n - n % ts, seed=n)
        r, c = compress(dlib, "blosc_compress_ctx", clevel, 1, ts, src, len(src) + 16, "lz4")
        assert r == len(src) + 16 and c[2] & 0x2                        # BLOSC_MEMCPYED
        st, nn = _rand_ranges(len(src) // ts, 300, 25, np.random.default_rng(n))
        _check(dlib, c[:r].copy(), src, ts, st, nn, capfd)


@pytest.mark.parametrize("k", [1, TILE - 1, TILE, TILE + 1, 5 * TILE + 37])
def test_plan_tile_boundaries_emu(dlib, capfd, k):
    """range counts on both sides of a scan tile, and enough for several tiles and look-back steps"""
    src = bench_words(200000)
    c = compress(dlib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4", 8192)[1]
    st, nn = _rand_ranges(len(src) // 4, 40, k, np.random.default_rng(k))
    _check(dlib, c, src, 4, st, nn, capfd)


def test_plan_many_blocks_emu(dlib, capfd):
    """more blocks than one scan tile: the coverage and slot scans span several tiles"""
    src = bench_words(2 * TILE * 128 + 4 * 1000 + 52)
    c = compress(dlib, "blosc_compress_ctx", 1, 0, 4, src, len(src) + 16, "lz4", 128)[1]
    nblocks = -(-len(src) // int(c[8:12].view(np.int32)[0]))
    assert nblocks > 2 * TILE, nblocks
    nit = len(src) // 4
    rng = np.random.default_rng(3)
    for st, nn in (_rand_ranges(nit, 100, 300, rng), (np.array([0], np.int32), np.array([nit], np.int32)),
                   (np.array([nit - 1, 5, 40000, 40000], np.int32), np.array([1, 3, 33, 33], np.int32))):
        _check(dlib, c, src, 4, st, nn, capfd)


def test_plan_empty_ranges_emu(dlib, capfd):
    """empty entries leading, interleaved and trailing stay in the GPU plan's table and copy nothing"""
    src = bench_words(70000)
    c = compress(dlib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4", 16384)[1]
    nit = len(src) // 4
    for pattern in ([(0, 0), (7, 0), (10, 5), (nit, 0), (3, 9)],
                    [(10, 5), (12, -2), (100, 0), (200, 300), (200, 0), (nit, 0)],
                    [(0, 0), (nit, 0), (5, -5)],
                    [(0, 0)] * 3 + [(4096 - 3, 7)] + [(9, 0)] * 4 + [(nit - 2, 2)] + [(nit, 0)] * 3):
        st = np.array([s for s, _ in pattern], np.int32)
        nn = np.array([n for _, n in pattern], np.int32)
        _check(dlib, c, src, 4, st, nn, capfd)


def test_plan_rejects_emu(dlib, capfd):
    """every reject of blosc_getitem, alone, after valid ranges and among several bad ones (the first decides): the
    same code, the same message and an untouched dest"""
    src = gen("i32", 40000)
    c = compress(dlib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4", 8192)[1]
    nit = 10000
    good = [(0, 10), (500, 20), (9000, 0)]
    bads = [(-1, 5), (nit + 1, 0), (nit - 2, 5), (2, 0x7fffffff), (0x7ffffff0, 0x20), (10, -20)]
    cases = [[b] for b in bads] + [good + [b] for b in bads] + [good[:1] + [b] + good[1:] for b in bads]
    cases += [good + [bads[2], bads[0]], [bads[3]] + good + [bads[1]], good + [bads[5], bads[4], bads[0]]]
    for ranges in cases:
        st = np.array([s for s, _ in ranges], np.int32)
        nn = np.array([n for _, n in ranges], np.int32)
        r, out, err = _both(dlib, c, st, nn, 256, capfd)
        assert r == -1 and (out == 0xAA).all() and "out of bounds" in err, (ranges, r, err)
    # header errors come before the lists are read
    for patch, code in ((lambda h: h.__setitem__(0, 3), -9), (lambda h: h[8:12].view(np.int32).__setitem__(0, 0), -1)):
        h = c.copy()
        patch(h)
        st = np.array([0, -1], np.int32)
        nn = np.array([4, 4], np.int32)
        r, out, err = _both(dlib, h, st, nn, 64, capfd)
        assert r == code and (out == 0xAA).all() and err == ""
    # nranges == 0 reads neither list
    for dev in (0, 1):
        dlib.emu_set_all_device(dev)
        try:
            out = np.full(16, 0xAA, np.uint8)
            assert dlib.blosc_b200_getitems(ptr(c), 0, None, None, ptr(out)) == 0 and (out == 0xAA).all()
        finally:
            dlib.emu_set_all_device(0)


def test_plan_damaged_stream_emu(dlib, capfd):
    """a touched block that fails to decode gives the host plan's code and leaves dest untouched; one no range
    touches is never read"""
    src = gen("i32", 40000)
    dlib.blosc_set_splitmode(NEVER_SPLIT)
    try:
        c = compress(dlib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4", 8192)[1]
    finally:
        dlib.blosc_set_splitmode(FORWARD_COMPAT_SPLIT)
    for damage in ("bstart", "payload"):
        h = c.copy()
        b2 = int(h[16 + 8:16 + 12].view(np.int32)[0])
        if damage == "bstart":
            h[16 + 8:16 + 12].view(np.int32)[0] = 0x7fff0000
        else:
            h[b2:b2 + 4].view(np.int32)[0] = 0x7fffffff                # the first stream's size prefix of block 2
        st = np.array([0, 2 * 2048 + 5, 100], np.int32)
        nn = np.array([10, 3, 0], np.int32)
        r, out, err = _both(dlib, h, st, nn, 256, capfd)
        assert r < 0 and (out == 0xAA).all(), (damage, r)
        _check(dlib, h, src, 4, np.array([0, 2048 + 5], np.int32), np.array([10, 3], np.int32), capfd)


def test_frame_getitems_device_lists_emu(dlib):
    src = gen("i32", 3 * 24000 + 400)
    fb = dlib.blosc_b200_frame_bound(len(src), 4, 24000)
    frame = np.zeros(fb, np.uint8)
    fb = dlib.blosc_b200_frame_compress(5, 1, 4, len(src), ptr(src), ptr(frame), fb, b"lz4", 4096, 24000, 1)
    assert fb > 0
    nit = len(src) // 4
    st = np.array([5997, 0, nit - 1, 5, 11999, 100], np.uint64)
    nn = np.array([10, nit, 1, 0, 6002, 7], np.uint64)
    want = np.concatenate([src[4 * s:4 * (s + n)] for s, n in zip(st.tolist(), nn.tolist())])
    for dev in (1, 0):
        dlib.emu_set_all_device(dev)
        try:
            out = np.full(len(want) + 8, 0xAA, np.uint8)
            r = dlib.blosc_b200_frame_getitems(ptr(frame), fb, len(st), st.ctypes.data, nn.ctypes.data, ptr(out))
            assert r == len(want) and (out[:r] == want).all() and (out[r:] == 0xAA).all()
            bad = st.copy()
            bad[2] = nit + 1
            out[:] = 0xAA
            assert dlib.blosc_b200_frame_getitems(ptr(frame), fb, len(st), bad.ctypes.data, nn.ctypes.data, ptr(out)) == -1
            assert (out == 0xAA).all()
        finally:
            dlib.emu_set_all_device(0)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the CUDA library
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def glib(pkg):
    return _bind(pkg.lib)


def _gpu_matrix(pkg, torch, chunk, src, ts, st, nn, capfd=None):
    """every mix of chunk (device, pinned, pageable), dest (device, host) and lists (device, host, one of each): for
    each chunk, every call equals the host-list call, and valid requests the concatenation of the ranges; returns the
    device chunk's result"""
    want = _want(src, ts, st, nn)
    chunks = {"device": torch.from_numpy(chunk).cuda(), "pinned": torch.from_numpy(chunk).pin_memory(),
              "pageable": chunk}
    d_st, d_nn = torch.from_numpy(st).cuda(), torch.from_numpy(nn).cuda()
    lists = {"host": (st, nn), "device": (d_st, d_nn), "starts": (d_st, nn), "nitems": (st, d_nn)}
    results = []
    for cname, cbuf in chunks.items():
        first = None
        for dest_dev in (True, False):
            for lname, (a, b) in lists.items():
                if dest_dev:
                    out = torch.full((len(want) + 16,), 0xAA, dtype=torch.uint8, device="cuda")
                else:
                    out = np.full(len(want) + 16, 0xAA, np.uint8)
                if capfd is not None:
                    capfd.readouterr()
                r = pkg.getitems(cbuf, a, b, out)
                err = capfd.readouterr().err if capfd is not None else ""
                got = out.cpu().numpy() if dest_dev else out
                res = (r, err, got.tobytes())
                if first is None:
                    first = res
                assert res == first, (cname, dest_dev, lname, r, first[0], err, first[1])
        r, err, got = first
        got = np.frombuffer(got, np.uint8)
        if r >= 0:
            assert r == len(want) and (got[:r] == want).all() and (got[r:] == 0xAA).all(), cname
        results.append((r, err, got))
    return results[0]


@pytest.mark.gpu
@pytest.mark.parametrize("comp,switch", CODECS)
def test_plans_agree_gpu(pkg, glib, cuda, monkeypatch, comp, switch):
    n = 3 * 262144 + 4800                                         # default blocksizes: several blocks, a short one
    for i, ts in enumerate(TYPESIZES):
        src = (gen("mixed", n, seed=ts) if i % 2 else bench_words(n))[:n - n % ts].copy()
        for split in (FORWARD_COMPAT_SPLIT, NEVER_SPLIT):
            chunk = _compress(glib, comp, 5, i % 3, ts, src, 0, monkeypatch, switch, split)
            nit = len(src) // ts
            bs_items = int(chunk[8:12].view(np.int32)[0]) // ts
            st, nn = _rand_ranges(nit, 2 * bs_items, 60, np.random.default_rng(ts + split))
            st[:2], nn[:2] = (0, nit - 3), (nit, 3)
            _gpu_matrix(pkg, cuda, chunk, src, ts, st, nn)


@pytest.mark.gpu
def test_plans_agree_memcpyed_gpu(pkg, glib, cuda):
    for ts, n in ((4, 100), (4, 400000), (3, 999), (16, 1 << 20)):
        src = gen("rand", n - n % ts, seed=n)
        r, c = compress(glib, "blosc_compress_ctx", 0, 1, ts, src, len(src) + 16, "lz4")
        assert r == len(src) + 16 and c[2] & 0x2
        st, nn = _rand_ranges(len(src) // ts, 500, 50, np.random.default_rng(n))
        _gpu_matrix(pkg, cuda, c[:r].copy(), src, ts, st, nn)


@pytest.mark.gpu
def test_plan_rejects_gpu(pkg, glib, cuda, capfd):
    src = gen("i32", 400000)
    c = compress(glib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4", 16384)[1]
    c = c[:int(c[12:16].view(np.int32)[0])].copy()
    nit = 100000
    good = [(0, 10), (500, 20), (9000, 0)]
    bads = [(-1, 5), (nit + 1, 0), (nit - 2, 5), (2, 0x7fffffff), (0x7ffffff0, 0x20), (10, -20)]
    for ranges in [[b] for b in bads] + [good + [b] for b in bads] + [good + [bads[2], bads[0]]]:
        st = np.array([s for s, _ in ranges], np.int32)
        nn = np.array([n for _, n in ranges], np.int32)
        r, err, got = _gpu_matrix(pkg, cuda, c, src, 4, st, nn, capfd)
        assert r == -1 and "out of bounds" in err and (got == 0xAA).all(), (ranges, r, err)
    h = c.copy()
    h[16 + 8:16 + 12].view(np.int32)[0] = 0x7fff0000                # block 2's bstarts entry
    st = np.array([0, 2 * 16384 + 5], np.int32)
    nn = np.array([10, 3], np.int32)
    r, err, got = _gpu_matrix(pkg, cuda, h, src, 4, st, nn, capfd)
    assert r < 0 and (got == 0xAA).all()
    _gpu_matrix(pkg, cuda, h, src, 4, np.array([0, 16384 + 5], np.int32), nn, capfd)
    h = c.copy()
    h[0] = 3
    r, err, got = _gpu_matrix(pkg, cuda, h, src, 4, st, nn, capfd)
    assert r == -9 and (got == 0xAA).all()


@pytest.mark.gpu
def test_plan_million_ranges_gpu(pkg, glib, cuda):
    """2^20 random ranges, many of them empty, on a 256 MiB chunk against a full decompress and a torch index"""
    torch = cuda
    n = 256 << 20
    i = torch.arange(n // 4, dtype=torch.int32, device="cuda")
    d_src = (((i << 26) ^ (i << 18) ^ (i << 11) ^ (i << 3) ^ i) & ((1 << 19) - 1)).view(torch.uint8)
    d_chunk = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(5, 1, 4, n, d_src, d_chunk, n + 16, "lz4")
    assert cb > 0
    full = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert pkg.decompress_ctx(d_chunk, full, n) == n
    k = 1 << 20
    g = torch.Generator(device="cuda").manual_seed(7)
    st = torch.randint(0, n // 4 + 1, (k,), device="cuda", generator=g, dtype=torch.int64)
    nn = torch.randint(0, 65, (k,), device="cuda", generator=g, dtype=torch.int64)
    nn = torch.minimum(nn, n // 4 - st)
    nn[torch.rand(k, device="cuda", generator=g) < 0.4] = 0
    st, nn = st.to(torch.int32), nn.to(torch.int32)
    total = int(nn.sum()) * 4
    out = torch.full((total + 16,), 0xAA, dtype=torch.uint8, device="cuda")
    assert pkg.getitems(d_chunk, st, nn, out) == total
    idx = torch.repeat_interleave(st.long(), nn.long())
    idx += torch.arange(idx.numel(), device="cuda") - torch.repeat_interleave(torch.cumsum(nn.long(), 0) - nn.long(), nn.long())
    want = full.view(torch.int32)[idx].view(torch.uint8)
    assert torch.equal(out[:total], want) and bool((out[total:] == 0xAA).all())


@pytest.mark.gpu
def test_plan_launch_count_gpu(pkg, cuda):
    """a device-list call on a device chunk launches the same kernels whatever the number of ranges"""
    torch = cuda
    src = bench_words(32 << 20)
    r, c = compress(pkg.lib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4")
    chunk = torch.from_numpy(c[:r].copy()).cuda()
    nit = len(src) // 4
    grown = []
    pkg.set_profiling(True)
    try:
        for k in (1, 16, 4096, 65536):
            st = torch.from_numpy(np.random.default_rng(k).integers(0, nit - 64, k).astype(np.int32)).cuda()
            out = torch.zeros(64 * 4 * k, dtype=torch.uint8, device="cuda")
            pkg.prof_reset()
            before = pkg.launch_count()
            assert pkg.getitems(chunk, st, torch.full((k,), 64, dtype=torch.int32, device="cuda"), out) == 64 * 4 * k
            grown.append(pkg.launch_count() - before)
            prof = pkg.prof_get()
            assert prof["plan"][1] == 4 and prof["decode"][1] == 1 and prof["gather"][1] == 1, prof
            s = st.cpu().numpy()
            assert (out.cpu().numpy() == np.concatenate([src[4 * x:4 * (x + 64)] for x in s])).all()
    finally:
        pkg.set_profiling(False)
    assert grown == [7] * 4


@pytest.mark.gpu
def test_plan_dtypes_gpu(pkg, cuda):
    torch = cuda
    src = bench_words(1 << 20)
    r, c = compress(pkg.lib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4")
    chunk = torch.from_numpy(c[:r].copy()).cuda()
    out = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    for dt in (torch.int64, torch.int16, torch.float32):
        with pytest.raises(TypeError):
            pkg.getitems(chunk, torch.zeros(2, dtype=dt, device="cuda"), [1, 2], out)
    with pytest.raises(TypeError):
        pkg.frame_getitems(chunk, r, torch.zeros(2, dtype=torch.int32, device="cuda"), [1, 2], out)
    base = torch.arange(0, 400, dtype=torch.int32, device="cuda").reshape(20, 20)
    st = base[:, 3]                                               # not contiguous
    assert not st.is_contiguous()
    assert pkg.getitems(chunk, st, torch.full((20,), 2, dtype=torch.int32, device="cuda"), out) == 160
    want = np.concatenate([src[4 * x:4 * (x + 2)] for x in st.cpu().numpy()])
    assert (out[:160].cpu().numpy() == want).all()


@pytest.mark.gpu
def test_plan_wrong_device_gpu(pkg, cuda):
    torch = cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    src = bench_words(1 << 20)
    r, c = compress(pkg.lib, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "lz4")
    chunk = torch.from_numpy(c[:r].copy()).to("cuda:0")
    out = torch.full((64,), 0xAA, dtype=torch.uint8, device="cuda:0")
    st = torch.tensor([0, 5], dtype=torch.int32, device="cuda:1")
    nn = torch.tensor([2, 2], dtype=torch.int32, device="cuda:0")
    assert pkg.getitems(chunk, st, nn, out) == -1
    assert bool((out == 0xAA).all())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["int64", "uint64"])
def test_frame_getitems_device_lists_gpu(pkg, glib, cuda, dtype):
    torch = cuda
    src = bench_words(3 * 1000000 + 4000)
    fb = glib.blosc_b200_frame_bound(len(src), 4, 1000000)
    frame = np.zeros(fb, np.uint8)
    fb = glib.blosc_b200_frame_compress(5, 1, 4, len(src), ptr(src), ptr(frame), fb, b"lz4", 4096, 1000000, 1)
    assert fb > 0
    nit = len(src) // 4
    rng = np.random.default_rng(5)
    st = rng.integers(0, nit, 200)
    nn = np.minimum(rng.integers(0, 300000, 200), nit - st)
    st[:3], nn[:3] = (249990, 0, 2 * 250000 - 1), (20, nit, 250002)          # across chunk boundaries, everything
    nn[10:20] = 0
    want = np.concatenate([src[4 * s:4 * (s + n)] for s, n in zip(st.tolist(), nn.tolist())])
    tdt = getattr(torch, dtype)
    d_st = torch.from_numpy(st.astype(np.int64)).cuda().to(tdt)
    d_nn = torch.from_numpy(nn.astype(np.int64)).cuda().to(tdt)
    for f in (frame[:fb], torch.from_numpy(frame[:fb].copy()).cuda()):
        for a, b in ((d_st, d_nn), (d_st, nn), (st, d_nn), (st, nn)):
            out = torch.full((len(want) + 8,), 0xAA, dtype=torch.uint8, device="cuda")
            assert pkg.frame_getitems(f, fb, a, b, out) == len(want)
            got = out.cpu().numpy()
            assert (got[:len(want)] == want).all() and (got[len(want):] == 0xAA).all()
    bad = st.copy()
    bad[7] = nit + 1
    out = torch.full((len(want),), 0xAA, dtype=torch.uint8, device="cuda")
    assert pkg.frame_getitems(frame[:fb], fb, torch.from_numpy(bad.astype(np.int64)).cuda(), d_nn.to(torch.int64),
                              out) == -1
    assert bool((out == 0xAA).all())

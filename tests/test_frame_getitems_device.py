"""blosc_b200_frame_getitems with starts / nitems in device memory: the frame is planned on the GPU (dev_chunk.cuh
fplan_check_kernel, plan_scan_kernel, fplan_scatter_kernel) into one piece list per chunk, and each touched chunk is then
read by the chunk's GPU plan.  A call must give exactly what the host plan gives for the same lists in host memory: the
return value, the stderr message and the bytes in dest; valid requests must also equal the source slices.

CPU: the emulated library runs each request in all-device mode (frame, dest and lists count as device memory, so the
GPU plan runs) and in all-host mode (the host plan).  GPU: the CUDA library with every mix of frame, dest and list
memory, 2^20 ranges on a 1 GiB frame, launch counts, lists on another device and two threads at once."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from datagen import bench_words, ci, gen, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ll = C.c_longlong
CODECS = (("blosclz", None), ("lz4", None), ("lz4hc", None), ("snappy", "BLOSC_B200_SNAPPY"),
          ("zlib", "BLOSC_B200_ZLIB"), ("zstd", "BLOSC_B200_ZSTD"))
TYPESIZES = (1, 2, 3, 4, 8, 16)
TILE = 2048                                          # PLAN_TILE (b2_args.h): items per CTA of a plan scan
U64_MAX = (1 << 64) - 1
OOB = "`start`+`nitems` out of bounds"


def _bind(lib):
    lib.blosc_b200_frame_getitems.restype = ll
    lib.blosc_b200_frame_getitems.argtypes = [C.c_void_p, sz, sz, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.blosc_b200_frame_compress.restype = ll
    lib.blosc_b200_frame_compress.argtypes = [ci, ci, sz, sz, C.c_void_p, C.c_void_p, sz, C.c_char_p, sz, sz, ci]
    lib.blosc_b200_frame_bound.restype = sz
    lib.blosc_b200_frame_bound.argtypes = [sz, sz, sz]
    return lib


@pytest.fixture(scope="module")
def flib(emu):
    """the emulated library (tests/emu), with the frame calls' signatures"""
    return _bind(emu)


@pytest.fixture(scope="module")
def slib(tmp_path_factory):
    """the emulated library with the launch counters of tests/emu/fplan_stage.cpp, built into a temporary directory"""
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("fplan_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "c-blosc_b200", "csrc", "blosc_b200.c"), "-o",
                    str(d / "host.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "fplan_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    path = str(d / "libfplan_stage.so")
    subprocess.run(["g++", "-shared", "-o", path, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    return _bind(C.CDLL(path))


def _frame(lib, src, ts, shuf, comp, chunksize, bs, clevel=5):
    fb = lib.blosc_b200_frame_bound(len(src), ts, chunksize)
    frame = np.zeros(fb, np.uint8)
    r = lib.blosc_b200_frame_compress(clevel, shuf, ts, len(src), ptr(src), ptr(frame), fb, comp.encode(), bs,
                                      chunksize, 1)
    assert r > 0, (comp, ts, shuf, r)
    return frame[:r].copy()


def _ipc(frame, ts):
    """items per chunk"""
    return int(frame[24:28].view(np.uint32)[0]) // ts


def _chunks(frame):
    """(offset, header flags) of every chunk"""
    nc = int(frame[28:32].view(np.uint32)[0])
    return [(int(o), int(frame[int(o) + 2])) for o in frame[32:32 + 8 * nc].view(np.uint64)]


def _lists(ranges):
    return (np.array([s for s, _ in ranges], np.uint64), np.array([n for _, n in ranges], np.uint64))


def _want(src, ts, ranges):
    parts = [src[ts * s:ts * (s + n)] for s, n in ranges if n > 0]
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


def _touched(ranges, ipc):
    return {c for s, n in ranges if n > 0 for c in range(s // ipc, (s + n - 1) // ipc + 1)}


def _call(lib, frame, ranges, dest_len, capfd):
    st, nn = _lists(ranges)
    out = np.full(dest_len + 16, 0xAA, np.uint8)
    capfd.readouterr()
    r = lib.blosc_b200_frame_getitems(ptr(frame), len(frame), len(st), st.ctypes.data, nn.ctypes.data, ptr(out))
    return r, out, capfd.readouterr().err


def _both(lib, frame, ranges, dest_len, capfd, same_bytes=True):
    """the same request through the GPU plan (all-device) and the host plan (all-host): the same return value and
    message, and the same dest unless the call failed in a chunk; returns both results"""
    lib.emu_set_all_device(1)
    try:
        dev = _call(lib, frame, ranges, dest_len, capfd)
    finally:
        lib.emu_set_all_device(0)
    host = _call(lib, frame, ranges, dest_len, capfd)
    assert dev[0] == host[0] and dev[2] == host[2], (dev[0], host[0], dev[2], host[2])
    if same_bytes:
        assert (dev[1] == host[1]).all()
    return dev, host


def _check(lib, frame, src, ts, ranges, capfd):
    want = _want(src, ts, ranges)
    (r, out, err), _ = _both(lib, frame, ranges, len(want), capfd)
    assert r == len(want) and err == "", (r, len(want), err)
    assert (out[:r] == want).all() and (out[r:] == 0xAA).all()


def _ranges(nit, ipc, rng, k=12):
    """empty ranges (at 0, on a chunk boundary, at the end), the whole frame, ranges that start or end on a chunk
    boundary, ranges over many chunks, random ones, two repeated; in random order"""
    b1, b2 = ipc, 2 * ipc
    out = [(0, 0), (nit, 0), (b1, 0), (0, nit), (b1, ipc), (b2 - 7, 7), (b1 - 3, ipc + 6), (ipc // 2, nit - ipc),
           (nit - 1, 1), (b2, nit - b2)]
    for _ in range(k):
        s = int(rng.integers(0, nit + 1))
        out.append((s, int(rng.integers(0, min(nit - s, 3 * ipc) + 1))))
    out += [out[4], out[7]]
    return [out[i] for i in rng.permutation(len(out))]


# ---------------------------------------------------------------------------------------------------------------
# CPU: the emulator
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("comp,switch", CODECS)
def test_frame_plans_agree_emu(flib, monkeypatch, capfd, comp, switch):
    """every codec, typesize and shuffle, on frames of five chunks of several blocks and a short last chunk"""
    if switch:
        monkeypatch.setenv(switch, "1")
    for i, ts in enumerate(TYPESIZES):
        for shuf in ((0, 1, 2) if ts == 4 else (i % 3,)):
            n = 5 * 3000 + 700
            src = (gen("mixed", n, seed=ts) if i % 2 else bench_words(n))[:n - n % ts].copy()
            frame = _frame(flib, src, ts, shuf, comp, 3000, 1024)
            nit, ipc = len(src) // ts, _ipc(frame, ts)
            assert nit // ipc == 5 and nit % ipc
            _check(flib, frame, src, ts, _ranges(nit, ipc, np.random.default_rng(10 * ts + shuf)), capfd)


def test_frame_plans_agree_memcpyed_emu(flib, capfd):
    """a frame of memcpyed chunks only, and one where memcpyed chunks sit between compressed ones"""
    ts, cs = 4, 4096
    noisy = gen("rand", 6 * cs + 500, seed=1)
    mixed = noisy.copy()
    for c in range(0, 7, 2):
        mixed[c * cs:(c + 1) * cs] = bench_words(cs, start=c * cs // 4)[:len(mixed[c * cs:(c + 1) * cs])]
    for src, clevel, want_flags in ((bench_words(6 * cs + 500), 0, {True}), (mixed, 5, {True, False})):
        frame = _frame(flib, src, ts, 1, "lz4", cs, 1024, clevel)
        assert {bool(f & 0x2) for _, f in _chunks(frame)} == want_flags
        nit = len(src) // ts
        _check(flib, frame, src, ts, _ranges(nit, _ipc(frame, ts), np.random.default_rng(clevel)), capfd)


@pytest.mark.parametrize("k", [1, TILE - 1, TILE, TILE + 1, 5 * TILE + 37])
def test_frame_plan_tile_boundaries_emu(flib, capfd, k):
    """range counts on both sides of a scan tile, and enough for several tiles and look-back steps"""
    src = bench_words(200000)
    frame = _frame(flib, src, 4, 1, "lz4", 16384, 4096)
    nit = len(src) // 4
    rng = np.random.default_rng(k)
    st = rng.integers(0, nit + 1, k)
    nn = np.minimum(rng.integers(0, 41, k), nit - st)
    nn[rng.random(k) < 0.3] = 0
    _check(flib, frame, src, 4, list(zip(st.tolist(), nn.tolist())), capfd)


def test_frame_plan_many_chunks_emu(flib, capfd):
    """more chunks than one scan tile: the chunk scans span several tiles"""
    ts, cs = 4, 256
    src = bench_words((2 * TILE + 50) * cs + 100)
    frame = _frame(flib, src, ts, 1, "lz4", cs, 0)
    assert len(_chunks(frame)) > 2 * TILE
    nit, ipc = len(src) // ts, cs // ts
    ranges = [(TILE * ipc - 3, 7), (nit - 10, 10), (2040 * ipc + 5, 20 * ipc), (2 * TILE * ipc, ipc), (7, 1),
              (TILE * ipc, 0), (4100 * ipc + 1, 3), (TILE * ipc - 3, 7)]
    _check(flib, frame, src, ts, ranges, capfd)


def test_frame_plan_rejects_emu(flib, capfd):
    """each bad range alone, after good ones and among them, u64 extremes and a start + nitems that wraps: -1, the host
    plan's message and an untouched dest"""
    src = gen("i32", 5 * 4000 + 100)
    frame = _frame(flib, src, 4, 1, "lz4", 4000, 1024)
    nit = len(src) // 4
    good = [(0, 10), (nit - 5, 5), (nit, 0), (999, 3000)]
    bads = [(nit + 1, 0), (nit - 2, 3), (0, nit + 1), (nit, 1), (U64_MAX, 0), (0, U64_MAX), (U64_MAX, U64_MAX),
            (5, U64_MAX - 2), (U64_MAX - 2, 5)]
    cases = [[b] for b in bads] + [good + [b] for b in bads] + [good[:2] + [b] + good[2:] for b in bads]
    cases += [good + [bads[1], bads[6]], [bads[7]] + good + [bads[0]]]
    for ranges in cases:
        (r, out, err), _ = _both(flib, frame, ranges, 256, capfd)
        assert r == -1 and err == OOB and (out == 0xAA).all(), (ranges, r, err)


def test_frame_plan_damaged_chunk_emu(flib, capfd):
    """a corrupt bstarts entry or version byte in a middle chunk: the host plan's code, and nothing written at or past
    the request's total; a request that avoids the chunk still reads"""
    src = bench_words(6 * 8192 + 300)
    frame = _frame(flib, src, 4, 1, "lz4", 8192, 2048)
    ipc = _ipc(frame, 4)
    o = _chunks(frame)[2][0]
    ranges = [(ipc + 5, 2 * ipc), (2 * ipc + 600, 3), (10, 0), (4 * ipc - 1, 2)]
    total = 4 * sum(n for _, n in ranges)
    for damage in ("bstart", "version"):
        f = frame.copy()
        if damage == "bstart":
            f[o + 16 + 4:o + 16 + 8].view(np.int32)[0] = 0x7fff0000          # block 1 of chunk 2
        else:
            f[o] = 3
        dev, host = _both(flib, f, ranges, total, capfd, same_bytes=False)
        assert dev[0] < 0 and (dev[0] == -9) == (damage == "version"), (damage, dev[0])
        assert (dev[1][total:] == 0xAA).all() and (host[1][total:] == 0xAA).all()
        _check(flib, f, src, 4, [(5, ipc), (3 * ipc + 1, 2 * ipc)], capfd)


def test_frame_plan_no_chunks_emu(flib, capfd):
    """a frame without chunks: 0 when every count is 0, whatever the starts, else -1, with no message"""
    fb = flib.blosc_b200_frame_bound(0, 4, 0)
    frame = np.zeros(fb, np.uint8)
    fb = flib.blosc_b200_frame_compress(5, 1, 4, 0, None, ptr(frame), fb, b"lz4", 0, 0, 1)
    assert fb > 0 and not _chunks(frame[:fb])
    frame = frame[:fb].copy()
    for ranges, code in (([(0, 0)], 0), ([(5, 0), (U64_MAX, 0)], 0), ([(0, 0), (0, 1)], -1), ([(U64_MAX, U64_MAX)], -1)):
        (r, out, err), _ = _both(flib, frame, ranges, 16, capfd)
        assert r == code and err == "" and (out == 0xAA).all(), (ranges, r, err)


def test_frame_plan_launches_emu(slib):
    """the frame plan's own launches do not grow with the number of ranges; each touched compressed chunk is one
    chunk plan (4 launches), one decode and one gather"""
    src = bench_words(8 * 4096 + 1000)
    frame = _frame(slib, src, 4, 1, "lz4", 4096, 1024)
    assert not any(f & 0x2 for _, f in _chunks(frame))
    nit, ipc = len(src) // 4, _ipc(frame, 4)
    frame_launches = []
    for k in (1, 16, 4096, 65536):
        rng = np.random.default_rng(k)
        st = rng.integers(0, nit - 2, k)
        ranges = list(zip(st.tolist(), [2] * k))
        st_a, nn_a = _lists(ranges)
        out = np.zeros(8 * k + 16, np.uint8)
        before, after = (ll * 3)(), (ll * 3)()
        slib.emu_set_all_device(1)
        try:
            slib.emu_frame_launches(before)
            assert slib.blosc_b200_frame_getitems(ptr(frame), len(frame), k, st_a.ctypes.data, nn_a.ctypes.data,
                                                  ptr(out)) == 8 * k
            slib.emu_frame_launches(after)
        finally:
            slib.emu_set_all_device(0)
        assert (out[:8 * k] == _want(src, 4, ranges)).all()
        decode, gather, plan = (after[i] - before[i] for i in range(3))
        touched = len(_touched(ranges, ipc))
        assert decode == touched and gather == touched, (k, decode, gather, touched)
        frame_launches.append(plan - 4 * touched)
    assert frame_launches == [6] * 4, frame_launches


# ---------------------------------------------------------------------------------------------------------------
# GPU: the CUDA library
# ---------------------------------------------------------------------------------------------------------------
def _gpu_frames(torch, frame):
    return {"device": torch.from_numpy(frame).cuda(), "pinned": torch.from_numpy(frame).pin_memory(), "pageable": frame}


def _gpu_matrix(pkg, torch, frame, src, ts, ranges, capfd):
    """every mix of frame (device, pinned, pageable), dest (device, host) and lists (int64 / uint64 tensors, both or one
    of them on the device): each call equals the host-list call on the same frame, and valid requests the source
    slices; returns the host-list call's result on the device frame"""
    want = _want(src, ts, ranges)
    st, nn = _lists(ranges)
    results = []
    for fname, f in _gpu_frames(torch, frame).items():
        first = None
        for dest_dev in (True, False):
            lists = [("host", st, nn)]
            for dt in (torch.int64, torch.uint64):
                d_st = torch.from_numpy(st.view(np.int64)).cuda().view(dt)
                d_nn = torch.from_numpy(nn.view(np.int64)).cuda().view(dt)
                lists += [(f"device {dt}", d_st, d_nn), (f"starts {dt}", d_st, nn), (f"nitems {dt}", st, d_nn)]
            for lname, a, b in lists:
                if dest_dev:
                    out = torch.full((len(want) + 16,), 0xAA, dtype=torch.uint8, device="cuda")
                else:
                    out = np.full(len(want) + 16, 0xAA, np.uint8)
                capfd.readouterr()
                r = pkg.frame_getitems(f, len(frame), a, b, out)
                err = capfd.readouterr().err
                got = out.cpu().numpy() if dest_dev else out
                res = (r, err, got.tobytes())
                if first is None:
                    first = res
                assert res == first, (fname, dest_dev, lname, r, first[0], err, first[1])
        r, err, got = first
        got = np.frombuffer(got, np.uint8)
        if r >= 0:
            assert r == len(want) and err == "" and (got[:r] == want).all() and (got[r:] == 0xAA).all(), fname
        results.append((r, err, got))
    return results[0]


@pytest.mark.gpu
def test_frame_plans_agree_gpu(pkg, cuda, capfd):
    torch = cuda
    cs = 1 << 20
    for ts, shuf, comp, src in ((4, 1, "lz4", bench_words(6 * cs + 1236)),
                                (8, 2, "blosclz", np.concatenate([bench_words(3 * cs), gen("rand", 2 * cs + 808, 3)]))):
        frame = _frame(pkg.lib, src, ts, shuf, comp, cs, 0)
        nit, ipc = len(src) // ts, _ipc(frame, ts)
        for seed in (1, 2):
            _gpu_matrix(pkg, torch, frame, src, ts, _ranges(nit, ipc, np.random.default_rng(seed), k=200), capfd)
        for bad in ((nit + 1, 0), (U64_MAX, 0), (5, U64_MAX - 2)):
            r, err, got = _gpu_matrix(pkg, torch, frame, src, ts, [(0, 10), bad, (nit, 0)], capfd)
            assert r == -1 and err == OOB and (got == 0xAA).all(), (bad, r, err)


@pytest.mark.gpu
def test_frame_million_ranges_gpu(pkg, cuda):
    """2^20 random ranges, 40 % of them empty, on a 1 GiB frame of 256 MiB chunks against a full frame_decompress and
    a torch index"""
    torch = cuda
    n, cs = 1 << 30, 256 << 20
    i = torch.arange(n // 4, dtype=torch.int32, device="cuda")
    d_src = (((i << 26) ^ (i << 18) ^ (i << 11) ^ (i << 3) ^ i) & ((1 << 19) - 1)).view(torch.uint8)
    del i
    fb = pkg.frame_bound(n, 4, cs)
    d_frame = torch.empty(fb, dtype=torch.uint8, device="cuda")
    fb = pkg.frame_compress(5, 1, 4, n, d_src, d_frame, fb, "lz4", 0, cs)
    assert fb > 0
    del d_src
    full = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert pkg.frame_decompress(d_frame, fb, full, n) == n
    k, nit, ipc = 1 << 20, n // 4, cs // 4
    g = torch.Generator(device="cuda").manual_seed(7)
    st = torch.randint(0, nit + 1, (k,), device="cuda", generator=g, dtype=torch.int64)
    nn = torch.randint(0, 65, (k,), device="cuda", generator=g, dtype=torch.int64)
    nn = torch.minimum(nn, nit - st)
    nn[torch.rand(k, device="cuda", generator=g) < 0.4] = 0
    st[:3] = torch.tensor([ipc - 10, 2 * ipc - 1, 3 * ipc - 500], device="cuda")      # across chunk boundaries
    nn[:3] = torch.tensor([20, 2, 1000], device="cuda")
    total = int(nn.sum()) * 4
    out = torch.full((total + 16,), 0xAA, dtype=torch.uint8, device="cuda")
    assert pkg.frame_getitems(d_frame, fb, st, nn, out) == total
    idx = torch.repeat_interleave(st, nn)
    idx += torch.arange(idx.numel(), device="cuda") - torch.repeat_interleave(torch.cumsum(nn, 0) - nn, nn)
    want = full.view(torch.int32)[idx].view(torch.uint8)
    assert torch.equal(out[:total], want) and bool((out[total:] == 0xAA).all())


@pytest.mark.gpu
def test_frame_launch_counts_gpu(pkg, cuda):
    """with device lists, each touched compressed chunk is one decode, one gather and one chunk plan (4 plan launches);
    the frame plan adds 6, whatever the number of ranges"""
    torch = cuda
    cs = 4 << 20
    src = bench_words(8 * cs)
    frame = _frame(pkg.lib, src, 4, 1, "lz4", cs, 0)
    assert not any(f & 0x2 for _, f in _chunks(frame))
    d_frame = torch.from_numpy(frame).cuda()
    nit, ipc = len(src) // 4, cs // 4
    pkg.set_profiling(True)
    try:
        for k in (1, 16, 4096, 65536):
            st = np.random.default_rng(k).integers(0, nit - 64, k)
            ranges = list(zip(st.tolist(), [64] * k))
            out = torch.zeros(64 * 4 * k, dtype=torch.uint8, device="cuda")
            d_st = torch.from_numpy(st.astype(np.int64)).cuda()
            pkg.prof_reset()
            assert pkg.frame_getitems(d_frame, len(frame), d_st, torch.full((k,), 64, dtype=torch.int64, device="cuda"),
                                      out) == 64 * 4 * k
            prof = pkg.prof_get()
            touched = len(_touched(ranges, ipc))
            assert prof["decode"][1] == touched and prof["gather"][1] == touched, (k, touched, prof)
            assert prof["plan"][1] == 4 * touched + 6, (k, touched, prof)
            assert (out.cpu().numpy() == _want(src, 4, ranges)).all()
    finally:
        pkg.set_profiling(False)


@pytest.mark.gpu
def test_frame_lists_on_another_device_gpu(pkg, cuda):
    """lists on a device other than the call's are copied to the host and planned there, as before"""
    torch = cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    src = bench_words(3 * (1 << 20) + 400)
    frame = _frame(pkg.lib, src, 4, 1, "lz4", 1 << 20, 0)
    ranges = [(5, 300000), (262140, 10), (0, 0)]
    want = _want(src, 4, ranges)
    st, nn = _lists(ranges)
    d_frame = torch.from_numpy(frame).to("cuda:0")
    out = torch.full((len(want) + 8,), 0xAA, dtype=torch.uint8, device="cuda:0")
    d_st = torch.from_numpy(st.view(np.int64)).to("cuda:1")
    assert pkg.frame_getitems(d_frame, len(frame), d_st, nn, out) == len(want)
    got = out.cpu().numpy()
    assert (got[:len(want)] == want).all() and (got[len(want):] == 0xAA).all()


@pytest.mark.gpu
def test_frame_two_threads_gpu(pkg, cuda):
    """two host threads reading the same frame at once, each with its own device lists"""
    torch = cuda
    src = bench_words(6 * (1 << 20) + 400)
    frame = _frame(pkg.lib, src, 4, 1, "lz4", 1 << 20, 0)
    d_frame = torch.from_numpy(frame).cuda()
    nit, ipc = len(src) // 4, _ipc(frame, 4)
    errors = []

    def reader(seed):
        try:
            for rep in range(4):
                ranges = _ranges(nit, ipc, np.random.default_rng(100 * seed + rep), k=300)
                want = _want(src, 4, ranges)
                st, nn = _lists(ranges)
                out = torch.full((len(want) + 8,), 0xAA, dtype=torch.uint8, device="cuda")
                r = pkg.frame_getitems(d_frame, len(frame), torch.from_numpy(st.view(np.int64)).cuda(),
                                       torch.from_numpy(nn.view(np.int64)).cuda(), out)
                got = out.cpu().numpy()
                if r != len(want) or not (got[:r] == want).all() or not (got[r:] == 0xAA).all():
                    errors.append((seed, rep, r, len(want)))
        except Exception as e:                                      # noqa: BLE001 -- reported below
            errors.append((seed, repr(e)))

    threads = [threading.Thread(target=reader, args=(s,)) for s in (1, 2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors

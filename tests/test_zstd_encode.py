"""Writing "zstd" chunks (csrc/dev_zstdenc.cuh), opt-in with BLOSC_B200_ZSTD=1.

Every chunk must decode with this library and with the reference (oracle/_ref, built with zstd 1.5.6), every
non-raw stream must be a zstd frame that ZSTD_decompress accepts on its own, and the 12 header bytes in front of
cbytes must be the reference's zstd header for the same call (the MEMCPYED bit may differ where the two encoders
reach different fit verdicts).  The frames are not ZSTD_compress's bytes.  CPU: the device code inside the SIMT
emulator.  GPU: the real library must produce the emulator's bytes, from host and device buffers."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from datagen import bench_words, ci, compress, decompress, gen, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "zstd_reference_cbytes.json")

KINDS = ("bench", "text", "lowent", "rand", "zeros", "i32", "mixed")
FILTERS = ((1, 0), (3, 1), (4, 1), (8, 2))                  # (typesize, shuffle)
# (nbytes, forced blocksize): empty, one byte, below MIN_BUFFERSIZE, ragged with a leftover block, and a forced
# blocksize above 128 KiB so that every frame holds several zstd blocks
SIZES = ((0, 0), (1, 0), (100, 0), (70001, 0), (300003, 0), (700001, 300000))


@pytest.fixture
def zstd_on(monkeypatch):
    monkeypatch.setenv("BLOSC_B200_ZSTD", "1")


def _bind(lib):
    for f in ("blosc_compress_ctx", "blosc_decompress_ctx", "blosc_getitem"):
        getattr(lib, f).restype = C.c_int
    return lib


def _zstd(ref):
    if not hasattr(ref, "ZSTD_decompress"):
        pytest.skip("oracle/_ref was built without zstd")
    ref.ZSTD_decompress.restype = C.c_size_t
    ref.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    ref.ZSTD_isError.restype = C.c_uint
    ref.ZSTD_isError.argtypes = [C.c_size_t]
    return _bind(ref)


def _src(kind, n):
    return bench_words(n) if kind == "bench" else gen(kind, n, 7)


def _streams(chunk, n):
    """(block, stream bytes, uncompressed length) of an unsplit chunk, located through bstarts"""
    bs = int.from_bytes(chunk[8:12].tobytes(), "little")
    for b in range((n + bs - 1) // bs):
        st = int.from_bytes(chunk[16 + 4 * b:20 + 4 * b].tobytes(), "little")
        cs = int.from_bytes(chunk[st:st + 4].tobytes(), "little")
        yield b, chunk[st + 4:st + 4 + cs], min(bs, n - b * bs)


def _check_chunk(emu, ref, src, chunk, ts, shuf, clevel, bs):
    """decodes here and with the reference; header = the reference's; every frame passes ZSTD_decompress"""
    n = len(src)
    r, out = decompress(emu, "blosc_decompress_ctx", chunk, n)
    assert r == n and (out[:n] == src).all()
    assert chunk[0] == 2 and chunk[1] == 1 and chunk[3] == ts and (chunk[2] >> 5) == 4 and (chunk[2] & 0x10 or n < 128 or clevel == 0)
    if ref is None:
        return
    r, out = decompress(ref, "blosc_decompress_ctx", chunk, n)
    assert r == n and (out[:n] == src).all()
    rcb, rch = compress(ref, "blosc_compress_ctx", clevel, shuf, ts, src, n + 16, "zstd", bs)
    assert rcb > 0
    assert (chunk[:2] == rch[:2]).all() and (chunk[3:12] == rch[3:12]).all()
    assert (int(chunk[2]) ^ int(rch[2])) & ~0x02 == 0                # MEMCPYED may differ
    if chunk[2] & 0x02 or n == 0:
        return
    for b, fr, ln in _streams(chunk, n):
        if len(fr) == ln:
            continue                                                  # stored raw
        out = np.zeros(ln + 16, np.uint8)
        r = ref.ZSTD_decompress(ptr(out), ln, ptr(fr), len(fr))
        assert not ref.ZSTD_isError(r) and r == ln, (b, len(fr), ln)


@pytest.mark.parametrize("kind", KINDS)
def test_zstd_round_trip_and_reference_decode_emu(emu, ref_if_built, zstd_on, kind):
    emu = _bind(emu)
    ref = _zstd(ref_if_built) if ref_if_built is not None else None
    for n, bs in SIZES:
        src = _src(kind, n)
        for ts, shuf in FILTERS:
            for clevel in (1, 5, 9):
                cb, ch = compress(emu, "blosc_compress_ctx", clevel, shuf, ts, src, n + 16, "zstd", bs)
                assert cb >= 16, (kind, n, ts, clevel, cb)
                assert (ch[cb:] == 0xAA).all()                        # nothing written past the chunk
                chunk = ch[:cb].copy()
                _check_chunk(emu, ref, src, chunk, ts, shuf, clevel, bs)
                if cb > 17 and not chunk[2] & 0x02:
                    small, ch2 = compress(emu, "blosc_compress_ctx", clevel, shuf, ts, src, cb - 1, "zstd", bs)
                    assert small == 0 and (ch2[cb - 1:] == 0xAA).all(), (kind, n, ts, clevel, small)


def test_zstd_getitem_across_blocks_emu(emu, zstd_on):
    emu = _bind(emu)
    for kind in ("bench", "text", "mixed"):
        src = _src(kind, 600000)
        cb, ch = compress(emu, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "zstd", 200000)
        assert cb > 0
        chunk = ch[:cb].copy()
        for start, nitems in ((0, 10), (49990, 20), (49000, 60000), (149999, 1), (0, 150000)):
            item = np.full(nitems * 4 + 8, 0x33, np.uint8)
            assert emu.blosc_getitem(ptr(chunk), ci(start), ci(nitems), ptr(item)) == nitems * 4
            assert (item[:nitems * 4] == src[start * 4:(start + nitems) * 4]).all() and (item[nitems * 4:] == 0x33).all()


def test_zstd_names_follow_the_switch_emu(emu, monkeypatch):
    emu.blosc_compname_to_compcode.argtypes = [C.c_char_p]
    emu.blosc_compcode_to_compname.argtypes = [C.c_int, C.POINTER(C.c_char_p)]
    emu.blosc_list_compressors.restype = C.c_char_p
    emu.blosc_get_complib_info.argtypes = [C.c_char_p, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p)]
    emu.blosc_set_compressor.argtypes = [C.c_char_p]
    name = C.c_char_p()
    lib, ver = C.c_char_p(), C.c_char_p()
    monkeypatch.delenv("BLOSC_B200_ZSTD", raising=False)
    assert emu.blosc_compname_to_compcode(b"zstd") == -1
    assert emu.blosc_compcode_to_compname(5, C.byref(name)) == -1 and name.value == b"zstd"
    assert emu.blosc_list_compressors() == b"blosclz,lz4,lz4hc"
    assert emu.blosc_get_complib_info(b"zstd", C.byref(lib), C.byref(ver)) == -1
    assert emu.blosc_set_compressor(b"zstd") == -1
    monkeypatch.setenv("BLOSC_B200_ZSTD", "1")
    assert emu.blosc_compname_to_compcode(b"zstd") == 5
    assert emu.blosc_compcode_to_compname(5, C.byref(name)) == 5 and name.value == b"zstd"
    assert emu.blosc_list_compressors() == b"blosclz,lz4,lz4hc,zstd"
    assert emu.blosc_get_complib_info(b"zstd", C.byref(lib), C.byref(ver)) == 4 and lib.value == b"Zstd"
    assert emu.blosc_compcode_to_compname(4, C.byref(name)) == -1          # zlib, snappy: still not built
    assert emu.blosc_compname_to_compcode(b"zlib") == -1
    # the global API: blosc_set_compressor and BLOSC_COMPRESSOR
    src = bench_words(200000)
    dest = np.zeros(200016, np.uint8)
    emu.blosc_compress.restype = C.c_int
    assert emu.blosc_set_compressor(b"zstd") == 5
    cb = emu.blosc_compress(ci(5), ci(1), sz(4), sz(len(src)), ptr(src), ptr(dest), sz(len(dest)))
    assert cb > 0 and (dest[2] >> 5) == 4
    emu.blosc_set_compressor(b"blosclz")
    monkeypatch.setenv("BLOSC_COMPRESSOR", "zstd")
    cb = emu.blosc_compress(ci(5), ci(1), sz(4), sz(len(src)), ptr(src), ptr(dest), sz(len(dest)))
    assert cb > 0 and (dest[2] >> 5) == 4
    r, out = decompress(emu, "blosc_decompress_ctx", dest[:cb].copy(), len(src))
    assert r == len(src) and (out[:len(src)] == src).all()
    monkeypatch.delenv("BLOSC_COMPRESSOR")
    emu.blosc_set_compressor(b"blosclz")


# ratio: deterministic, so checked in the emulator.  Inputs of 1 MiB with each kind's natural filter.
RATIO_CASES = (("bench", 4, 1), ("bench", 8, 2), ("text", 1, 0), ("lowent", 4, 1), ("rand", 1, 0), ("zeros", 4, 1),
               ("i32", 4, 1), ("mixed", 1, 0))


def _cbytes(lib, kind, ts, shuf, clevel, comp):
    src = _src(kind, 1 << 20)
    cb, _ = compress(lib, "blosc_compress_ctx", clevel, shuf, ts, src, len(src) + 16, comp)
    assert cb > 0
    return cb


def test_zstd_ratio_against_lz4hc_emu(emu, zstd_on):
    """zstd never loses to this library's own "lz4hc" where that compresses at all (ratio > 1.1) and the
    reference's zstd blocksize is not smaller than lz4hc's: at clevel 1 the reference gives zstd 32 KiB blocks but
    lz4hc 128 KiB ones, and a Blosc block is always a zstd frame of its own."""
    emu = _bind(emu)
    for kind, ts, shuf in RATIO_CASES:
        for clevel in (5, 9):
            zs = _cbytes(emu, kind, ts, shuf, clevel, "zstd")
            hc = _cbytes(emu, kind, ts, shuf, clevel, "lz4hc")
            if (1 << 20) / hc > 1.1:
                assert zs <= hc, (kind, ts, clevel, zs, hc)


def test_zstd_ratio_against_the_reference_emu(emu, ref_if_built, zstd_on):
    """clevel 5: within 1.25x of the reference's zstd cbytes on text and lowent, 2x on the bench.c data"""
    emu = _bind(emu)
    want = json.load(open(GOLDEN))
    for kind, ts, shuf, bound in (("text", 1, 0, 1.25), ("lowent", 4, 1, 1.25), ("bench", 4, 1, 2.0), ("bench", 8, 2, 2.0)):
        key = f"{kind}-ts{ts}-shuf{shuf}-cl5-1MiB"
        if ref_if_built is not None:
            assert _cbytes(_bind(ref_if_built), kind, ts, shuf, 5, "zstd") == want[key]
        zs = _cbytes(emu, kind, ts, shuf, 5, "zstd")
        assert zs <= bound * want[key], (key, zs, want[key])


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_zstd_chunks_equal_emulator_chunks_gpu(pkg, emu, ref_if_built, cuda, zstd_on, kind):
    torch = cuda
    emu = _bind(emu)
    ref = _zstd(ref_if_built) if ref_if_built is not None else None
    for n, bs in SIZES + ((4 << 20, 0),):
        src = _src(kind, n)
        for ts, shuf in FILTERS:
            for clevel in (1, 5, 9):
                want, wch = compress(emu, "blosc_compress_ctx", clevel, shuf, ts, src, n + 16, "zstd", bs)
                dest = np.full(n + 16 + 64, 0xAA, np.uint8)
                cb = pkg.compress_ctx(clevel, shuf, ts, n, src, dest, n + 16, "zstd", bs)
                assert cb == want and (dest[:cb] == wch[:cb]).all() and (dest[cb:] == 0xAA).all(), (kind, n, ts, clevel)
                if n:
                    d_src = torch.from_numpy(src).cuda()
                    d_dst = torch.full((n + 16 + 64,), 0xAA, dtype=torch.uint8, device="cuda")
                    assert pkg.compress_ctx(clevel, shuf, ts, n, d_src, d_dst, n + 16, "zstd", bs) == cb
                    h = d_dst.cpu().numpy()
                    assert (h[:cb] == wch[:cb]).all() and (h[cb:] == 0xAA).all()
                    d_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
                    assert pkg.decompress_ctx(d_dst, d_out, n) == n and torch.equal(d_out, d_src)
                if ref is not None and n:
                    r, out = decompress(ref, "blosc_decompress_ctx", dest[:cb].copy(), n)
                    assert r == n and (out[:n] == src).all()


@pytest.mark.gpu
def test_zstd_frames_api_gpu(pkg, ref_if_built, cuda, zstd_on):
    """a frame of several zstd chunks, and a device-resident one larger than 2 GiB; every chunk decodes with the
    reference"""
    torch = cuda
    ref = _zstd(ref_if_built) if ref_if_built is not None else None
    src = np.concatenate([bench_words(3 << 20), gen("text", (1 << 20) + 13, 2), gen("lowent", 1 << 20, 3)])
    n, cs = len(src), 1 << 20
    bound = pkg.frame_bound(n, 4, cs)
    frame = np.full(bound + 64, 0xAA, np.uint8)
    fb = pkg.frame_compress(5, 1, 4, n, src, frame, bound, "zstd", 0, cs)
    assert fb > 0 and (frame[fb:] == 0xAA).all()
    info = pkg.frame_info(frame, fb)
    assert info == (n, fb, cs, (n + cs - 1) // cs)
    for i in range(info[3]):
        off, cb = pkg.frame_chunk(frame, fb, i)
        piece = src[i * cs:(i + 1) * cs]
        assert (frame[off + 2] >> 5) == 4
        if ref is not None:
            r, out = decompress(ref, "blosc_decompress_ctx", frame[off:off + cb].copy(), len(piece))
            assert r == len(piece) and (out[:len(piece)] == piece).all()
    out = np.zeros(n, np.uint8)
    assert pkg.frame_decompress(frame, fb, out, n) == n and (out == src).all()

    chunk = 256 << 20
    nbig = 9 * chunk
    one = torch.from_numpy(bench_words(chunk)).cuda()
    d_src = one.repeat(9)
    bound = pkg.frame_bound(nbig, 4, chunk)
    d_frame = torch.empty(bound, dtype=torch.uint8, device="cuda")
    fb = pkg.frame_compress(5, 1, 4, nbig, d_src, d_frame, bound, "zstd", 0, chunk)
    assert fb > 0
    sizes = {pkg.frame_chunk(d_frame, fb, i)[1] for i in range(9)}
    assert len(sizes) == 1                                     # nine equal slices, nine equal chunks
    d_out = torch.empty(nbig, dtype=torch.uint8, device="cuda")
    assert pkg.frame_decompress(d_frame, fb, d_out, nbig) == nbig
    assert torch.equal(d_out, d_src)
    del d_out, d_src
    if ref is not None:
        for i in (0, 8):
            off, cb = pkg.frame_chunk(d_frame, fb, i)
            r, out = decompress(ref, "blosc_decompress_ctx", d_frame[off:off + cb].cpu().numpy(), chunk)
            assert r == chunk and (out[:chunk] == one.cpu().numpy()).all()


@pytest.mark.gpu
def test_zstd_bench_buffer_ratio_gpu(pkg, cuda, zstd_on):
    """cfg 2 data (256 MiB bench.c words, shuffle, typesize 4, clevel 5): zstd compresses at least as well as
    this library's lz4hc"""
    torch = cuda
    n = 256 << 20
    d_src = torch.from_numpy(bench_words(n)).cuda()
    d_dst = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    zs = pkg.compress_ctx(5, 1, 4, n, d_src, d_dst, n + 16, "zstd")
    d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert pkg.decompress_ctx(d_dst, d_out, n) == n and torch.equal(d_out, d_src)
    hc = pkg.compress_ctx(5, 1, 4, n, d_src, d_dst, n + 16, "lz4hc")
    assert 0 < zs <= hc, (zs, hc)


@pytest.mark.gpu
def test_zstd_reference_programs_gpu(ref_if_built, cuda, tmp_path):
    """Drop-in evidence: the reference's own bench.c "test" suite passes its memcmp check on "zstd" chunks, and
    `filegen compress` (compat/filegen.c) writes a zstd chunk that the reference library decodes."""
    import subprocess
    bindir = os.path.join(ROOT, "oracle", "_ref", "tests")
    if not os.path.exists(os.path.join(bindir, "bench")):
        pytest.skip("oracle/_ref/tests not built (needs the reference sources at build time)")
    env = dict(os.environ, BLOSC_B200_ZSTD="1")
    r = subprocess.run([os.path.join(bindir, "bench"), "zstd", "shuffle", "test"], capture_output=True, text=True,
                       timeout=900, env=env, cwd=tmp_path)
    assert r.returncode == 0 and "OK" in r.stdout, (r.stdout[-400:], r.stderr[-300:])
    out = tmp_path / "zstd.cdata"
    r = subprocess.run([os.path.join(bindir, "filegen"), "compress", "zstd", str(out)], capture_output=True, text=True,
                       timeout=300, env=env, cwd=tmp_path)
    assert r.returncode == 0 and "Wrote" in r.stdout, (r.stdout[-400:], r.stderr[-300:])
    chunk = np.fromfile(out, np.uint8)
    assert (chunk[2] >> 5) == 4
    if ref_if_built is not None:
        ref = _zstd(ref_if_built)
        r2, dec = decompress(ref, "blosc_decompress_ctx", chunk, 4000000)
        assert r2 == 4000000 and (dec[:4000000] == np.arange(1000000, dtype=np.int32).view(np.uint8)).all()

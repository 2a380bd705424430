"""zstd chunks (SURVEY.md section 8, row f4): decode-only GPU zstd frame decoder.

The algorithm lives in a third-party library of the reference (zstd 1.5.6, vendored under
internal-complibs/ and absent from this repository), so parity is pinned on (1) the reference's
own golden chunks compat/blosc-*-zstd*.cdata and (2) frames written and judged by that very
library (oracle/_ref is built with it): all levels, raw / RLE / compressed blocks, Huffman and
FSE table modes, multi-block frames with repeat modes, checksums; damaged frames must get
ZSTD_decompress()'s accept/reject verdict.  CPU: the device code inside the SIMT emulator.

The verdict rule and its STRICT exceptions (frames the RFC forbids but ZSTD_decompress accepts, refused here) are
stated in tests/test_zstd_decode_edges.py, which tests the decoder branch by branch on frames written to order."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

from datagen import bench_words, ci, compress, decompress, gen, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _zstd(ref):
    if not hasattr(ref, "ZSTD_compress"):
        pytest.skip("oracle/_ref was built without zstd")
    ref.ZSTD_compress.restype = C.c_size_t
    ref.ZSTD_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    ref.ZSTD_decompress.restype = C.c_size_t
    ref.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    ref.ZSTD_isError.restype = C.c_uint
    ref.ZSTD_isError.argtypes = [C.c_size_t]
    ref.ZSTD_compressBound.restype = C.c_size_t
    ref.ZSTD_compressBound.argtypes = [C.c_size_t]
    ref.ZSTD_createCCtx.restype = C.c_void_p
    ref.ZSTD_CCtx_setParameter.restype = C.c_size_t
    ref.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
    ref.ZSTD_compress2.restype = C.c_size_t
    ref.ZSTD_compress2.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    ref.ZSTD_freeCCtx.argtypes = [C.c_void_p]
    return ref


def _frames(ref):
    datas = {
        "bench": bench_words(400000),
        "plane": (bench_words(1 << 20).view(np.uint32) >> 8).astype(np.uint8),   # a shuffled byte-plane
        "text": gen("text", 300000, 1),
        "rand": gen("rand", 50000, 2),
        "zeros": np.zeros(300000, np.uint8),
        "i32": gen("i32", 200000),
        "mixed": gen("mixed", 400000, 3),
        "lowent": gen("lowent", 150000, 4),
        "tiny": np.frombuffer(b"abcabcabcabcabcabcabcabcabcabcabc", np.uint8).copy(),
        "one": np.frombuffer(b"x", np.uint8).copy(),
        "empty": np.zeros(0, np.uint8),
    }
    out = []
    for name, d in datas.items():
        n = len(d)
        for level in (1, 3, 5, 9, 15, 19, 22, -5):
            buf = np.zeros(int(ref.ZSTD_compressBound(n)) + 16, np.uint8)
            r = ref.ZSTD_compress(ptr(buf), len(buf), ptr(d), n, level)
            assert not ref.ZSTD_isError(r)
            out.append((f"{name}-l{level}", d, buf[:r].copy()))
        cctx = ref.ZSTD_createCCtx()                           # with checksum, without content size, small window
        for prm, val in ((100, 3), (201, 1), (200, 0), (101, 12)):   # compressionLevel, checksumFlag, contentSizeFlag, windowLog
            assert not ref.ZSTD_isError(ref.ZSTD_CCtx_setParameter(cctx, prm, val))
        buf = np.zeros(int(ref.ZSTD_compressBound(n)) + 16, np.uint8)
        r = ref.ZSTD_compress2(cctx, ptr(buf), len(buf), ptr(d), n)
        assert not ref.ZSTD_isError(r)
        out.append((f"{name}-cksum", d, buf[:r].copy()))
        ref.ZSTD_freeCCtx(cctx)
    return out


def _verdict(ref, frame, cap):
    out = np.zeros(cap + 16, np.uint8)
    r = ref.ZSTD_decompress(ptr(out), cap, ptr(frame), len(frame))
    return None if ref.ZSTD_isError(r) else out[:r]


def test_zstd_frames_emu(emu, ref):
    ref = _zstd(ref)
    emu.emu_zstd_decode.restype = C.c_int
    for name, d, fr in _frames(ref):
        for cap in (len(d), len(d) + 9, max(len(d) - 1, 0)):
            out = np.full(cap + 16, 0x77, np.uint8)
            r = emu.emu_zstd_decode(ptr(fr), ci(len(fr)), ptr(out), ci(cap))
            want = _verdict(ref, fr, cap)
            if want is None:
                assert r == -1, (name, cap, r)
            else:
                assert r == len(want) and (out[:r] == want).all() and (out[cap:] == 0x77).all(), (name, cap, r)


def test_zstd_rejects_what_zstd_rejects_emu(emu, ref):
    ref = _zstd(ref)
    emu.emu_zstd_decode.restype = C.c_int
    rng = np.random.default_rng(21)
    nbad = ngood = nstrict = 0
    for name, d, fr in _frames(ref):
        if len(d) > 310000 or len(fr) < 12 or not any(t in name for t in ("l3", "l19", "cksum")):
            continue
        for trial in range(20):
            c = fr.copy()
            kind = trial % 5
            if kind == 0:
                c = c[:rng.integers(1, len(c))]
            elif kind == 1:
                c[rng.integers(0, min(len(c), 16))] ^= 1 << rng.integers(0, 8)
            elif kind == 2:
                c = np.concatenate([c, rng.integers(0, 256, 3, dtype=np.uint8)])
            else:
                for pos in rng.integers(0, len(c), kind - 2):
                    c[pos] = rng.integers(0, 256)
            out = np.full(len(d) + 16, 0x77, np.uint8)
            r = emu.emu_zstd_decode(ptr(c), ci(len(c)), ptr(out), ci(len(d)))
            want = _verdict(ref, c, len(d))
            if want is None:
                assert r == -1, (name, trial, kind, r)
                nbad += 1
            elif r == -1:
                # zstd's table-driven Huffman fast loops do not verify that a damaged literal stream is
                # used up exactly (they then emit garbage); this decoder does, and refuses such frames
                assert emu.emu_zstd_fail_line() > 0
                nstrict += 1
            else:
                assert r == len(want) and (out[:r] == want).all(), (name, trial, kind, r)
                ngood += 1
            assert (out[len(d):] == 0x77).all()
    assert nbad > 200 and nstrict <= nbad // 20, (nbad, ngood, nstrict)


def _compat_zstd_files():
    return sorted(f for f in glob.glob(os.path.join(ROOT, "tests", "golden", "compat", "*.cdata")) if "zstd" in f)


def test_compat_zstd_goldens_and_reference_chunks_emu(emu, ref):
    want = np.arange(1000000, dtype=np.int32).view(np.uint8)
    files = _compat_zstd_files()
    assert len(files) == 3
    for f in files:
        chunk = np.fromfile(f, np.uint8)
        out = np.zeros(4000000 + 64, np.uint8)
        assert emu.blosc_decompress_ctx(ptr(chunk), ptr(out), sz(4000000), ci(1)) == 4000000, f
        assert (out[:4000000] == want).all()
    ref = _zstd(ref)
    for f in files:
        chunk = np.fromfile(f, np.uint8)
        for div in (2, 3):                                      # no checksum in these frames: damage may go unnoticed
            bad = chunk.copy(); bad[len(bad) // div] ^= 0x55
            r, o1 = decompress(emu, "blosc_decompress_ctx", bad, 4000000)
            r_ref, o2 = decompress(ref, "blosc_decompress_ctx", bad, 4000000)
            if r_ref < 0:
                assert r == -1, (f, div)
            elif r >= 0:
                assert r == r_ref and (o1[:r] == o2[:r]).all(), (f, div)
    for kind, n in (("bench", 600000), ("text", 100001), ("mixed", 300000), ("rand", 50000)):
        src = gen(kind, n, 4)
        for ts, shuf, clevel in ((4, 1, 5), (8, 2, 1), (1, 0, 9), (3, 1, 6)):
            cb, chunk = compress(ref, "blosc_compress_ctx", clevel, shuf, ts, src, n + 16, "zstd")
            assert cb > 0
            r, out = decompress(emu, "blosc_decompress_ctx", chunk, n)
            assert r == n and (out[:n] == src).all() and (out[n:] == 0).all(), (kind, ts, shuf, clevel)
    # getitem decodes only the blocks it needs (one zstd frame per block)
    cb, chunk = compress(ref, "blosc_compress_ctx", 5, 1, 4, want, len(want) + 16, "zstd")
    emu.blosc_getitem.restype = C.c_int
    for start, nitems in ((0, 10), (65000, 3000), (999000, 1000), (131071, 2)):
        item = np.full(nitems * 4 + 8, 0x33, np.uint8)
        assert emu.blosc_getitem(ptr(chunk), ci(start), ci(nitems), ptr(item)) == nitems * 4
        assert (item[:nitems * 4] == want[start * 4:(start + nitems) * 4]).all() and (item[nitems * 4:] == 0x33).all()
    assert emu.blosc_compress_ctx(ci(5), ci(1), sz(4), sz(1000), ptr(want), ptr(out), sz(2000), b"zstd", sz(0), ci(1)) == -5   # decode only


@pytest.mark.gpu
def test_compat_zstd_goldens_gpu(pkg, ref, cuda):
    want = np.arange(1000000, dtype=np.int32).view(np.uint8)
    files = _compat_zstd_files()
    assert len(files) == 3
    ref = _zstd(ref)
    for f in files:
        chunk = np.fromfile(f, np.uint8)
        out = np.zeros(4000000 + 64, np.uint8)
        assert pkg.decompress_ctx(chunk, out, 4000000) == 4000000, f
        assert (out[:4000000] == want).all() and (out[4000000:] == 0).all()
        for div in (2, 3, 5):                                   # zstd frames carry no checksum here: damage may go unnoticed,
            bad = chunk.copy(); bad[len(bad) // div] ^= 0x55    # in which case both decoders must produce the same bytes
            r = pkg.decompress_ctx(bad, out, 4000000)
            r_ref, out_ref = decompress(ref, "blosc_decompress_ctx", bad, 4000000)
            if r_ref < 0:
                assert r == -1, (f, div)
            elif r >= 0:
                assert r == r_ref and (out[:r] == out_ref[:r]).all(), (f, div)


@pytest.mark.gpu
def test_zstd_chunks_from_the_reference_gpu(pkg, ref, cuda):
    ref = _zstd(ref)
    for kind, n in (("bench", 4 << 20), ("text", 300001), ("mixed", 1 << 20)):
        src = gen(kind, n, 4)
        for ts, shuf, clevel in ((4, 1, 5), (8, 2, 1), (1, 0, 9), (3, 1, 6)):
            cb, chunk = compress(ref, "blosc_compress_ctx", clevel, shuf, ts, src, n + 16, "zstd")
            assert cb > 0
            out = np.zeros(n + 64, np.uint8)
            assert pkg.decompress_ctx(chunk, out, n) == n
            assert (out[:n] == src).all() and (out[n:] == 0).all()

"""Writing "zlib" chunks (csrc/dev_deflate.cuh), opt-in with BLOSC_B200_ZLIB=1.

Every chunk must decode with this library and with the reference (oracle/_ref, built with zlib 1.3.1), every non-raw
stream must be a zlib stream that Python's zlib and this library's inflate (emu_zlib_decode) accept on their own and
that yields its split of the filtered block, and the 12 header bytes in front of cbytes must be the reference's zlib
header for the same call (the MEMCPYED bit may differ where the two encoders reach different fit verdicts).  The
streams are not compress2's bytes.  CPU: the device code inside the SIMT emulator.  GPU: the real library must produce
the emulator's bytes, from host and device buffers."""
import ctypes as C
import json
import os
import zlib

import numpy as np
import pytest

import deflate_read
from datagen import bench_words, ci, compress, decompress, gen, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "zlib_reference_cbytes.json")

KINDS = ("bench", "text", "lowent", "rand", "zeros", "i32", "mixed")
FILTERS = ((1, 0), (3, 1), (4, 1), (8, 2))                  # (typesize, shuffle)
# (nbytes, forced blocksize): empty, one byte, below MIN_BUFFERSIZE, ragged with a leftover block, and a forced
# blocksize above 128 KiB so that streams hold several DEFLATE blocks
SIZES = ((0, 0), (1, 0), (100, 0), (70001, 0), (300003, 0), (700001, 300000))
SEG, SEG_RECS = 256, 64
SPLITMODES = {"always": 1, "never": 2, "auto": 3, "forward_compat": 4}


@pytest.fixture(scope="session")
def stage(tmp_path_factory):
    """the DEFLATE entropy stage alone (tests/emu/deflate_stage.cpp: emu_deflate_stream) in the SIMT emulator, built
    into a temporary directory"""
    import subprocess
    emu_dir = os.path.join(ROOT, "tests", "emu")
    lib = str(tmp_path_factory.mktemp("deflate_stage") / "libdeflate_stage.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++",
                    os.path.join(emu_dir, "deflate_stage.cpp"), os.path.join(emu_dir, "simt_emu.cpp"), "-o", lib,
                    "-lpthread"], check=True)
    out = C.CDLL(lib)
    out.emu_deflate_stream.restype = C.c_int
    return out


@pytest.fixture
def zlib_on(monkeypatch):
    monkeypatch.setenv("BLOSC_B200_ZLIB", "1")


def _bind(lib):
    for f in ("blosc_compress_ctx", "blosc_decompress_ctx", "blosc_getitem"):
        getattr(lib, f).restype = C.c_int
    return lib


def _src(kind, n):
    return bench_words(n) if kind == "bench" else gen(kind, n, 7)


def _inflate_here(emu, stream, n):
    emu.emu_zlib_decode.restype = C.c_int
    out = np.zeros(n + 16, np.uint8)
    s = np.frombuffer(bytes(stream), np.uint8).copy()
    r = emu.emu_zlib_decode(ptr(s), ci(len(s)), ptr(out), ci(n))
    return r, out[:max(r, 0)].tobytes()


def _splits(chunk, n):
    """(block, split, stream bytes or None when stored raw, the split's length) of a chunk, through bstarts"""
    flags, ts = int(chunk[2]), int(chunk[3])
    bs = int.from_bytes(chunk[8:12].tobytes(), "little")
    for b in range((n + bs - 1) // bs):
        blen = min(bs, n - b * bs)
        ns = ts if not flags & 0x10 and blen == bs else 1
        p = int.from_bytes(chunk[16 + 4 * b:20 + 4 * b].tobytes(), "little")
        for j in range(ns):
            ln = blen // ns
            cs = int.from_bytes(chunk[p:p + 4].tobytes(), "little")
            yield b, j, (None if cs == ln else chunk[p + 4:p + 4 + cs].tobytes()), ln
            p += 4 + cs


def _filtered(emu, src, ts, shuf, bs):
    """the bytes the codec sees: each block shuffled / bitshuffled as blosc_b200_filter does it"""
    n = len(src)
    if not ((shuf == 1 and ts > 1) or shuf == 2):
        return src
    out = src.copy()
    for b0 in range(0, n, bs):
        blk = np.ascontiguousarray(src[b0:b0 + bs])
        dst = np.zeros(len(blk), np.uint8)
        assert emu.blosc_b200_filter(ci(0 if shuf == 1 else 2), sz(ts), sz(len(blk)), ptr(blk), ptr(dst)) == 0
        out[b0:b0 + bs] = dst
    return out


def _check_chunk(emu, ref, src, chunk, ts, shuf, clevel, bs, streams=True):
    """decodes here and with the reference; header = the reference's; every stream passes two inflates"""
    n = len(src)
    r, out = decompress(emu, "blosc_decompress_ctx", chunk, n)
    assert r == n and (out[:n] == src).all()
    assert chunk[0] == 2 and chunk[1] == 1 and chunk[3] == ts and (chunk[2] >> 5) == 3
    if ref is not None:
        r, out = decompress(ref, "blosc_decompress_ctx", chunk, n)
        assert r == n and (out[:n] == src).all()
        rcb, rch = compress(ref, "blosc_compress_ctx", clevel, shuf, ts, src, n + 16, "zlib", bs)
        assert rcb > 0
        assert (chunk[:2] == rch[:2]).all() and (chunk[3:12] == rch[3:12]).all()
        assert (int(chunk[2]) ^ int(rch[2])) & ~0x02 == 0                # MEMCPYED may differ
    if chunk[2] & 0x02 or n == 0 or not streams:
        return
    cbs = int.from_bytes(chunk[8:12].tobytes(), "little")
    filt = _filtered(emu, src, ts, shuf, cbs).tobytes()
    for b, j, st, ln in _splits(chunk, n):
        if st is None:
            continue
        want = filt[b * cbs + j * ln:b * cbs + (j + 1) * ln]
        assert zlib.decompress(st) == want, (b, j)
        assert st[:2] == zlib.compress(want, clevel)[:2]
        assert int.from_bytes(st[-4:], "big") == zlib.adler32(want)
        assert len(st) < ln
        r, got = _inflate_here(emu, st, ln)
        assert r == ln and got == want, (b, j, r)


@pytest.mark.parametrize("kind", KINDS)
def test_zlib_round_trip_and_reference_decode_emu(emu, ref_if_built, zlib_on, kind):
    emu = _bind(emu)
    ref = _bind(ref_if_built) if ref_if_built is not None else None
    for n, bs in SIZES:
        src = _src(kind, n)
        for ts, shuf in FILTERS:
            for clevel in (1, 5, 9):
                cb, ch = compress(emu, "blosc_compress_ctx", clevel, shuf, ts, src, n + 16, "zlib", bs)
                assert cb >= 16, (kind, n, ts, clevel, cb)
                assert (ch[cb:] == 0xAA).all()                        # nothing written past the chunk
                chunk = ch[:cb].copy()
                _check_chunk(emu, ref, src, chunk, ts, shuf, clevel, bs)
                if cb > 17 and not chunk[2] & 0x02:
                    small, ch2 = compress(emu, "blosc_compress_ctx", clevel, shuf, ts, src, cb - 1, "zlib", bs)
                    assert small == 0 and (ch2[cb - 1:] == 0xAA).all(), (kind, n, ts, clevel, small)


@pytest.mark.parametrize("mode", sorted(SPLITMODES))
def test_zlib_split_modes_emu(emu, ref_if_built, zlib_on, mode):
    """the split flag and the stream count follow blosc_set_splitmode as in the reference"""
    emu = _bind(emu)
    ref = _bind(ref_if_built) if ref_if_built is not None else None
    libs = [emu] + ([ref] if ref is not None else [])
    try:
        for lib in libs:
            lib.blosc_set_splitmode(ci(SPLITMODES[mode]))
        for kind, ts, shuf in (("bench", 4, 1), ("text", 1, 0), ("i32", 8, 2)):
            src = _src(kind, 300003)
            cb, ch = compress(emu, "blosc_compress_ctx", 5, shuf, ts, src, len(src) + 16, "zlib")
            assert cb > 16
            chunk = ch[:cb].copy()
            split = not chunk[2] & 0x10
            assert split == {"always": True, "never": False, "auto": False, "forward_compat": True}[mode] or \
                (mode == "forward_compat" and ts == 1 and split)
            nstreams = len(list(_splits(chunk, len(src))))
            bs = int.from_bytes(chunk[8:12].tobytes(), "little")
            nfull = len(src) // bs
            assert nstreams == nfull * (ts if split else 1) + (1 if len(src) % bs else 0)
            _check_chunk(emu, ref, src, chunk, ts, shuf, 5, 0)
    finally:
        for lib in libs:
            lib.blosc_set_splitmode(ci(4))


def test_zlib_getitem_across_blocks_and_splits_emu(emu, zlib_on):
    emu = _bind(emu)
    for kind, ts, shuf, bs in (("bench", 4, 1, 200000), ("text", 4, 0, 0), ("mixed", 4, 2, 65536)):
        src = _src(kind, 600000)
        cb, ch = compress(emu, "blosc_compress_ctx", 5, shuf, ts, src, len(src) + 16, "zlib", bs)
        assert cb > 0
        chunk = ch[:cb].copy()
        for start, nitems in ((0, 10), (49990, 20), (49000, 60000), (149999, 1), (0, 150000)):
            item = np.full(nitems * 4 + 8, 0x33, np.uint8)
            assert emu.blosc_getitem(ptr(chunk), ci(start), ci(nitems), ptr(item)) == nitems * 4
            assert (item[:nitems * 4] == src[start * 4:(start + nitems) * 4]).all() and (item[nitems * 4:] == 0x33).all()


@pytest.mark.parametrize("zl,zs", ((0, 0), (1, 0), (0, 1), (1, 1)))
def test_zlib_names_follow_the_switches_emu(emu, monkeypatch, zl, zs):
    emu.blosc_compname_to_compcode.argtypes = [C.c_char_p]
    emu.blosc_compcode_to_compname.argtypes = [C.c_int, C.POINTER(C.c_char_p)]
    emu.blosc_list_compressors.restype = C.c_char_p
    emu.blosc_get_complib_info.argtypes = [C.c_char_p, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p)]
    emu.blosc_set_compressor.argtypes = [C.c_char_p]
    for var, on in (("BLOSC_B200_ZLIB", zl), ("BLOSC_B200_ZSTD", zs)):
        if on:
            monkeypatch.setenv(var, "1")
        else:
            monkeypatch.delenv(var, raising=False)
    name, lib, ver = C.c_char_p(), C.c_char_p(), C.c_char_p()
    assert emu.blosc_compname_to_compcode(b"zlib") == (4 if zl else -1)
    assert emu.blosc_compcode_to_compname(4, C.byref(name)) == (4 if zl else -1) and name.value == b"zlib"
    assert emu.blosc_compname_to_compcode(b"zstd") == (5 if zs else -1)
    assert emu.blosc_compcode_to_compname(5, C.byref(name)) == (5 if zs else -1)
    assert emu.blosc_list_compressors() == b"blosclz,lz4,lz4hc" + (b",zlib" if zl else b"") + (b",zstd" if zs else b"")
    if zl:
        assert emu.blosc_get_complib_info(b"zlib", C.byref(lib), C.byref(ver)) == 3
        assert lib.value == b"Zlib" and ver.value == b"1.3.1"
    else:
        assert emu.blosc_get_complib_info(b"zlib", C.byref(lib), C.byref(ver)) == -1
    src = bench_words(200000)
    dest = np.zeros(200016, np.uint8)
    emu.blosc_compress.restype = C.c_int
    assert emu.blosc_set_compressor(b"zlib") == (4 if zl else -1)
    if zl:
        cb = emu.blosc_compress(ci(5), ci(1), sz(4), sz(len(src)), ptr(src), ptr(dest), sz(len(dest)))
        assert cb > 0 and (dest[2] >> 5) == 3
    emu.blosc_set_compressor(b"blosclz")
    monkeypatch.setenv("BLOSC_COMPRESSOR", "zlib")
    cb = emu.blosc_compress(ci(5), ci(1), sz(4), sz(len(src)), ptr(src), ptr(dest), sz(len(dest)))
    if zl:
        assert cb > 0 and (dest[2] >> 5) == 3
        r, out = decompress(emu, "blosc_decompress_ctx", dest[:cb].copy(), len(src))
        assert r == len(src) and (out[:len(src)] == src).all()
    else:
        assert cb < 0
    monkeypatch.delenv("BLOSC_COMPRESSOR")
    emu = _bind(emu)
    r, _ = compress(emu, "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "zlib")
    assert (r > 0) if zl else r == -5
    emu.blosc_set_compressor(b"blosclz")


# ------------------------------------------------------------------------------------------------
# the entropy stage, branch by branch, from chosen records (emu_deflate_stream, tests/emu/deflate_stage.cpp)
# ------------------------------------------------------------------------------------------------
def _records(n, matches):
    """matches (pos, length, distance) -> the parse's records: cut at segment ends, a piece shorter than 4 bytes is
    left to the literals; the encoder merges a continuation that starts its segment with the same distance"""
    nseg = max((n + SEG - 1) // SEG, 1)
    rec = np.zeros(nseg * SEG_RECS, np.uint32)
    cnt = np.zeros(nseg, np.uint32)
    end = [k * SEG for k in range(nseg)]
    for pos, ml, off in matches:
        a, b = pos, pos + ml
        while a < b:
            k = a // SEG
            e = min(b, (k + 1) * SEG, n)
            if e - a >= 4:
                rec[k * SEG_RECS + int(cnt[k])] = (a - end[k]) | ((e - a - 4) << 8) | (off << 16)
                cnt[k] += 1
                end[k] = e
            a = e
    return rec, cnt


class Build:
    """a source and the matches it was made with"""

    def __init__(self, seed=1):
        self.buf, self.matches, self.rng = bytearray(), [], np.random.default_rng(seed)

    def lit(self, data):
        self.buf += bytes(data)

    def rand(self, k, alphabet=256):
        self.buf += self.rng.integers(0, alphabet, k, dtype=np.uint8).tobytes()

    def match(self, ml, off):
        pos = len(self.buf)
        assert 4 <= ml and 1 <= off <= min(pos, 32768)
        for _ in range(ml):
            self.buf.append(self.buf[-off])
        self.matches.append((pos, ml, off))

    def src(self):
        return np.frombuffer(bytes(self.buf), np.uint8).copy()


def _deflate(emu, stage, src, matches):
    """-> (stream or None when stored, blocks as deflate_read reports them); checked by three inflates"""
    n = len(src)
    rec, cnt = _records(n, matches)
    out = np.full(n + 64, 0xAA, np.uint8)
    r = stage.emu_deflate_stream(ptr(src), ci(n), ptr(rec), ptr(cnt), ptr(out))
    assert 0 < r <= n and (out[n:] == 0xAA).all()
    if r == n:
        return None, []
    st = out[:r].tobytes()
    assert zlib.decompress(st) == src.tobytes()
    got, blocks = deflate_read.read(st)
    assert got == src.tobytes()
    rr, here = _inflate_here(emu, st, n)
    assert rr == n and here == src.tobytes()
    return st, blocks


def test_deflate_literals_only_emu(emu, stage):
    b = Build()
    b.rand(3000, 40)
    st, blocks = _deflate(emu, stage, b.src(), [])
    assert len(blocks) == 1 and blocks[0]["btype"] == 2 and blocks[0]["nmatch"] == 0
    assert blocks[0]["hdist"] == 1 and blocks[0]["dl"] == [1]              # one distance code of length 1


def test_deflate_single_distance_code_emu(emu, stage):
    b = Build()
    b.rand(2000, 30)
    for _ in range(40):
        b.rand(7, 30)
        b.match(20, 700)
    st, blocks = _deflate(emu, stage, b.src(), b.matches)
    (blk,) = blocks
    assert blk["btype"] == 2 and blk["dists"] == {700} and sum(1 for x in blk["dl"] if x) == 1


def test_deflate_every_length_and_merged_runs_emu(emu, stage):
    b = Build()
    b.rand(600, 50)
    for ml in range(4, 257):                                 # every length a segment holds (4..256)
        if len(b.buf) % SEG + ml > SEG:
            b.rand(-len(b.buf) % SEG, 50)
        b.match(ml, 300)
        b.rand(2, 50)
    # merged runs across segments: 258 exactly, and 259, 260, 516, 1000 cut into pieces of 3..258
    for run in (258, 259, 260, 516, 1000):
        b.rand(-len(b.buf) % SEG + 100, 50)
        b.match(run, 64)
    src = b.src()
    st, blocks = _deflate(emu, stage, src, b.matches)
    lens = set().union(*(x.get("lengths", set()) for x in blocks))
    assert set(range(4, 259)) <= lens and 3 in lens                     # 259 -> 256 + 3 and 260 -> 257 + 3
    assert all(x["btype"] in (1, 2) for x in blocks)


def test_deflate_every_distance_code_emu(emu, stage):
    b = Build()
    b.rand(40000, 256)
    dists = [1, 2, 3, 4] + [base for base in deflate_read.DBASE[4:]] + [x - 1 for x in deflate_read.DBASE[5:]] + [32768]
    for d in dists:
        if len(b.buf) % SEG + 12 > SEG:
            b.rand(-len(b.buf) % SEG, 256)
        b.match(12, d)
        b.rand(3, 256)
    st, blocks = _deflate(emu, stage, b.src(), b.matches)
    got = set().union(*(x.get("dists", set()) for x in blocks))
    assert set(dists) <= got and 32768 in got


def test_deflate_length_limits_emu(emu, stage):
    """all 256 literals with Fibonacci-like counts: unlimited Huffman would need more than 15 bits, and the
    code-length code more than 7"""
    fib = [1, 1]
    while len(fib) < 22:
        fib.append(fib[-1] + fib[-2])
    data = bytearray()
    for s in range(256):
        data += bytes([s]) * (fib[s] if s < 22 else 1)
    rng = np.random.default_rng(3)
    data = bytes(rng.permutation(np.frombuffer(bytes(data), np.uint8)))
    st, blocks = _deflate(emu, stage, np.frombuffer(data, np.uint8).copy(), [])
    assert all(x["btype"] == 2 for x in blocks)
    ll = blocks[0]["ll"]
    assert max(ll) == 15 and all(ll[s] for s in range(256))
    assert max(blocks[0]["cl"]) <= 7


def test_deflate_code_length_runs_emu(emu, stage):
    """16 / 17 / 18 with the repeat counts 3, 6, 10, 11 and 138"""
    seen = set()
    cases = [[0, 4, 15, 26, 200], [0, 1, 2, 3, 4, 5, 6, 7, 150], list(range(20)) + [100, 114, 126, 140, 255]]
    for present in cases:
        rng = np.random.default_rng(len(present))
        src = rng.choice(np.array(present, np.uint8), 5000)
        for blk in _deflate(emu, stage, src, [])[1]:
            seen |= set(blk.get("items", []))
    # symbols 0..7, 100 times each: the end-of-block code takes one bit from symbol 0, so 1..7 share a length
    src = np.frombuffer(bytes(range(8)) * 100, np.uint8).copy()
    for blk in _deflate(emu, stage, src, [])[1]:
        seen |= set(blk.get("items", []))
    assert {(16, 3), (16, 6), (17, 3), (17, 10), (18, 11), (18, 138)} <= seen, sorted(x for x in seen if x[0] >= 16)


def test_deflate_fixed_beats_dynamic_emu(emu, stage):
    """a short block: the dynamic header costs more than fixed codes save"""
    b = Build()
    b.lit(b"the quick brown fox jumps over the lazy dog")
    b.match(200, 43)
    st, blocks = _deflate(emu, stage, b.src(), b.matches)
    assert [x["btype"] for x in blocks] == [1]


def test_deflate_stored_blocks_emu(emu, stage):
    """random data with a few matches: stored wins, in pieces of at most 65535 bytes (one of exactly 65535)"""
    b = Build(9)
    b.rand(131072 - 40)
    b.match(40, 1000)
    b.rand(20000)
    src = b.src()
    rec, cnt = _records(len(src), b.matches)
    out = np.full(len(src) + 64, 0xAA, np.uint8)
    r = stage.emu_deflate_stream(ptr(src), ci(len(src)), ptr(rec), ptr(cnt), ptr(out))
    assert r == len(src)                                     # the whole stream would not be smaller: stored raw
    # a block that does not shrink between compressible ones is written stored
    b = Build(10)
    b.lit(b"a" * 131072)
    b.rand(131072)
    b.lit(b"b" * 131072)
    src = b.src()
    st, blocks = _deflate(emu, stage, src, [(1, 131071, 1), (262145, 131071, 1)])
    stored = [x for x in blocks if x["btype"] == 0]
    assert [x["len"] for x in stored] == [65535, 65535, 2]
    assert [x["bfinal"] for x in blocks] == [0] * (len(blocks) - 1) + [1]


def test_deflate_multi_block_bfinal_emu(emu, stage):
    b = Build(4)
    b.rand(1000, 20)
    while len(b.buf) < 400000:
        b.rand(5, 20)
        if len(b.buf) % SEG + 30 <= SEG:
            b.match(30, 999)
    st, blocks = _deflate(emu, stage, b.src(), b.matches)
    assert len(blocks) == 4 and [x["bfinal"] for x in blocks] == [0, 0, 0, 1]
    assert [x["end"] - x["start"] for x in blocks][:3] == [131072] * 3


# ------------------------------------------------------------------------------------------------
# ratio: deterministic, so checked in the emulator.  Inputs of 1 MiB with each kind's natural filter.
# ------------------------------------------------------------------------------------------------
RATIO_CASES = (("bench", 4, 1), ("bench", 8, 2), ("text", 1, 0), ("lowent", 4, 1), ("rand", 1, 0), ("zeros", 4, 1),
               ("i32", 4, 1), ("mixed", 1, 0))
# upper bounds of cbytes / the reference's zlib cbytes at clevel 5 (the stored sizes), and of cbytes / the sum of
# zlib.compress over the splits at clevels 5 and 9: what the emulator measures plus a few percent (DESIGN.md section 3c)
REF_BOUND = {"bench-ts4-shuf1": 1.05, "bench-ts8-shuf2": 0.85, "text-ts1-shuf0": 1.06, "lowent-ts4-shuf1": 1.03,
             "rand-ts1-shuf0": 1.0, "zeros-ts4-shuf1": 3.4, "i32-ts4-shuf1": 1.4, "mixed-ts1-shuf0": 1.02}
PY_BOUND = {"bench-ts4-shuf1": 1.15, "bench-ts8-shuf2": 2.15, "text-ts1-shuf0": 1.06, "lowent-ts4-shuf1": 1.04,
            "rand-ts1-shuf0": 1.0, "zeros-ts4-shuf1": 3.4, "i32-ts4-shuf1": 1.4, "mixed-ts1-shuf0": 1.02}


def _cbytes(lib, kind, ts, shuf, clevel, comp):
    src = _src(kind, 1 << 20)
    cb, ch = compress(lib, "blosc_compress_ctx", clevel, shuf, ts, src, len(src) + 16, comp)
    assert cb > 0
    return cb, ch[:cb].copy(), src


def test_zlib_ratio_against_the_reference_emu(emu, ref_if_built, zlib_on):
    emu = _bind(emu)
    want = json.load(open(GOLDEN))
    for kind, ts, shuf in RATIO_CASES:
        key = f"{kind}-ts{ts}-shuf{shuf}"
        if ref_if_built is not None:
            assert _cbytes(_bind(ref_if_built), kind, ts, shuf, 5, "zlib")[0] == want[key + "-cl5-1MiB"]
        cb = _cbytes(emu, kind, ts, shuf, 5, "zlib")[0]
        assert cb <= REF_BOUND[key] * want[key + "-cl5-1MiB"], (key, cb, want[key + "-cl5-1MiB"])


def test_zlib_ratio_against_lz4hc_emu(emu, zlib_on):
    """zlib is never larger than this library's own "lz4hc" where that compresses at all, except on unfiltered mixed
    data, whose repeats lie farther back than DEFLATE's 32 KiB window but inside LZ4's 64 KiB one"""
    emu = _bind(emu)
    for kind, ts, shuf in RATIO_CASES:
        for clevel in (5, 9):
            zl = _cbytes(emu, kind, ts, shuf, clevel, "zlib")[0]
            hc = _cbytes(emu, kind, ts, shuf, clevel, "lz4hc")[0]
            if (1 << 20) / hc > 1.1:
                assert zl <= (1.01 if kind == "mixed" else 1.0) * hc, (kind, ts, clevel, zl, hc)


def test_zlib_ratio_against_python_zlib_emu(emu, zlib_on):
    """against zlib.compress of every split at the same clevel, summed (plus the chunk's own bytes)"""
    emu = _bind(emu)
    for clevel in (5, 9):
        for kind, ts, shuf in RATIO_CASES:
            key = f"{kind}-ts{ts}-shuf{shuf}"
            cb, chunk, src = _cbytes(emu, kind, ts, shuf, clevel, "zlib")
            if chunk[2] & 0x02:
                continue
            bs = int.from_bytes(chunk[8:12].tobytes(), "little")
            filt = _filtered(emu, src, ts, shuf, bs).tobytes()
            total = 16 + 4 * ((len(src) + bs - 1) // bs)
            for b, j, st, ln in _splits(chunk, len(src)):
                z = zlib.compress(filt[b * bs + j * ln:b * bs + (j + 1) * ln], clevel)
                total += 4 + min(len(z), ln)
            assert cb <= PY_BOUND[key] * total, (key, clevel, cb, total)


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_zlib_chunks_equal_emulator_chunks_gpu(pkg, emu, ref_if_built, cuda, zlib_on, kind):
    torch = cuda
    emu = _bind(emu)
    ref = _bind(ref_if_built) if ref_if_built is not None else None
    for n, bs in SIZES + ((4 << 20, 0),):
        src = _src(kind, n)
        for ts, shuf in FILTERS:
            for clevel in (1, 5, 9):
                want, wch = compress(emu, "blosc_compress_ctx", clevel, shuf, ts, src, n + 16, "zlib", bs)
                dest = np.full(n + 16 + 64, 0xAA, np.uint8)
                cb = pkg.compress_ctx(clevel, shuf, ts, n, src, dest, n + 16, "zlib", bs)
                assert cb == want and (dest[:cb] == wch[:cb]).all() and (dest[cb:] == 0xAA).all(), (kind, n, ts, clevel)
                if n:
                    d_src = torch.from_numpy(src).cuda()
                    d_dst = torch.full((n + 16 + 64,), 0xAA, dtype=torch.uint8, device="cuda")
                    assert pkg.compress_ctx(clevel, shuf, ts, n, d_src, d_dst, n + 16, "zlib", bs) == cb
                    h = d_dst.cpu().numpy()
                    assert (h[:cb] == wch[:cb]).all() and (h[cb:] == 0xAA).all()
                    d_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
                    assert pkg.decompress_ctx(d_dst, d_out, n) == n and torch.equal(d_out, d_src)
                if ref is not None and n:
                    r, out = decompress(ref, "blosc_decompress_ctx", dest[:cb].copy(), n)
                    assert r == n and (out[:n] == src).all()


@pytest.mark.gpu
def test_zlib_frames_api_gpu(pkg, ref_if_built, cuda, zlib_on):
    """a mixed 5 MiB frame whose chunks each decode in the reference, and a device-resident 9 x 256 MiB frame"""
    torch = cuda
    ref = _bind(ref_if_built) if ref_if_built is not None else None
    src = np.concatenate([bench_words(3 << 20), gen("text", (1 << 20) + 13, 2), gen("lowent", 1 << 20, 3)])
    n, cs = len(src), 1 << 20
    bound = pkg.frame_bound(n, 4, cs)
    frame = np.full(bound + 64, 0xAA, np.uint8)
    fb = pkg.frame_compress(5, 1, 4, n, src, frame, bound, "zlib", 0, cs)
    assert fb > 0 and (frame[fb:] == 0xAA).all()
    info = pkg.frame_info(frame, fb)
    assert info == (n, fb, cs, (n + cs - 1) // cs)
    for i in range(info[3]):
        off, cb = pkg.frame_chunk(frame, fb, i)
        piece = src[i * cs:(i + 1) * cs]
        assert (frame[off + 2] >> 5) == 3
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
    fb = pkg.frame_compress(5, 1, 4, nbig, d_src, d_frame, bound, "zlib", 0, chunk)
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
def test_zlib_reference_programs_gpu(ref_if_built, cuda, tmp_path):
    """The reference's own bench.c "test" suite passes its memcmp check on "zlib" chunks, and `filegen compress`
    (compat/filegen.c) writes a zlib chunk that the reference library decodes."""
    import subprocess
    bindir = os.path.join(ROOT, "oracle", "_ref", "tests")
    if not os.path.exists(os.path.join(bindir, "bench")):
        pytest.skip("oracle/_ref/tests not built (needs the reference sources at build time)")
    env = dict(os.environ, BLOSC_B200_ZLIB="1")
    r = subprocess.run([os.path.join(bindir, "bench"), "zlib", "shuffle", "test"], capture_output=True, text=True,
                       timeout=900, env=env, cwd=tmp_path)
    assert r.returncode == 0 and "OK" in r.stdout, (r.stdout[-400:], r.stderr[-300:])
    out = tmp_path / "zlib.cdata"
    r = subprocess.run([os.path.join(bindir, "filegen"), "compress", "zlib", str(out)], capture_output=True, text=True,
                       timeout=300, env=env, cwd=tmp_path)
    assert r.returncode == 0 and "Wrote" in r.stdout, (r.stdout[-400:], r.stderr[-300:])
    chunk = np.fromfile(out, np.uint8)
    assert (chunk[2] >> 5) == 3
    if ref_if_built is not None:
        r2, dec = decompress(_bind(ref_if_built), "blosc_decompress_ctx", chunk, 4000000)
        assert r2 == 4000000 and (dec[:4000000] == np.arange(1000000, dtype=np.int32).view(np.uint8)).all()

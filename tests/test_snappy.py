"""Reading and writing "snappy" chunks (csrc/dev_snappy.cuh), opt-in with BLOSC_B200_SNAPPY=1.

Snappy is not installed and the reference is built without it, so the streams are checked with tests/snappy_read.py,
a reader written from snappy's format_description.txt that the four snappy goldens (blosc 1.3.0 ... 1.14.0) pin, and
with the library's own decoder (emu_snappy_decode).  The header is checked against the oracle's blosclz chunk for the
same call: snappy's compute_blocksize and split_block are blosclz's.  Which splits are raw follows blosc_c's snappy
maxout rule, restated here in Python.  CPU: the device code inside the SIMT emulator.  GPU: the real library must
produce the emulator's bytes, decode the goldens and refuse the bad streams."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

import snappy_read
import snappy_write as sw
from datagen import bench_words, ci, compress, decompress, gen, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "compat", "*-snappy.cdata")))
KINDS = ("bench", "text", "lowent", "rand", "zeros", "i32", "mixed")
FILTERS = ((1, 0), (3, 1), (4, 1), (8, 2))                  # (typesize, shuffle)
SIZES = ((0, 0), (1, 0), (100, 0), (70001, 0), (300003, 0), (700001, 300000))
SEG, SEG_RECS = 256, 64
SPLITMODES = {"always": 1, "never": 2, "auto": 3, "forward_compat": 4}
RING = 16384                                                # LZ4D_RING
HITS = ("DENSE", "DENSE_RING", "DENSE_GLOBAL", "DENSE_BAD", "DENSE_FEW", "LIT_TAG", "LIT_1", "LIT_2", "LIT_3", "LIT_4",
        "LIT_BUMP", "COPY1", "COPY2", "COPY4", "RING", "GLOBAL", "OVERLAP")     # SN_H_* in dev_snappy.cuh


@pytest.fixture(scope="session")
def snappy_emu(tmp_path_factory):
    """the emulated library with the snappy entry points of tests/emu/snappy_stage.cpp (which includes
    backend_emu.cpp whole), built into a temporary directory"""
    import subprocess
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("snappy_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "c-blosc_b200", "csrc", "blosc_b200.c"), "-o",
                    str(d / "host.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "snappy_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    lib = str(d / "libsnappy_stage.so")
    subprocess.run(["g++", "-shared", "-o", lib, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    out = C.CDLL(lib)
    out.blosc_b200_filter.restype = C.c_int
    return _bind(out)


@pytest.fixture
def snappy_on(monkeypatch):
    monkeypatch.setenv("BLOSC_B200_SNAPPY", "1")


def _bind(lib):
    for f in ("blosc_compress_ctx", "blosc_decompress_ctx", "blosc_getitem"):
        getattr(lib, f).restype = C.c_int
    for f in ("emu_snappy_decode", "emu_snappy_fail_line", "emu_snappy_stream", "emu_snappy_hits"):
        if hasattr(lib, f):
            getattr(lib, f).restype = C.c_int
    return lib


def _src(kind, n):
    return bench_words(n) if kind == "bench" else gen(kind, n, 7)


def _u32(a, i):
    return int.from_bytes(bytes(a[i:i + 4]), "little")


def _splits(chunk, n):
    """(block, split, stream bytes or None when stored raw, the split's length) of a chunk, through bstarts"""
    flags, ts, bs = int(chunk[2]), int(chunk[3]), _u32(chunk, 8)
    for b in range((n + bs - 1) // bs):
        blen = min(bs, n - b * bs)
        ns = ts if not flags & 0x10 and blen == bs and ts <= 16 and bs // ts >= 128 else 1
        p = _u32(chunk, 16 + 4 * b)
        for j in range(ns):
            ln = blen // ns
            cs = _u32(chunk, p)
            yield b, j, (None if cs == ln else bytes(chunk[p + 4:p + 4 + cs])), ln
            p += 4 + cs


def _filtered(emu, src, ts, shuf, bs):
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


def _decode_here(emu, st, n):
    s = np.frombuffer(bytes(st), np.uint8).copy() if len(st) else np.zeros(1, np.uint8)
    out = np.zeros(n + 64, np.uint8)
    r = emu.emu_snappy_decode(ptr(s), ci(len(st)), ptr(out), ci(n))
    return r, out[:max(r, 0)].tobytes(), emu.emu_snappy_fail_line()


def _check_chunk(emu, orc, src, chunk, ts, shuf, clevel, bs, nt=1, fn="orc_compress_ctx"):
    n = len(src)
    r, out = decompress(emu, "blosc_decompress_ctx", chunk, n)
    assert r == n and (out[:n] == src).all()
    assert chunk[0] == 2 and chunk[1] == 1 and chunk[3] == ts and (chunk[2] >> 5) == 2
    if orc is not None:
        ocb, och = compress(orc, fn, clevel, shuf, ts, src, n + 16, "blosclz", bs, nt)
        assert ocb > 0
        assert (chunk[3:12] == och[3:12]).all() and chunk[0] == och[0]
        assert (int(chunk[2]) ^ int(och[2])) & ~0xe2 == 0              # codec format and MEMCPYED may differ
    if chunk[2] & 0x02 or n == 0:
        return
    cbs = _u32(chunk, 8)
    filt = _filtered(emu, src, ts, shuf, cbs).tobytes()
    for b, j, st, ln in _splits(chunk, n):
        if st is None:
            continue
        want = filt[b * cbs + j * ln:b * cbs + (j + 1) * ln]
        got, why = snappy_read.read(st, ln)
        assert why is None and got == want, (b, j, why)
        rr, here, _ = _decode_here(emu, st, ln)
        assert rr == ln and here == want, (b, j, rr)
        assert len(st) < ln


# ------------------------------------------------------------------------------------------------
# goldens
# ------------------------------------------------------------------------------------------------
def test_snappy_goldens_decode_emu(snappy_emu, snappy_on):
    """the four snappy goldens decode to data[i] = i, so every compat golden does; snappy_read reads every stream"""
    emu = _bind(snappy_emu)
    want = np.arange(1000000, dtype=np.int32).view(np.uint8)
    files = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "compat", "*.cdata")))
    assert len(files) == 29 and len(GOLDENS) == 4
    for f in files:
        chunk = np.fromfile(f, np.uint8)
        r, out = decompress(emu, "blosc_decompress_ctx", chunk, 4000000)
        assert r == 4000000 and (out[:4000000] == want).all(), f
    for f in GOLDENS:
        chunk = np.fromfile(f, np.uint8)
        bs = _u32(chunk, 8)
        filt = _filtered(emu, want.copy(), 4, 1, bs).tobytes()
        nst = 0
        for b, j, st, ln in _splits(chunk, 4000000):
            assert st is not None
            got, why = snappy_read.read(st, ln)
            assert why is None and got == filt[b * bs + j * ln:b * bs + (j + 1) * ln]
            nst += 1
        assert nst > 0


def test_snappy_goldens_refused_without_the_switch_emu(snappy_emu, monkeypatch):
    monkeypatch.delenv("BLOSC_B200_SNAPPY", raising=False)
    emu = _bind(snappy_emu)
    for f in GOLDENS:
        r, _ = decompress(emu, "blosc_decompress_ctx", np.fromfile(f, np.uint8), 4000000)
        assert r == -5
    r, _ = compress(emu, "blosc_compress_ctx", 5, 1, 4, bench_words(100000), 100016, "snappy")
    assert r == -5


def test_snappy_wrong_codec_version_emu(snappy_emu, snappy_on):
    emu = _bind(snappy_emu)
    chunk = np.fromfile(GOLDENS[0], np.uint8)
    chunk[1] = 2
    r, _ = decompress(emu, "blosc_decompress_ctx", chunk, 4000000)
    assert r == -9


# ------------------------------------------------------------------------------------------------
# round trips
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_snappy_round_trip_emu(snappy_emu, orc, snappy_on, kind):
    emu = _bind(snappy_emu)
    for n, bs in SIZES:
        src = _src(kind, n)
        for ts, shuf in FILTERS:
            for clevel in (1, 5, 9):
                cb, ch = compress(emu, "blosc_compress_ctx", clevel, shuf, ts, src, n + 16, "snappy", bs)
                assert cb >= 16, (kind, n, ts, clevel, cb)
                assert (ch[cb:] == 0xAA).all()
                _check_chunk(emu, orc, src, ch[:cb].copy(), ts, shuf, clevel, bs)


@pytest.mark.parametrize("mode", sorted(SPLITMODES))
def test_snappy_split_modes_emu(snappy_emu, ref_if_built, snappy_on, mode):
    """the split flag follows blosc_set_splitmode; the header is the reference's blosclz header where it is built"""
    emu = _bind(snappy_emu)
    ref = ref_if_built
    libs = [emu] + ([ref] if ref is not None else [])
    try:
        for lib in libs:
            lib.blosc_set_splitmode(ci(SPLITMODES[mode]))
        for kind, ts, shuf in (("bench", 4, 1), ("text", 1, 0), ("i32", 8, 2)):
            src = _src(kind, 300003)
            cb, ch = compress(emu, "blosc_compress_ctx", 5, shuf, ts, src, len(src) + 16, "snappy")
            assert cb > 16
            chunk = ch[:cb].copy()
            split = not chunk[2] & 0x10
            assert split == (mode != "never") or (ts == 1 and split)
            _check_chunk(emu, ref, src, chunk, ts, shuf, 5, 0, fn="blosc_compress_ctx")
    finally:
        for lib in libs:
            lib.blosc_set_splitmode(ci(4))


def test_snappy_getitem_across_blocks_and_splits_emu(snappy_emu, snappy_on):
    emu = _bind(snappy_emu)
    for kind, ts, shuf, bs in (("bench", 4, 1, 200000), ("text", 4, 0, 0), ("mixed", 4, 2, 65536)):
        src = _src(kind, 600000)
        cb, ch = compress(emu, "blosc_compress_ctx", 5, shuf, ts, src, len(src) + 16, "snappy", bs)
        assert cb > 0
        chunk = ch[:cb].copy()
        for start, nitems in ((0, 10), (49990, 20), (49000, 60000), (149999, 1), (0, 150000)):
            item = np.full(nitems * 4 + 8, 0x33, np.uint8)
            assert emu.blosc_getitem(ptr(chunk), ci(start), ci(nitems), ptr(item)) == nitems * 4
            assert (item[:nitems * 4] == src[start * 4:(start + nitems) * 4]).all() and (item[nitems * 4:] == 0x33).all()


def test_snappy_frames_emu(snappy_emu, snappy_on):
    emu = _bind(snappy_emu)
    ll = C.c_longlong
    emu.blosc_b200_frame_bound.restype = C.c_size_t
    emu.blosc_b200_frame_compress.restype = ll
    emu.blosc_b200_frame_decompress.restype = ll
    emu.blosc_b200_frame_getitem.restype = ll
    src = np.concatenate([bench_words(300000), gen("text", 200013, 2), gen("lowent", 100000, 3)])
    n, cs = len(src), 131072
    bound = emu.blosc_b200_frame_bound(sz(n), sz(4), sz(cs))
    frame = np.full(bound + 64, 0xAA, np.uint8)
    fb = emu.blosc_b200_frame_compress(ci(5), ci(1), sz(4), sz(n), ptr(src), ptr(frame), sz(bound), b"snappy", sz(0),
                                       sz(cs), ci(1))
    assert fb > 0 and (frame[fb:] == 0xAA).all()
    out = np.zeros(n, np.uint8)
    assert emu.blosc_b200_frame_decompress(ptr(frame), sz(fb), ptr(out), sz(n), ci(1)) == n and (out == src).all()
    item = np.zeros(4000, np.uint8)
    assert emu.blosc_b200_frame_getitem(ptr(frame), sz(fb), sz(30000), sz(1000), ptr(item)) == 4000
    assert (item == src[120000:124000]).all()


# ------------------------------------------------------------------------------------------------
# names
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sn,zl,zs", [(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)])
def test_snappy_names_follow_the_switches_emu(snappy_emu, monkeypatch, sn, zl, zs):
    emu = snappy_emu
    emu.blosc_compname_to_compcode.argtypes = [C.c_char_p]
    emu.blosc_compcode_to_compname.argtypes = [C.c_int, C.POINTER(C.c_char_p)]
    emu.blosc_list_compressors.restype = C.c_char_p
    emu.blosc_get_complib_info.argtypes = [C.c_char_p, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p)]
    emu.blosc_set_compressor.argtypes = [C.c_char_p]
    emu.blosc_compress.restype = C.c_int
    for var, on in (("BLOSC_B200_SNAPPY", sn), ("BLOSC_B200_ZLIB", zl), ("BLOSC_B200_ZSTD", zs)):
        if on:
            monkeypatch.setenv(var, "1")
        else:
            monkeypatch.delenv(var, raising=False)
    want = b"blosclz,lz4,lz4hc" + (b",snappy" if sn else b"") + (b",zlib" if zl else b"") + (b",zstd" if zs else b"")
    assert emu.blosc_list_compressors() == want
    name, lib, ver = C.c_char_p(), C.c_char_p(), C.c_char_p()
    for comp, code, on, clib, cname in ((b"snappy", 3, sn, 2, b"Snappy"), (b"zlib", 4, zl, 3, b"Zlib"),
                                        (b"zstd", 5, zs, 4, b"Zstd")):
        assert emu.blosc_compname_to_compcode(comp) == (code if on else -1)
        assert emu.blosc_compcode_to_compname(code, C.byref(name)) == (code if on else -1) and name.value == comp
        assert emu.blosc_get_complib_info(comp, C.byref(lib), C.byref(ver)) == (clib if on else -1)
        if on:
            assert lib.value == cname
    if sn:
        emu.blosc_get_complib_info(b"snappy", C.byref(lib), C.byref(ver))
        assert ver.value == b"unknown"
    src = bench_words(200000)
    dest = np.zeros(200016, np.uint8)
    assert emu.blosc_set_compressor(b"snappy") == (3 if sn else -1)
    if sn:
        cb = emu.blosc_compress(ci(5), ci(1), sz(4), sz(len(src)), ptr(src), ptr(dest), sz(len(dest)))
        assert cb > 0 and (dest[2] >> 5) == 2
    emu.blosc_set_compressor(b"blosclz")
    monkeypatch.setenv("BLOSC_COMPRESSOR", "snappy")
    cb = emu.blosc_compress(ci(5), ci(1), sz(4), sz(len(src)), ptr(src), ptr(dest), sz(len(dest)))
    if sn:
        assert cb > 0 and (dest[2] >> 5) == 2
        r, out = decompress(_bind(emu), "blosc_decompress_ctx", dest[:cb].copy(), len(src))
        assert r == len(src) and (out[:len(src)] == src).all()
    else:
        assert cb < 0
    monkeypatch.delenv("BLOSC_COMPRESSOR")
    r, _ = compress(_bind(emu), "blosc_compress_ctx", 5, 1, 4, src, len(src) + 16, "snappy")
    assert (r > 0) if sn else r == -5
    emu.blosc_set_compressor(b"blosclz")


# ------------------------------------------------------------------------------------------------
# blosc_c's snappy maxout rule
# ------------------------------------------------------------------------------------------------
def _bound(n):
    return 32 + n + n // 6                                  # snappy_max_compressed_length


def _predict(pre, n, bs, nsplits, ts, destsize, nthreads):
    """blosc_c / serial_blosc / t_blosc for snappy, from the streams' own sizes `pre` (stream order, == length when
    the encoder stored the split raw).  -> (sizes, bstarts, cbytes) or "memcpyed" or 0"""
    nfull, left = n // bs, n % bs
    blocks = [[bs // nsplits] * nsplits for _ in range(nfull)] + ([[left]] if left else [])
    serial = nthreads == 1 or n // bs <= 1
    pos = 16 + 4 * len(blocks)
    k, sizes, starts, give_up = 0, [], [], False
    for lens in blocks:
        starts.append(pos)
        nt = 0
        for ln in lens:
            c = pre[k]
            k += 1
            nt += 4
            room = (destsize - (pos + 4)) if serial else (bs + 4 * ts - nt)
            if room < _bound(ln):
                if room >= ln:
                    c = ln
                else:
                    give_up = True
            sizes.append(c)
            nt += c
            pos += 4 + c
    if give_up or pos > destsize:
        return "memcpyed" if n + 16 <= destsize else 0
    return sizes, starts, pos


MAXOUT_CASES = (
    # kind, nbytes, typesize, shuffle, forced blocksize, destsize below nbytes + 16
    ("bench", 300003, 4, 1, 0, 0),        # leftover block
    ("bench", 262144 * 3, 1, 0, 65536, 0),  # typesize 1: pool stores every full block raw
    ("lowent", 262147, 1, 0, 65536, 0),
    ("text", 300000, 4, 0, 32768, 0),
    ("bench", 300003, 4, 1, 0, 250000),   # a tight destsize: the clamp binds in serial mode
    ("zeros", 200000, 8, 1, 16384, 199000),
    ("mixed", 400000, 4, 2, 65536, 20000),
)


@pytest.mark.parametrize("nthreads", (1, 4))
@pytest.mark.parametrize("case", range(len(MAXOUT_CASES)))
def test_snappy_maxout_rule_emu(snappy_emu, snappy_on, nthreads, case):
    emu = _bind(snappy_emu)
    kind, n, ts, shuf, fbs, tight = MAXOUT_CASES[case]
    src = _src(kind, n)
    destsize = n + 16 - tight
    nstreams_max = n // 16 + 64
    pre = np.full(nstreams_max, -1, np.int32)
    emu.emu_snappy_presizes(ptr(pre), ci(nstreams_max))
    try:
        cb, ch = compress(emu, "blosc_compress_ctx", 5, shuf, ts, src, destsize, "snappy", fbs, nthreads)
    finally:
        emu.emu_snappy_presizes(None, ci(0))
    assert cb >= 0
    bs = _u32(ch, 8)
    flags = int(ch[2])
    nsplits = ts if not flags & 0x10 and ts <= 16 and bs // ts >= 128 else 1
    want = _predict([int(x) for x in pre], n, bs, nsplits, ts, destsize, nthreads)
    if want == 0:
        assert cb == 0
        return
    if want == "memcpyed":
        assert cb == n + 16 and flags & 0x02
        return
    sizes, starts, total = want
    assert cb == total and not flags & 0x02
    chunk = ch[:cb].copy()
    assert [_u32(chunk, 16 + 4 * b) for b in range(len(starts))] == starts
    got = [len(st) if st is not None else ln for _, _, st, ln in _splits(chunk, n)]
    assert got == sizes
    r, out = decompress(emu, "blosc_decompress_ctx", chunk, n)
    assert r == n and (out[:n] == src).all()


def test_snappy_maxout_rule_pool_unsplit_blocks_are_raw_emu(snappy_emu, snappy_on):
    """typesize 1 in the pool: a full block's room is blocksize + 4 - 4 < its bound, so it is stored raw however well
    it compresses; the short leftover block still compresses"""
    emu = _bind(snappy_emu)
    n = 65536 * 4 + 5000
    src = gen("zeros", n, 1)
    cb, ch = compress(emu, "blosc_compress_ctx", 5, 0, 1, src, n + 16, "snappy", 65536, 4)
    chunk = ch[:cb].copy()
    got = [(st is None) for _, _, st, _ in _splits(chunk, n)]
    assert got == [True] * 4 + [False]
    cb1, ch1 = compress(emu, "blosc_compress_ctx", 5, 0, 1, src, n + 16, "snappy", 65536, 1)
    assert cb1 < cb and all(st is not None for _, _, st, _ in _splits(ch1[:cb1].copy(), n))


# ------------------------------------------------------------------------------------------------
# the stream writer, from chosen records (emu_snappy_stream)
# ------------------------------------------------------------------------------------------------
def _records(n, matches):
    """matches (pos, length, offset) -> the parse's records, cut at segment ends (pieces shorter than 4 bytes are left
    to the literals); the writer merges a continuation that starts its segment with the same offset"""
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
    def __init__(self, seed=1):
        self.buf, self.matches, self.rng = bytearray(), [], np.random.default_rng(seed)

    def rand(self, k):
        self.buf += self.rng.integers(0, 256, k, dtype=np.uint8).tobytes()

    def match(self, ml, off):
        pos = len(self.buf)
        for _ in range(ml):
            self.buf.append(self.buf[-off])
        self.matches.append((pos, ml, off))

    def src(self):
        return np.frombuffer(bytes(self.buf), np.uint8).copy()


def _write(emu, src, matches):
    """-> the stream (None when stored raw) and its elements; checked by both readers"""
    n = len(src)
    rec, cnt = _records(n, matches)
    out = np.full(n + 64, 0xAA, np.uint8)
    r = emu.emu_snappy_stream(ptr(src), ci(n), ptr(rec), ptr(cnt), ptr(out))
    assert 0 < r <= n and (out[r if r < n else 0:] == 0xAA).all() if r == n else (out[r:] == 0xAA).all()
    if r == n:
        return None, []
    st = out[:r].tobytes()
    got, why = snappy_read.read(st, n)
    assert why is None and got == src.tobytes()
    rr, here, _ = _decode_here(emu, st, n)
    assert rr == n and here == src.tobytes()
    return st, snappy_read.elements(st)


def test_snappy_writer_literal_length_forms_emu(snappy_emu):
    """literal runs at every length-encoding boundary: 60/61, 256/257, 65536/65537, 2^24/2^24+1"""
    emu = _bind(snappy_emu)
    for ln, tagbytes in ((60, 1), (61, 2), (256, 2), (257, 3), (65536, 3), (65537, 4), (1 << 24, 4), ((1 << 24) + 1, 5)):
        b = Build(ln)
        b.rand(ln)
        b.match(64, 1)                                      # makes the stream smaller than its input
        b.match(64, 1)
        b.match(64, 1)
        b.match(64, 1)
        st, els = _write(emu, b.src(), b.matches)
        assert els[0][0] == "lit" and els[0][1] == ln
        pre = len(sw.varint(len(b.buf)))
        assert els[0][2] == pre + tagbytes                  # the literals start after the tag and its length bytes


def test_snappy_writer_copy1_against_copy2_emu(snappy_emu):
    emu = _bind(snappy_emu)
    b = Build(3)
    b.rand(2100)
    for ml, off in ((11, 2047), (12, 2047), (11, 2048), (4, 100), (5, 2047)):
        if len(b.buf) % SEG + ml > SEG:
            b.rand(-len(b.buf) % SEG + 3)
        b.match(ml, off)
        b.rand(3)
    b.buf += b"\0" * 400
    b.match(64, 1)
    st, els = _write(emu, b.src(), b.matches)
    copies = [(k, ln, off) for k, ln, off in els if k != "lit"]
    assert copies[:5] == [("c1", 11, 2047), ("c2", 12, 2047), ("c2", 11, 2048), ("c1", 4, 100), ("c1", 5, 2047)]


def test_snappy_writer_long_matches_cut_and_merged_emu(snappy_emu):
    """64, 65, 68 and 128+3 byte matches cut into the fewest pieces (none shorter than 4), and a same-offset match
    that goes on across segments merged before the cut"""
    emu = _bind(snappy_emu)
    b = Build(5)
    b.rand(300)
    for ml in (64, 65, 68, 131):
        b.rand(-len(b.buf) % SEG + 5)                        # each match inside one segment
        b.match(ml, 200)
    b.rand(-len(b.buf) % SEG + 100)
    b.match(156 + 256 + 20, 90)                               # crosses two segment ends: one run of 432 bytes
    st, els = _write(emu, b.src(), b.matches)
    copies = [ln for k, ln, off in els if k != "lit"]
    assert copies[:8] == [64, 61, 4, 64, 4, 64, 63, 4]
    tail = copies[8:]
    assert sum(tail) == 432 and len(tail) == (432 + 63) // 64 and min(tail) >= 4


def test_snappy_writer_raw_exactly_at_size_emu(snappy_emu):
    """the stream is kept when it is smaller than its split and stored raw (nothing written) when it is not"""
    emu = _bind(snappy_emu)
    for extra, raw in ((0, True), (1, False)):
        # n literals + one 64-byte copy at offset 64: size = varint(n) + lit tag bytes + lits + 3
        lits = 1000
        n = lits + 64 - extra
        src = np.frombuffer(np.random.default_rng(9).integers(0, 256, lits, dtype=np.uint8).tobytes(), np.uint8)
        b = Build()
        b.buf += bytes(src)
        b.match(64 - extra, 64)
        size = len(sw.varint(n)) + 3 + lits + 3
        assert (size >= n) == (size == n + extra - 1 >= n)
        st, _ = _write(emu, b.src(), b.matches)
        assert (st is None) == (size >= n)
        if st is not None:
            assert len(st) == size


# ------------------------------------------------------------------------------------------------
# the decoder, from hand-built streams (snappy_write)
# ------------------------------------------------------------------------------------------------
def _hits(emu):
    h = (C.c_longlong * 64)()
    k = emu.emu_snappy_hits(h)
    return {HITS[i]: h[i] for i in range(k)}


def _accept(emu, elems):
    want = sw.expand(elems)
    st = sw.stream(len(want), elems)
    got, why = snappy_read.read(st, len(want))
    assert why is None and got == want
    r, here, line = _decode_here(emu, st, len(want))
    assert r == len(want) and here == want, (r, line)


def test_snappy_decoder_paths_emu(snappy_emu):
    emu = _bind(snappy_emu)
    rng = np.random.default_rng(4)
    _hits(emu)
    r = lambda k: rng.integers(0, 256, k, dtype=np.uint8).tobytes()
    # every tag form, 1..4 literal length bytes, copy-4
    _accept(emu, [("lit", r(5)), ("lit", r(61), 1), ("lit", r(300), 2), ("lit", r(70000), 3), ("lit", r(20), 4),
                  ("c1", 7, 100), ("c2", 64, 30000), ("c4", 33, 70000)])
    # overlapping copies at offsets 1..8, in every form
    for off in range(1, 9):
        _accept(emu, [("lit", r(8)), ("c1", 11, off), ("c2", 64, off), ("c4", 40, off)])
    # sources in the ring and in global memory: offsets on both sides of the ring
    big = r(40000)
    for off in (RING - 200, RING - 64, RING - 63, RING, RING + 1, 30000):
        _accept(emu, [("lit", big), ("c2", 50, off), ("c4", 64, off)])
    # a literal run longer than the ring
    _accept(emu, [("lit", r(RING + 500)), ("c2", 30, 20)])
    # dense runs of copy-2 tags, broken by a literal and by a copy-1
    plane = r(3000)
    els = [("lit", plane)] + [("c2", 64, 3000)] * 40 + [("lit", r(3))] + [("c2", 60, 2900)] * 40 + [("c1", 8, 1000)] + \
          [("c2", 64, 20000 if i % 2 else 2500) for i in range(40)] + [("c2", 64, 8)] + [("c2", 64, 2000)] * 60
    _accept(emu, [("lit", r(20000))] + els)
    h = _hits(emu)
    assert all(h[k] > 0 for k in HITS), {k: v for k, v in h.items() if v == 0}


def test_snappy_stream_longer_than_its_split_emu(snappy_emu, snappy_on):
    """a snappy stream longer than its split (snappy's bound allows it) is kept by the reference and decoded, not taken
    for a raw split: only cs == neblock means raw"""
    emu = _bind(snappy_emu)
    n = 256
    data = np.random.default_rng(2).integers(0, 256, n, dtype=np.uint8).tobytes()
    st = sw.stream(n, [("lit", data[:100], 4), ("lit", data[100:], 4)])
    assert len(st) > n
    chunk = bytearray(16 + 4 + 4) + st
    chunk[0:4] = bytes([2, 1, 0x10 | (2 << 5), 1])
    chunk[4:8] = n.to_bytes(4, "little")
    chunk[8:12] = n.to_bytes(4, "little")
    chunk[12:16] = len(chunk).to_bytes(4, "little")
    chunk[16:20] = (20).to_bytes(4, "little")
    chunk[20:24] = len(st).to_bytes(4, "little")
    r, out = decompress(emu, "blosc_decompress_ctx", np.frombuffer(bytes(chunk), np.uint8).copy(), n)
    assert r == n and out[:n].tobytes() == data


# every reject: (name, stream bytes, split length, snappy_read's reason)
def _rejects():
    x = bytes(range(1, 41))
    out = [
        ("preamble_6_bytes", b"\x80\x80\x80\x80\x80\x01" + sw.lit(x), 40, "preamble"),
        ("preamble_over_32_bits", b"\xa8\x80\x80\x80\x10" + sw.lit(x), 40, "preamble"),
        ("preamble_cut", b"\x80", 40, "preamble"),
        ("length_mismatch", sw.stream(41, [("lit", x)]), 40, "length"),
        ("offset_0", sw.stream(40, [("lit", x[:8]), ("c2", 32, 0)]), 40, "offset"),
        ("offset_past_output", sw.stream(40, [("lit", x[:8]), ("c2", 32, 9)]), 40, "offset"),
        ("copy4_offset_past_output", sw.stream(40, [("lit", x[:8]), ("c4", 32, 1 << 31)]), 40, "offset"),
        ("copy1_offset_cut", sw.stream(40, [("lit", x[:8])]) + b"\x01", 40, "tag_input"),
        ("copy2_offset_cut", sw.stream(40, [("lit", x[:8])]) + b"\x7e\x08", 40, "tag_input"),
        ("copy4_offset_cut", sw.stream(40, [("lit", x[:8])]) + b"\x7f\x08\x00\x00", 40, "tag_input"),
        ("literal_length_cut", sw.varint(40) + b"\xfc\x27\x00", 40, "tag_input"),
        ("literal_past_input", sw.stream(40, [("lit", x)])[:-1], 40, "literal_input"),
        ("literal_past_output", sw.stream(30, [("lit", x)]), 30, "output"),
        ("copy_past_output", sw.stream(20, [("lit", x[:8]), ("c2", 13, 8)]), 20, "output"),
        ("input_left_over", sw.stream(40, [("lit", x)]) + b"\x00", 40, "leftover"),
        ("input_ends_early", sw.stream(40, [("lit", x[:8]), ("c2", 16, 8)]), 40, "short"),
        ("empty", b"", 40, "preamble"),
    ]
    return out


REJECTS = _rejects()


@pytest.mark.parametrize("case", range(len(REJECTS)))
def test_snappy_rejects_emu(snappy_emu, snappy_on, case):
    """every reject, by the reader and by the decoder at a check of its own; through a chunk the call returns the code
    of a refused LZ4 split"""
    emu = _bind(snappy_emu)
    name, st, n, reason = REJECTS[case]
    got, why = snappy_read.read(st, n)
    assert got is None and why == reason, (name, why)
    r, _, line = _decode_here(emu, st, n)
    assert r == -1 and line > 0, name
    lines = {}
    for nm, s2, n2, rs in REJECTS:
        lines.setdefault(rs, set()).add(_decode_here(emu, s2, n2)[2])
    others = set().union(*(v for k, v in lines.items() if k not in (reason, "short", "preamble", "length")))
    if reason not in ("short", "preamble", "length"):
        assert line not in others or reason in ("tag_input", "literal_input"), name
    assert _chunk_code(emu, st, n) == _lz4_chunk_code(emu, n)


def _chunk_of(st, n, fmt):
    chunk = bytearray(24) + bytes(st)
    chunk[0:4] = bytes([2, 1, 0x10 | (fmt << 5), 1])
    chunk[4:8] = n.to_bytes(4, "little")
    chunk[8:12] = n.to_bytes(4, "little")
    chunk[12:16] = len(chunk).to_bytes(4, "little")
    chunk[16:20] = (20).to_bytes(4, "little")
    chunk[20:24] = len(st).to_bytes(4, "little")
    return np.frombuffer(bytes(chunk), np.uint8).copy()


def _chunk_code(lib, st, n):
    return decompress(lib, "blosc_decompress_ctx", _chunk_of(st, n, 2), n)[0]


def _lz4_chunk_code(lib, n):
    return decompress(lib, "blosc_decompress_ctx", _chunk_of(b"\x00", n, 1), n)[0]        # a refused LZ4 split


# ------------------------------------------------------------------------------------------------
# ratio
# ------------------------------------------------------------------------------------------------
def test_snappy_ratio_against_the_goldens_emu(snappy_emu, snappy_on):
    """the goldens' input with each golden's own parameters (clevel 9, shuffle, typesize 4); 1.21 enlarges a forced
    blocksize by typesize for splitting codecs, so 65536 / 131072 give the goldens' 262144 / 524288"""
    emu = _bind(snappy_emu)
    src = np.arange(1000000, dtype=np.int32).view(np.uint8).copy()
    for f in GOLDENS:
        g = np.fromfile(f, np.uint8)
        gbs, gcb = _u32(g, 8), _u32(g, 12)
        cb, ch = compress(emu, "blosc_compress_ctx", 9, 1, 4, src, len(src) + 16, "snappy", gbs // 4)
        assert _u32(ch, 8) == gbs
        assert 16 < cb <= 1.05 * gcb, (f, cb, gcb)


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_snappy_chunks_equal_emulator_chunks_gpu(pkg, emu, cuda, snappy_on, kind):
    torch = cuda
    emu = _bind(emu)
    for n, bs in SIZES + ((4 << 20, 0),):
        src = _src(kind, n)
        for ts, shuf in FILTERS:
            for clevel in ((5,) if n > 1 << 20 else (1, 5, 9)):      # (the emulator is slow on the 4 MiB buffer)
                want, wch = compress(emu, "blosc_compress_ctx", clevel, shuf, ts, src, n + 16, "snappy", bs)
                dest = np.full(n + 16 + 64, 0xAA, np.uint8)
                cb = pkg.compress_ctx(clevel, shuf, ts, n, src, dest, n + 16, "snappy", bs)
                assert cb == want and (dest[:cb] == wch[:cb]).all() and (dest[cb:] == 0xAA).all(), (kind, n, ts, clevel)
                out = np.zeros(n + 16, np.uint8)
                assert pkg.decompress_ctx(dest, out, n) == n and (out[:n] == src).all()
                if n:
                    d_src = torch.from_numpy(src).cuda()
                    d_dst = torch.full((n + 16 + 64,), 0xAA, dtype=torch.uint8, device="cuda")
                    assert pkg.compress_ctx(clevel, shuf, ts, n, d_src, d_dst, n + 16, "snappy", bs) == cb
                    h = d_dst.cpu().numpy()
                    assert (h[:cb] == wch[:cb]).all() and (h[cb:] == 0xAA).all()
                    d_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
                    assert pkg.decompress_ctx(d_dst, d_out, n) == n and torch.equal(d_out, d_src)


@pytest.mark.gpu
def test_snappy_maxout_rule_gpu(pkg, emu, cuda, snappy_on):
    emu = _bind(emu)
    for kind, n, ts, shuf, fbs, tight in MAXOUT_CASES:
        src = _src(kind, n)
        for nt in (1, 4):
            want, wch = compress(emu, "blosc_compress_ctx", 5, shuf, ts, src, n + 16 - tight, "snappy", fbs, nt)
            dest = np.full(n + 16 + 64, 0xAA, np.uint8)
            cb = pkg.compress_ctx(5, shuf, ts, n, src, dest, n + 16 - tight, "snappy", fbs, nt)
            assert cb == want and (dest[:max(cb, 0)] == wch[:max(cb, 0)]).all(), (kind, n, nt)


@pytest.mark.gpu
def test_snappy_goldens_decode_gpu(pkg, cuda, snappy_on):
    """29 of 29 compat goldens decode through the C ABI, from host and device buffers"""
    torch = cuda
    want = np.arange(1000000, dtype=np.int32).view(np.uint8)
    files = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "compat", "*.cdata")))
    assert len(files) == 29
    for f in files:
        chunk = np.fromfile(f, np.uint8)
        out = np.zeros(4000000, np.uint8)
        assert pkg.decompress_ctx(chunk, out, 4000000) == 4000000 and (out == want).all(), f
        d_chunk = torch.from_numpy(chunk).cuda()
        d_out = torch.zeros(4000000, dtype=torch.uint8, device="cuda")
        assert pkg.decompress_ctx(d_chunk, d_out, 4000000) == 4000000
        assert (d_out.cpu().numpy() == want).all(), f
    chunk = np.fromfile(GOLDENS[0], np.uint8)
    item = np.zeros(4000, np.uint8)
    assert pkg.getitem(chunk, 123456, 1000, item) == 4000 and (item == want[123456 * 4:124456 * 4]).all()


@pytest.mark.gpu
def test_snappy_frames_api_gpu(pkg, cuda, snappy_on):
    torch = cuda
    src = np.concatenate([bench_words(3 << 20), gen("text", (1 << 20) + 13, 2), gen("lowent", 1 << 20, 3)])
    n, cs = len(src), 1 << 20
    bound = pkg.frame_bound(n, 4, cs)
    frame = np.full(bound + 64, 0xAA, np.uint8)
    fb = pkg.frame_compress(5, 1, 4, n, src, frame, bound, "snappy", 0, cs)
    assert fb > 0 and (frame[fb:] == 0xAA).all()
    info = pkg.frame_info(frame, fb)
    assert info == (n, fb, cs, (n + cs - 1) // cs)
    out = np.zeros(n, np.uint8)
    assert pkg.frame_decompress(frame, fb, out, n) == n and (out == src).all()
    d_src = torch.from_numpy(bench_words(64 << 20)).cuda()
    nb = d_src.numel()
    bound = pkg.frame_bound(nb, 4, 16 << 20)
    d_frame = torch.empty(bound, dtype=torch.uint8, device="cuda")
    fb = pkg.frame_compress(5, 1, 4, nb, d_src, d_frame, bound, "snappy", 0, 16 << 20)
    assert fb > 0
    d_out = torch.empty(nb, dtype=torch.uint8, device="cuda")
    assert pkg.frame_decompress(d_frame, fb, d_out, nb) == nb and torch.equal(d_out, d_src)


@pytest.mark.gpu
def test_snappy_rejects_gpu(pkg, cuda, snappy_on):
    """every reject stream, once, through the C ABI: the code a refused LZ4 split gets, from host and device"""
    torch = cuda
    lz4 = None
    for name, st, n, _ in REJECTS:
        chunk = _chunk_of(st, n, 2)
        out = np.zeros(n + 16, np.uint8)
        r = pkg.decompress_ctx(chunk, out, n)
        if lz4 is None:
            lz4 = pkg.decompress_ctx(_chunk_of(b"\x00", n, 1), out, n)
            assert lz4 < 0
        assert r == lz4, name
        d_out = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
        assert pkg.decompress_ctx(torch.from_numpy(chunk).cuda(), d_out, n) == lz4, name

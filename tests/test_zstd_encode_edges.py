"""The zstd encoder (csrc/dev_zstdenc.cuh) branch by branch.

The entropy stage runs on sequence records chosen here (emu_zstd_frame, the emulator's hook into zse_frame_serial),
so that rare branches are reached on purpose: repeat-offset cases, a raw block between compressed ones, the three
sequence-count forms, every LL / ML / OF code, every literals and table mode, the frame-header forms.  Every frame
is decoded three ways -- by tests/zstd_frame.py (an independent, strict RFC 8878 decoder), by this library's decoder
(emu_zstd_decode) and by the reference's ZSTD_decompress when oracle/_ref is built -- and then the structure each
scenario is for is asserted from zstd_frame's record of the frame, so a scenario that stops reaching its branch
fails.  test_coverage_ledger lists every branch and asserts that the CPU corpus reaches each one.

Parser-driven inputs go through blosc_compress_ctx (the real zparse records) in the emulator and, on the GPU, through
the library, which must write the emulator's bytes."""
import bisect
import ctypes as C
import os
import re
import threading

import numpy as np
import pytest

import zstd_frame as zf
from datagen import bench_words, compress, decompress, gen, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEG, SEG_RECS, BLOCK = 256, 64, 128 * 1024           # FAST_SEG, ZE_SEG_RECS, ZS_BLOCKMAX


# ------------------------------------------------------------------------------------------------
# a stream and its parse, built together
# ------------------------------------------------------------------------------------------------
class Parse:
    """Appends literals and matches; the bytes of a match are copied from `off` back (overlap allowed), so the
    parse is valid by construction."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.buf = bytearray()
        self.matches = []                             # (pos, ml, off)

    def lit(self, data):
        self.buf += bytes(data)

    def rand(self, k, alphabet=256, p=None):
        if k > 0:
            self.buf += self.rng.choice(alphabet, k, p=p).astype(np.uint8).tobytes() if p is not None else \
                self.rng.integers(0, alphabet, k, dtype=np.uint8).tobytes()

    def match(self, ml, off):
        pos = len(self.buf)
        assert 4 <= ml and 1 <= off <= min(pos, 65535), (pos, ml, off)
        if off >= ml:
            self.buf += self.buf[pos - off:pos - off + ml]
        else:
            pat = bytes(self.buf[pos - off:])
            self.buf += (pat * (ml // off + 1))[:ml]
        self.matches.append((pos, ml, off))

    def pad_to(self, mult, alphabet=16):
        self.rand(-len(self.buf) % mult, alphabet)

    def fits(self, nbytes):
        """the next `nbytes` stay inside the current segment; otherwise literals up to the next one"""
        if len(self.buf) % SEG + nbytes > SEG:
            self.pad_to(SEG)

    def src(self):
        return np.frombuffer(bytes(self.buf), np.uint8).copy()


def make_records(n, matches):
    """matches -> zse_parse_lane's records: a match is cut at segment ends, a piece shorter than 4 bytes is left
    to the literals, and the encoder merges a continuation that starts its segment with LL = 0"""
    nseg = max((n + SEG - 1) // SEG, 1)
    rec = np.zeros(nseg * SEG_RECS, np.uint32)
    cnt = np.zeros(nseg, np.uint32)
    end = [k * SEG for k in range(nseg)]              # end of the last match in each segment, or its start
    for pos, ml, off in matches:
        a, b = pos, pos + ml
        while a < b:
            k = a // SEG
            e = min(b, (k + 1) * SEG, n)
            if e - a >= 4:
                i = int(cnt[k])
                rec[k * SEG_RECS + i] = (a - end[k]) | ((e - a - 4) << 8) | (off << 16)
                cnt[k] += 1
                end[k] = e
            a = e
    return rec, cnt


def assert_record_contract(src, rec, cnt):
    """what zse_parse_lane guarantees the entropy stage"""
    n = len(src)
    nseg = (n + SEG - 1) // SEG
    assert len(cnt) >= nseg and len(rec) >= nseg * SEG_RECS
    for k in range(nseg):
        ss, se = k * SEG, min((k + 1) * SEG, n)
        c = int(cnt[k])
        assert c <= SEG_RECS
        p = ss
        for r in range(c):
            x = int(rec[k * SEG_RECS + r])
            ll, ml, off = x & 0xFF, ((x >> 8) & 0xFF) + 4, x >> 16
            a = p + ll
            assert a + ml <= se, (k, r)
            assert 1 <= off <= 65535 and off <= a, (k, r, off, a)
            assert (src[a:a + ml] == src[a - off:a - off + ml]).all(), (k, r)
            p = a + ml


# ------------------------------------------------------------------------------------------------
# the three decoders
# ------------------------------------------------------------------------------------------------
def _zstd_ref(ref_if_built):
    if ref_if_built is None or not hasattr(ref_if_built, "ZSTD_decompress"):
        return None
    ref_if_built.ZSTD_decompress.restype = C.c_size_t
    ref_if_built.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    ref_if_built.ZSTD_isError.restype = C.c_uint
    ref_if_built.ZSTD_isError.argtypes = [C.c_size_t]
    return ref_if_built


def check_frame(emu, zref, frame, n, want=None):
    """decodes `frame` with zstd_frame, emu_zstd_decode and (if built) ZSTD_decompress; all give `want` (or each
    other's bytes).  Returns zstd_frame's record."""
    frame = np.ascontiguousarray(frame, np.uint8)
    out, info = zf.decode_frame(frame.tobytes())
    assert len(out) == n
    if want is not None:
        assert out == bytes(want), "zstd_frame decodes other bytes"
    dst = np.full(n + 64, 0x5A, np.uint8)
    r = emu.emu_zstd_decode(ptr(frame), len(frame), ptr(dst), n)
    assert r == n and dst[:n].tobytes() == out and (dst[n:] == 0x5A).all(), "emu_zstd_decode disagrees"
    if zref is not None:
        dst = np.zeros(n + 64, np.uint8)
        r = zref.ZSTD_decompress(ptr(dst), n, ptr(frame), len(frame))
        assert not zref.ZSTD_isError(r) and r == n and dst[:n].tobytes() == out, "ZSTD_decompress disagrees"
    return info


def run_hook(emu, src, matches):
    """records from `matches` through emu_zstd_frame; returns (frame or None for stored, hook result)"""
    n = len(src)
    rec, cnt = make_records(n, matches)
    assert_record_contract(src, rec, cnt)
    out = np.full(n + 64, 0xAA, np.uint8)
    r = emu.emu_zstd_frame(ptr(src), n, rec.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), ptr(out))
    assert 0 < r <= n or n == 0, r
    assert (out[n:] == 0xAA).all(), "written past n"
    return (None if r == n else out[:r].copy()), r


def encode_and_check(emu, zref, p):
    src = p.src()
    frame, r = run_hook(emu, src, p.matches)
    if frame is None:
        return src, None, r
    return src, check_frame(emu, zref, frame, len(src), src), r


@pytest.fixture(scope="module")
def hook(emu):
    emu.emu_zstd_frame.restype = C.c_int
    emu.emu_zstd_frame.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    emu.emu_zstd_decode.restype = C.c_int
    emu.emu_zstd_decode.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    return emu


@pytest.fixture(scope="module")
def zref(ref_if_built):
    return _zstd_ref(ref_if_built)


# ------------------------------------------------------------------------------------------------
# records-driven scenarios.  Each returns {name: Parse}; the corpus fixture encodes and decodes them all once.
# ------------------------------------------------------------------------------------------------
A, B, Cc = 100, 200, 300


def _cycle(p):
    """new A, B, Cc; then rep1, rep2, rep3 with LL > 0; rep2, rep3, rep1 - 1 with LL = 0; then a new offset equal
    to rep1 with LL = 0 (which must not be coded as rep1)"""
    p.fits(95)
    for o in (A, B, Cc):
        p.rand(3, 16)
        p.match(8, o)                                  # history Cc, B, A
    p.rand(2, 16); p.match(8, Cc)                      # rep1
    p.rand(2, 16); p.match(8, B)                       # rep2 -> B, Cc, A
    p.rand(2, 16); p.match(8, A)                       # rep3 -> A, B, Cc
    p.match(8, B)                                      # LL 0: rep2 -> B, A, Cc
    p.match(8, Cc)                                     # LL 0: rep3 -> Cc, B, A
    p.match(8, Cc - 1)                                 # LL 0: rep1 - 1 -> Cc-1, Cc, B
    p.match(8, Cc - 1)                                 # LL 0: new offset == rep1


def _history(p, offs=(1000, 2000, 3000)):
    """ends with the history offs[::-1] (distinct, not in the cycle)"""
    p.fits(40)
    for o in offs:
        p.rand(2, 16)
        p.match(8, o)


def sc_repeats():
    p = Parse(1)
    p.rand(3000, 16)
    for blk in range(3):
        if blk:                                        # blocks 2 and 3 start from the history the block before left
            p.rand(4, 16); p.match(8, 3000)
            p.rand(4, 16); p.match(8, 2000)
        while len(p.buf) < (blk + 1) * BLOCK - 400:
            _cycle(p)
        _history(p)
        p.pad_to(BLOCK)
    return {"repeats": p}


def sc_raw_middle():
    p = Parse(2)
    p.rand(3000, 16)
    while len(p.buf) < BLOCK - 400:
        _cycle(p)
    _history(p)                                        # history 3000, 2000, 1000
    p.pad_to(BLOCK)
    p.rand(5000)                                       # block 2: random, one match at a fresh offset: stored raw
    p.fits(8)
    p.match(4, 777)
    p.rand(2 * BLOCK - len(p.buf))
    p.rand(4, 16); p.match(8, 3000)                    # block 3: rep1, then rep2, from block 1's history
    p.rand(4, 16); p.match(8, 2000)
    while len(p.buf) < 3 * BLOCK - 400:
        _cycle(p)
    p.pad_to(BLOCK)
    return {"raw_middle": p}


def _count_stream(ns, seed):
    """`ns` matches of 4 bytes with LL = 0, offsets alternating so that nothing merges"""
    p = Parse(seed)
    p.rand(8)
    for i in range(ns):
        p.match(4, 4 if i % 2 == 0 else 8)
    return p


def sc_counts():
    d = {f"count_{ns}": _count_stream(ns, 10 + i) for i, ns in enumerate((127, 128, 0x7EFF))}
    p = Parse(14)
    p.rand(8)
    p.match(200, 8)
    d["count_1"] = p
    d["count_max"] = _count_stream((BLOCK - 8) // 4, 15)   # 32 766 >= 0x7F00: 64 records in every segment
    p = Parse(16)
    p.rand(2 * BLOCK, 4)                               # a whole block of literals only: no sequences
    d["count_0"] = p
    return d


def sc_codes():
    d = {}
    for c in range(16, 36):                            # every LL code from 16: a literal run of its base (+1)
        p = Parse(100 + c)
        p.rand(zf.LL_BASE[c] + (1 if zf.LL_BITS[c] else 0), 4)
        p.match(300, 7)
        d[f"ll_code_{c}"] = p
    for c in range(1, 53):                             # every ML code: matches of base (+1), merged across segments
        p = Parse(200 + c)
        p.rand(16, 4)
        ml = zf.ML_BASE[c] + (1 if zf.ML_BITS[c] else 0)
        p.match(ml, 16)
        p.rand(-(len(p.buf)) % SEG + 4, 4)            # the match's last piece stays >= 4 bytes
        d[f"ml_code_{c}"] = p
    p = Parse(300)                                     # every OF code 2..16 (0 and 1 are repeat codes)
    p.rand(16, 4)
    p.match(65600, 16)
    p.rand(4, 4)
    for k in range(2, 17):
        off = (1 << k) - 2                             # offset value 2^k + 1: not a repeat offset
        p.fits(40)
        p.rand(3, 4)
        p.match(8, off)
    p.fits(40)
    p.rand(3, 4)
    p.match(8, 65535)
    d["of_codes"] = p
    p = Parse(301)                                     # LL codes 0..15 exactly, in one block
    p.rand(64, 4)
    for rep in range(3):
        for ll in range(16):
            p.fits(ll + 8)
            p.rand(ll, 4)
            p.match(8, 40 + ll + rep)
    d["ll_small"] = p
    return d


def _lit_stream(seed, lits, mlen=4096):
    """block 1 compresses to nothing; block 2 is a match of `mlen` (a whole number of segments) and then exactly
    `lits` as its only literals"""
    p = Parse(seed)
    p.rand(16, 4)
    p.match(BLOCK - 16, 16)
    if mlen:
        p.match(mlen, 16)
    p.lit(lits)
    return p


def _fib_literals(rng):
    f = [1, 1]
    while len(f) < 20:
        f.append(f[-1] + f[-2])
    lits = np.repeat(np.arange(20, dtype=np.uint8) * 7, f)
    return rng.permutation(lits)


# a histogram whose unconstrained Huffman code is deeper than 11 bits and where lengthening only the codes shorter
# than 10 bits, instead of all below 11, would end with a worse code
DEEP2 = [149, 1097, 3173, 5, 2, 563, 3, 132, 3, 2, 15, 2, 2, 15, 147, 13, 223, 2994, 1144, 147, 7899, 6, 29, 1715]


def _deep2_literals(rng):
    return rng.permutation(np.repeat((np.arange(len(DEEP2)) * 3).astype(np.uint8), DEEP2))


def huffman_lengths_limited(literals):
    """The encoder's rule for code lengths <= 11 (ze_huf_lengths), restated: a two-queue Huffman tree over the symbols
    sorted by count then value; depths clamped to 11; while the Kraft sum is above 2^11 lengthen, rarest first, every
    code below 11 bits; while there is room shorten, most frequent first, every code above 1 bit that fits."""
    hist = np.bincount(np.frombuffer(bytes(literals), np.uint8), minlength=256)
    leaf = sorted((s for s in range(256) if hist[s]), key=lambda s: (hist[s], s))
    n = len(leaf)
    w, par = [int(hist[s]) for s in leaf] + [0] * n, [0] * (2 * n)
    li, ni, nn = 0, n, n
    for _ in range(n - 1):
        pick = []
        for _ in range(2):
            if li < n and (ni >= nn or w[li] <= w[ni]):
                pick.append(li); li += 1
            else:
                pick.append(ni); ni += 1
        w[nn] = w[pick[0]] + w[pick[1]]
        par[pick[0]] = par[pick[1]] = nn
        nn += 1
    depth = [0] * (2 * n)
    for k in range(nn - 2, -1, -1):
        depth[k] = depth[par[k]] + 1
    ln = [0] * 256
    for i in range(n):
        ln[leaf[i]] = min(depth[i], 11)
    kraft = sum(1 << (11 - ln[s]) for s in leaf)
    while kraft > 2048:
        for s in leaf:
            if kraft <= 2048:
                break
            if ln[s] < 11:
                kraft -= 1 << (10 - ln[s]); ln[s] += 1
    while kraft < 2048:
        for s in reversed(leaf):
            if kraft >= 2048:
                break
            if ln[s] > 1 and 1 << (11 - ln[s]) <= 2048 - kraft:
                kraft += 1 << (11 - ln[s]); ln[s] -= 1
    return ln


def sc_literals():
    rng = np.random.default_rng(400)
    skew = lambda k: rng.choice(np.array([0, 1, 2, 3], np.uint8), k, p=[0.55, 0.25, 0.15, 0.05])
    wide = np.where(rng.random(20000) < 0.85, 0, rng.integers(1, 256, 20000)).astype(np.uint8)
    wide[:255] = np.arange(1, 256, dtype=np.uint8)
    d = {
        "lit_none": _lit_stream(401, b""),
        "lit_one": _lit_stream(402, b"\x07"),
        "lit_two_equal": _lit_stream(403, b"\x07\x07"),
        "lit_rle_3": _lit_stream(404, b"\x09" * 3),
        "lit_rle_100": _lit_stream(404, b"\x09" * 100),
        "lit_rle_5000": _lit_stream(404, b"\x09" * 5000),
        "lit_raw_31": _lit_stream(405, rng.integers(0, 256, 31, dtype=np.uint8)),
        "lit_raw_32": _lit_stream(406, rng.integers(0, 256, 32, dtype=np.uint8)),
        "lit_raw_4095": _lit_stream(407, rng.integers(0, 256, 4095, dtype=np.uint8)),
        "lit_raw_4096": _lit_stream(408, rng.integers(0, 256, 4096, dtype=np.uint8)),
        "lit_huf1_64": _lit_stream(409, skew(64)),
        "lit_huf1_1023": _lit_stream(410, skew(1023)),
        "lit_huf4_1024": _lit_stream(411, skew(1024)),
        "lit_huf4_16383": _lit_stream(412, skew(16383)),
        "lit_huf4_16384": _lit_stream(413, skew(16384)),
        "lit_huf4_block": _lit_stream(414, skew(BLOCK), 0),
        "lit_fse_weights": _lit_stream(415, wide),
        "lit_direct_weights": _lit_stream(416, skew(2000)),
        "lit_deep": _lit_stream(417, _fib_literals(rng)),
        "lit_deep2": _lit_stream(418, _deep2_literals(rng)),
    }
    return d


def sc_modes():
    d = {}
    p = Parse(500)                                     # FSE at the maximum accuracy logs: > 2048 sequences
    p.rand(2048, 16)
    rng = p.rng
    for i in range(3000):
        ll = int(rng.choice([0, 1, 2, 5, 9, 14, 20, 30], p=[.3, .2, .15, .1, .1, .05, .05, .05]))
        ml = int(rng.choice([4, 5, 6, 9, 13, 20, 40], p=[.3, .2, .15, .1, .1, .1, .05]))
        off = int(rng.choice([17, 40, 90, 300, 700, 1500]))
        p.fits(ll + ml)
        p.rand(ll, 16)
        p.match(ml, off)
    d["modes_maxlog"] = p
    p = Parse(501)                                     # zero runs: ML codes {1, 2, 40}, LL codes {0, 1, 10}
    p.rand(2048, 16)
    rng = p.rng
    for i in range(600):
        ll = int(rng.choice([0, 1, 10], p=[.5, .3, .2]))
        ml = int(rng.choice([4, 5, 70], p=[.5, .3, .2]))
        p.fits(ll + ml)
        p.rand(ll, 16)
        p.match(ml, int(rng.integers(100, 2000)))
    d["modes_zero_runs"] = p
    p = Parse(502)                                     # RLE for all three: every sequence has the same codes
    p.rand(64, 16)
    p.match(BLOCK - 64, 64)
    for i in range(100):                               # 8 bytes each: no literals pad a segment's end
        p.rand(2, 16)
        p.match(6, 64)
    d["modes_rle"] = p
    return d


def sc_frames():
    d = {}
    for n in (15, 16, 17, 255, 256, 65791, 65792, BLOCK, BLOCK + 1):
        p = Parse(600 + n % 1000)
        p.rand(1)
        p.match(n - 1 if n < BLOCK else n - 1 - (n - BLOCK), 1)
        if n > BLOCK:
            p.rand(1)
        d[f"frame_{n}"] = p
    p = Parse(610)
    p.rand(5000)
    d["frame_incompressible"] = p
    return d


def _edge_stream(k, m):
    """block 1 tiny; block 2 = k random literals, then one match of m at a repeat offset (predefined tables)"""
    p = Parse(620)
    p.rand(16, 4)
    p.match(BLOCK - 16, 16)
    p.rand(k)
    p.match(m, 16)
    return p


SCENARIOS = (sc_repeats, sc_raw_middle, sc_counts, sc_codes, sc_literals, sc_modes, sc_frames)


@pytest.fixture(scope="module")
def corpus(hook, zref):
    """name -> (src, zstd_frame record or None when stored, hook result), every frame checked three ways"""
    out = {}
    for sc in SCENARIOS:
        for name, p in sc().items():
            out[name] = encode_and_check(hook, zref, p)
    return out


def _blocks(corpus, name):
    src, info, _ = corpus[name]
    assert info is not None, f"{name}: stored, not a frame"
    return info.blocks


def _seqs(blk):
    return blk["seq"]["seqs"] if blk["type"] == "compressed" else []


# ------------------------------------------------------------------------------------------------
# the scenarios' intended structure
# ------------------------------------------------------------------------------------------------
def test_repeat_offsets_all_cases_across_blocks_emu(corpus):
    blocks = _blocks(corpus, "repeats")
    assert [b["type"] for b in blocks] == ["compressed"] * 3
    cases = {s[5] for b in blocks for s in _seqs(b)}
    assert {"rep1", "rep2", "rep3", "rep2_ll0", "rep3_ll0", "rep1m1_ll0", "new"} <= cases
    # a new offset equal to rep1 with LL = 0 is coded as a new offset
    assert any(s[5] == "new" and s[6] == 0 and s[4] == s[8] for b in blocks for s in _seqs(b))
    for b in blocks[1:]:                               # history carried over from the block before
        first = _seqs(b)[:2]
        assert [s[5] for s in first] == ["rep1", "rep2"] and [s[4] for s in first] == [3000, 2000]


def test_raw_block_keeps_the_decoders_repeat_offsets_emu(corpus):
    """block 2 is stored raw after the encoder has seen its match at a fresh offset; block 3 must code block 1's
    history as the decoder has it"""
    blocks = _blocks(corpus, "raw_middle")
    assert [b["type"] for b in blocks] == ["compressed", "raw", "compressed"]
    assert blocks[0]["rep_after"] == (3000, 2000, 1000)
    first = _seqs(blocks[2])[:2]
    assert [(s[5], s[4]) for s in first] == [("rep1", 3000), ("rep2", 2000)]


def test_sequence_count_forms_emu(corpus):
    for name, ns, nbytes in (("count_0", 0, 1), ("count_1", 1, 1), ("count_127", 127, 1), ("count_128", 128, 2),
                             ("count_32511", 0x7EFF, 2), ("count_max", 32766, 3)):
        blocks = _blocks(corpus, name)
        b = blocks[-1] if name == "count_0" else blocks[0]
        assert b["type"] == "compressed" and b["seq"]["count"] == ns and b["seq"]["count_bytes"] == nbytes, name
    b = _blocks(corpus, "count_max")[0]
    assert b["out"] == BLOCK and b["seq"]["modes"]["ml"] == "rle"


def test_every_code_emu(corpus):
    ll, ml, of = set(), set(), set()
    for name, (src, info, _) in corpus.items():
        if info is None:
            continue
        for b in info.blocks:
            for s in _seqs(b):
                ll.add(s[0]); ml.add(s[1]); of.add(s[2])
    assert ll == set(range(36))
    assert ml == set(range(1, 53))                     # ML code 0 is a match of 3 bytes: records are >= 4
    assert set(range(17)) <= of
    assert any(s[4] == 65535 for b in _blocks(corpus, "of_codes") for s in _seqs(b))
    assert any(s[0] == 35 for b in _blocks(corpus, "ll_code_35") for s in _seqs(b))
    assert any(s[1] == 52 and s[7] >= 65539 for b in _blocks(corpus, "ml_code_52") for s in _seqs(b))


LIT_EXPECT = {                                         # name: (type, size format, streams, weights)
    "lit_none": ("raw", 0, None, None), "lit_one": ("raw", 0, None, None), "lit_two_equal": ("raw", 0, None, None),
    "lit_rle_3": ("rle", 0, None, None), "lit_rle_100": ("rle", 1, None, None), "lit_rle_5000": ("rle", 3, None, None),
    "lit_raw_31": ("raw", 0, None, None), "lit_raw_32": ("raw", 1, None, None),
    "lit_raw_4095": ("raw", 1, None, None), "lit_raw_4096": ("raw", 3, None, None),
    "lit_huf1_64": ("compressed", 0, 1, None), "lit_huf1_1023": ("compressed", 0, 1, None),
    "lit_huf4_1024": ("compressed", 2, 4, None), "lit_huf4_16383": ("compressed", 2, 4, None),
    "lit_huf4_16384": ("compressed", 3, 4, None), "lit_huf4_block": ("compressed", 3, 4, None),
    "lit_fse_weights": ("compressed", None, None, "fse"), "lit_direct_weights": ("compressed", None, None, "direct"),
    "lit_deep": ("compressed", None, None, None), "lit_deep2": ("compressed", None, None, None),
}


@pytest.mark.parametrize("name", sorted(LIT_EXPECT))
def test_literals_section_forms_emu(corpus, name):
    src, info, _ = corpus[name]
    b = _blocks(corpus, name)[1]
    lit = b["lit"]
    t, sf, streams, weights = LIT_EXPECT[name]
    nlit = {"lit_none": 0, "lit_one": 1, "lit_two_equal": 2, "lit_huf4_block": BLOCK}.get(name)
    if nlit is None:
        nlit = int(name.rsplit("_", 1)[1]) if name.rsplit("_", 1)[1].isdigit() else lit["regen"]
    assert b["type"] == "compressed" and lit["regen"] == nlit
    assert lit["type"] == t, (name, lit["type"])
    if sf is not None:
        assert lit["size_format"] == sf, (name, lit["size_format"])
    if streams is not None:
        assert lit["streams"] == streams
    if weights is not None:
        assert lit["weights"] == weights
    if name == "lit_huf4_block":
        assert b["seq"]["count"] == 0
    if name == "lit_fse_weights":
        assert max(lit["literals"]) == 255 and len(set(lit["literals"])) > 129
    if name.startswith("lit_deep"):                    # the length limit: clamp and both Kraft loops
        assert zf.huffman_depth(lit["literals"]) > 11 and lit["max_bits"] == 11
    if lit["type"] == "compressed":                    # the code lengths written are the encoder's rule's
        assert lit["lengths"] == huffman_lengths_limited(lit["literals"]), name


def test_sequence_table_modes_emu(corpus):
    b = _blocks(corpus, "modes_maxlog")[0]
    assert b["seq"]["count"] > 2048
    assert b["seq"]["modes"] == {"ll": "fse", "of": "fse", "ml": "fse"}
    assert b["seq"]["logs"] == {"ll": 9, "of": 8, "ml": 9}
    b = _blocks(corpus, "modes_zero_runs")[0]
    assert b["seq"]["modes"]["ml"] == "fse" and b["seq"]["modes"]["ll"] == "fse"
    assert max(b["seq"]["zero_runs"]["ml"]) >= 24                   # 0xffff repeat of 24 zeros
    assert any(3 <= r < 24 for r in b["seq"]["zero_runs"]["ll"])
    b = _blocks(corpus, "count_1")[0]
    assert b["seq"]["modes"] == {"ll": "predefined", "of": "predefined", "ml": "predefined"}
    b = _blocks(corpus, "modes_rle")[1]
    assert b["seq"]["modes"] == {"ll": "rle", "of": "rle", "ml": "rle"} and b["seq"]["count"] == 100


def test_frame_header_forms_emu(corpus):
    assert corpus["frame_15"][1] is None and corpus["frame_15"][2] == 15
    assert corpus["frame_16"][1] is None and corpus["frame_16"][2] == 16      # the smallest frame is 16 bytes
    assert corpus["frame_incompressible"][1] is None
    for n, fb, fhd in ((17, 1, 0x20), (255, 1, 0x20), (256, 2, 0x60), (65791, 2, 0x60), (65792, 4, 0xA0),
                       (BLOCK, 4, 0xA0), (BLOCK + 1, 4, 0xA0)):
        src, info, _ = corpus[f"frame_{n}"]
        assert info.fcs_bytes == fb and info.fhd == fhd and info.fcs == n and info.single_segment
    assert [b["type"] for b in _blocks(corpus, f"frame_{BLOCK}")] == ["compressed"]
    blocks = _blocks(corpus, f"frame_{BLOCK + 1}")
    assert [(b["type"], b["out"]) for b in blocks] == [("compressed", BLOCK), ("raw", 1)] and blocks[1]["last"]


def test_block_of_blen_minus_one_stays_compressed_emu(hook, zref):
    """a block that codes to blen - 1 bytes stays compressed; the same block one match byte shorter codes to as
    many bytes (the single sequence's codes keep their extra-bit counts) but is one byte shorter, so it is raw"""
    found = None
    for k in (20, 40, 100):
        for m in range(5, 34):
            src, info, _ = encode_and_check(hook, zref, _edge_stream(k, m))
            b = info.blocks[1]
            if b["type"] == "compressed" and b["size"] == b["out"] - 1:
                found = (k, m, b)
                break
        if found:
            break
    assert found, "no match length gives a block of blen - 1"
    k, m, b = found
    s = b["seq"]["seqs"]
    assert len(s) == 1 and b["seq"]["modes"] == {"ll": "predefined", "of": "predefined", "ml": "predefined"}
    assert zf.ML_BITS[s[0][1]] == 0 and m - 1 >= 4
    src, info, _ = encode_and_check(hook, zref, _edge_stream(k, m - 1))
    assert info.blocks[1]["type"] == "raw" and info.blocks[1]["out"] == k + m - 1


def _plant_stream(rng, n):
    """random bytes over a random alphabet with repeats planted at random offsets (some copied from earlier
    plants, so that a range has several valid offsets): returns (Parse with no matches, plants)"""
    p = Parse(int(rng.integers(1 << 30)))
    alpha = int(rng.choice([2, 4, 16, 64, 256]))
    plants = []
    while len(p.buf) < n:
        p.rand(int(rng.integers(0, 300)), alpha)
        pos = len(p.buf)
        if pos < 8:
            continue
        ml = int(min(rng.choice([4, 8, 30, 200, 3000]) + rng.integers(0, 8), n - pos))
        if ml < 4:
            break
        off = int(rng.integers(1, min(pos, 65535) + 1)) if rng.random() < 0.7 else int(rng.integers(1, 17))
        p.match(ml, off)
        plants.append((pos, ml, off))
    p.buf = p.buf[:n]
    p.matches = []
    return p, [(a, min(m, n - a), o) for a, m, o in plants if n - a >= 4]


def _random_parse(rng, plants):
    """a valid parse that is not greedy: planted repeats trimmed, cut, sometimes dropped, with a random offset
    among the valid ones"""
    starts = [a for a, _, _ in plants]
    out = []
    for a, ml, off in plants:
        if rng.random() < 0.15:
            continue                                  # left as literals
        s = a + int(rng.integers(0, max(1, ml // 4)))
        e = a + ml - int(rng.integers(0, max(1, ml // 4)))
        while e - s >= 4:
            cut = min(e, s + 4 + int(rng.integers(0, e - s - 3)))
            if e - cut < 4:
                cut = e
            o = off
            j = bisect.bisect_right(starts, s - off) - 1          # the source range inside an earlier plant
            if j >= 0:
                a2, m2, o2 = plants[j]
                if a2 <= s - off and cut - off <= a2 + m2 and off + o2 <= min(s, 65535) and rng.random() < 0.5:
                    o = off + o2
            out.append((s, cut - s, o))
            s = cut + (int(rng.integers(0, 3)) if rng.random() < 0.2 else 0)
    return out


def test_fuzz_random_parses_emu(hook, zref):
    rng = np.random.default_rng(2024)
    frames = 0
    for it in range(200):
        n = int(np.exp(rng.uniform(np.log(1024), np.log(300 * 1024))))
        p, plants = _plant_stream(rng, n)
        p.matches = _random_parse(rng, plants)
        src = p.src()
        frame, r = run_hook(hook, src, p.matches)
        if frame is not None:
            check_frame(hook, zref, frame, n, src)
            frames += 1
    assert frames > 100


# ------------------------------------------------------------------------------------------------
# the shared code tables against the RFC
# ------------------------------------------------------------------------------------------------
def test_shared_code_tables_match_the_rfc():
    text = open(os.path.join(ROOT, "c-blosc_b200", "csrc", "dev_zstd.cuh")).read()

    def table(name):
        m = re.search(r"\b%s\[\d+\]\s*=\s*\{([^}]*)\}" % name, text)
        assert m, name
        return [int(x) for x in m.group(1).replace("\n", " ").split(",") if x.strip()]

    assert table("k_zs_ll_base") == zf.LL_BASE
    assert table("k_zs_ll_bits") == zf.LL_BITS
    assert table("k_zs_ml_base") == zf.ML_BASE
    assert table("k_zs_ml_bits") == zf.ML_BITS
    assert table("k_zs_ll_norm") == zf.LL_NORM
    assert table("k_zs_ml_norm") == zf.ML_NORM
    assert table("k_zs_of_norm") == zf.OF_NORM
    for norm, log in zf.PREDEF.values():               # the RFC's own distributions are complete
        assert sum(abs(x) for x in norm) == 1 << log


# ------------------------------------------------------------------------------------------------
# parser-driven inputs: blosc_compress_ctx with BLOSC_B200_ZSTD=1
# ------------------------------------------------------------------------------------------------
def _raw_middle_data():
    rng = np.random.default_rng(700)
    P = 3000
    per = rng.integers(0, 256, P, dtype=np.uint8)
    b1 = np.resize(per, BLOCK)
    b2 = rng.integers(0, 256, BLOCK, dtype=np.uint8)
    b2[90000:90008] = b2[80000:80008]                 # one planted repeat at a fresh offset
    b3 = np.resize(per, BLOCK)
    return np.concatenate([b1, b2, b3])


def _parser_inputs():
    """(label, src, typesize, shuffle, clevel, forced blocksize)"""
    ins = [("raw_middle", _raw_middle_data(), 1, 0, 5, 3 * BLOCK)]
    for left in (15, 16, 17, 255, 256, 257, 65791, 65792):
        ins.append((f"leftover_{left}", gen("text", BLOCK + left, left), 1, 0, 5, BLOCK))
    ins.append(("long_run", np.zeros(3 * BLOCK, np.uint8), 1, 0, 5, 0))
    rng = np.random.default_rng(701)
    lits = rng.integers(0, 64, 70000, dtype=np.uint8)
    ins.append(("long_literals", np.concatenate([lits, lits[10000:15000]]), 1, 0, 5, 75000))
    for ts in (2, 16, 32):
        ins.append((f"shuffle_ts{ts}", bench_words(300000), ts, 1, 5, 0))
    for ts in (1, 2, 16):
        ins.append((f"bitshuffle_ts{ts}", gen("i32", 300000), ts, 2, 5, 0))
    for cl in (2, 3, 4, 6, 7, 8):
        ins.append((f"clevel_{cl}", gen("text", 400000, cl), 4, 1, cl, 0))
    return ins


def _frames_of(chunk, n):
    """(block, frame bytes, uncompressed length) for the streams of an unsplit chunk that are not stored raw"""
    if chunk[2] & 0x02:
        return
    bs = int.from_bytes(chunk[8:12].tobytes(), "little")
    for b in range((n + bs - 1) // bs):
        st = int.from_bytes(chunk[16 + 4 * b:20 + 4 * b].tobytes(), "little")
        cs = int.from_bytes(chunk[st:st + 4].tobytes(), "little")
        ln = min(bs, n - b * bs)
        if cs != ln:
            yield b, chunk[st + 4:st + 4 + cs], ln


@pytest.fixture(scope="module")
def parser_corpus(hook, zref, ref_if_built, monkeypatch_module):
    """label -> (chunk, [zstd_frame record of every frame]); every chunk decodes here and with the reference"""
    monkeypatch_module.setenv("BLOSC_B200_ZSTD", "1")
    out = {}
    for label, src, ts, shuf, cl, bs in _parser_inputs():
        n = len(src)
        cb, ch = compress(hook, "blosc_compress_ctx", cl, shuf, ts, src, n + 16, "zstd", bs)
        assert cb > 16 and (ch[cb:] == 0xAA).all(), label
        chunk = ch[:cb].copy()
        r, dec = decompress(hook, "blosc_decompress_ctx", chunk, n)
        assert r == n and (dec[:n] == src).all(), label
        if ref_if_built is not None:
            r, dec = decompress(ref_if_built, "blosc_decompress_ctx", chunk, n)
            assert r == n and (dec[:n] == src).all(), label
        infos = [check_frame(hook, zref, fr, ln) for _, fr, ln in _frames_of(chunk, n)]
        out[label] = (chunk, infos)
    return out


@pytest.fixture(scope="module")
def monkeypatch_module():
    mp = pytest.MonkeyPatch()
    yield mp
    mp.undo()


def test_parser_driven_inputs_emu(parser_corpus):
    chunk, infos = parser_corpus["raw_middle"]
    assert len(infos) == 1
    blocks = infos[0].blocks
    assert [b["type"] for b in blocks] == ["compressed", "raw", "compressed"]
    assert _seqs(blocks[2])[0][5] in ("rep1", "rep2", "rep3", "rep2_ll0", "rep3_ll0", "rep1m1_ll0")
    assert any(s[1] == 52 for i in parser_corpus["long_run"][1] for b in i.blocks for s in _seqs(b))
    assert any(s[0] == 35 for i in parser_corpus["long_literals"][1] for b in i.blocks for s in _seqs(b))
    for left in (256, 257, 65791):                     # the leftover block is a frame of its own
        infos = parser_corpus[f"leftover_{left}"][1]
        assert infos[-1].fcs == left, left
    for label, (chunk, infos) in parser_corpus.items():
        assert infos or label.startswith("leftover_1"), label


# ------------------------------------------------------------------------------------------------
# the coverage ledger: every branch of the entropy stage, and that the CPU corpus reaches it
# ------------------------------------------------------------------------------------------------
LEDGER = (
    # block types (the encoder writes no RLE blocks)
    ["block:raw", "block:compressed"]
    # literals: modes, size formats, stream counts, weight encodings
    + ["lit:raw:sf0", "lit:raw:sf1", "lit:raw:sf3", "lit:rle:sf0", "lit:rle:sf1", "lit:rle:sf3",
       "lit:compressed:sf0", "lit:compressed:sf2", "lit:compressed:sf3", "lit:streams:1", "lit:streams:4",
       "weights:direct", "weights:fse", "huffman:clamped_to_11"]
    # sequence counts, table modes, FSE descriptions
    + ["count_bytes:1", "count_bytes:2", "count_bytes:3"]
    + [f"mode:{t}:{m}" for t in ("ll", "of", "ml") for m in ("predefined", "rle", "fse")]
    + ["fse_log_max:ll", "fse_log_max:of", "fse_log_max:ml", "zero_run:>=24", "zero_run:3-23"]
    # repeat offsets
    + [f"case:{c}" for c in ("new", "rep1", "rep2", "rep3", "rep2_ll0", "rep3_ll0", "rep1m1_ll0")]
    + ["case:new_equal_to_rep1_ll0", "raw_block_then_repeat_code"]
    # codes (ML code 0, a 3-byte match, cannot occur: records are >= 4 bytes)
    + [f"ll_code:{c}" for c in range(36)] + [f"ml_code:{c}" for c in range(1, 53)]
    + [f"of_code:{c}" for c in range(17)]
    # frame header
    + ["fcs_bytes:1", "fcs_bytes:2", "fcs_bytes:4", "stored"]
)


def _seen(info, seen):
    prev_raw = False
    for b in info.blocks:
        seen.add(f"block:{b['type']}")
        if b["type"] != "compressed":
            prev_raw = b["type"] == "raw"
            continue
        lit = b["lit"]
        seen.add(f"lit:{lit['type']}:sf{lit['size_format']}")
        if lit["streams"]:
            seen.add(f"lit:streams:{lit['streams']}")
        if lit["weights"]:
            seen.add(f"weights:{lit['weights']}")
        if lit["type"] == "compressed" and lit["max_bits"] == 11 and zf.huffman_depth(lit["literals"]) > 11:
            seen.add("huffman:clamped_to_11")
        sq = b["seq"]
        seen.add(f"count_bytes:{sq['count_bytes']}")
        if sq["count"]:
            for t, m in sq["modes"].items():
                seen.add(f"mode:{t}:{m}")
            for t, lg in sq["logs"].items():
                if lg == zf.MAX_LOG[t]:
                    seen.add(f"fse_log_max:{t}")
            for runs in sq["zero_runs"].values():
                for r in runs:
                    seen.add("zero_run:>=24" if r >= 24 else ("zero_run:3-23" if r >= 3 else "zero_run:<3"))
        for i, s in enumerate(sq["seqs"]):
            seen.add(f"case:{s[5]}")
            if s[5] == "new" and s[6] == 0 and s[4] == s[8]:
                seen.add("case:new_equal_to_rep1_ll0")
            seen.update((f"ll_code:{s[0]}", f"ml_code:{s[1]}", f"of_code:{s[2]}"))
            if i == 0 and prev_raw and s[5] != "new":
                seen.add("raw_block_then_repeat_code")
        prev_raw = False
    seen.add(f"fcs_bytes:{info.fcs_bytes}")


def test_coverage_ledger_emu(corpus, parser_corpus):
    seen = set()
    for src, info, r in corpus.values():
        if info is None:
            seen.add("stored")
        else:
            _seen(info, seen)
    for chunk, infos in parser_corpus.values():
        for info in infos:
            _seen(info, seen)
    missing = [x for x in LEDGER if x not in seen]
    assert not missing, missing


# ------------------------------------------------------------------------------------------------
# GPU: zparse_kernel / zenc_kernel under their own launch shape give the emulator's bytes
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_chunks(hook, monkeypatch_module):
    monkeypatch_module.setenv("BLOSC_B200_ZSTD", "1")
    out = []
    for label, src, ts, shuf, cl, bs in _parser_inputs():
        cb, ch = compress(hook, "blosc_compress_ctx", cl, shuf, ts, src, len(src) + 16, "zstd", bs)
        assert cb > 16
        out.append((label, src, ts, shuf, cl, bs, ch[:cb].copy()))
    return out


@pytest.mark.gpu
def test_parser_driven_inputs_equal_emulator_gpu(pkg, cuda, ref_if_built, emu_chunks):
    torch = cuda
    for label, src, ts, shuf, cl, bs, want in emu_chunks:
        n = len(src)
        dest = np.full(n + 16 + 64, 0xAA, np.uint8)
        cb = pkg.compress_ctx(cl, shuf, ts, n, src, dest, n + 16, "zstd", bs)
        assert cb == len(want) and (dest[:cb] == want).all() and (dest[cb:] == 0xAA).all(), label
        d_src = torch.from_numpy(src).cuda()
        d_dst = torch.full((n + 16 + 64,), 0xAA, dtype=torch.uint8, device="cuda")
        assert pkg.compress_ctx(cl, shuf, ts, n, d_src, d_dst, n + 16, "zstd", bs) == cb, label
        h = d_dst.cpu().numpy()
        assert (h[:cb] == want).all() and (h[cb:] == 0xAA).all(), label
        d_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
        assert pkg.decompress_ctx(d_dst, d_out, n) == n and torch.equal(d_out, d_src), label
        out = np.zeros(n, np.uint8)
        assert pkg.decompress_ctx(dest, out, n) == n and (out == src).all(), label
        if ref_if_built is not None:
            r, dec = decompress(ref_if_built, "blosc_decompress_ctx", want, n)
            assert r == n and (dec[:n] == src).all(), label


@pytest.mark.gpu
def test_two_threads_compress_at_once_gpu(pkg, cuda, emu_chunks):
    """two host threads, two workspaces, different inputs at the same time: both get the emulator's bytes"""
    picks = [c for c in emu_chunks if c[0] in ("raw_middle", "clevel_7", "shuffle_ts16", "long_literals")]
    errors = []

    def work(items):
        try:
            for _ in range(3):
                for label, src, ts, shuf, cl, bs, want in items:
                    n = len(src)
                    dest = np.full(n + 16 + 64, 0xAA, np.uint8)
                    cb = pkg.compress_ctx(cl, shuf, ts, n, src, dest, n + 16, "zstd", bs)
                    if cb != len(want) or not (dest[:cb] == want).all() or not (dest[cb:] == 0xAA).all():
                        errors.append(label)
        except Exception as e:                        # reported below, on the main thread
            errors.append(repr(e))

    th = [threading.Thread(target=work, args=(picks[i::2],)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors

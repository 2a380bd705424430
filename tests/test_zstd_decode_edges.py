"""The zstd decoder (csrc/dev_zstd.cuh, zs_frame_serial) branch by branch, on frames written to order.

tests/zstd_write.py writes frames from explicit descriptions, so every decode path is reached on purpose: treeless
literals, repeat table modes across raw and RLE blocks, every literals size format at its thresholds, four-stream
sections whose fourth stream is empty, 1 to 255 Huffman weights, FSE descriptions with zero runs and "-1"
probabilities at every accuracy log, the three sequence-count forms, all repeat-offset cases, every window
descriptor, dictionary-ID and content-size form, checksums, skippable frames and concatenated frames.

Accept corpus: each frame is decoded by zstd_frame.py (an independent, strict RFC 8878 decoder), by this library's
decoder (emu_zstd_decode, at cap = n and n + 9 with a canary after cap, and n - 1 refused) and, when oracle/_ref is
built, by ZSTD_decompress.  Then the structure the scenario exists for is asserted from zstd_frame's record.

Reject corpus: frames that are valid except for one defect, each naming the `return ZS_FAIL` line that must refuse
it; together with single-byte damage and truncations of small valid frames, the ledger test asserts that every
ZS_FAIL line of dev_zstd.cuh is reached.  The reference's verdicts and bytes for the crafted corpus are pinned in
tests/golden/reference_results.json, so they are checked where oracle/_ref is absent.

The verdict rule: never accept a frame that ZSTD_decompress rejects; never reject an RFC-valid frame that it
accepts; reject an RFC-invalid frame that it accepts only when the case is on STRICT below, each entry pinned by a
test of its own."""
import ctypes as C
import os
import random
import struct

import numpy as np
import pytest

import zstd_frame as zf
import zstd_write as zw
from datagen import assert_pinned, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "c-blosc_b200", "csrc", "dev_zstd.cuh")
BLOCK = 128 * 1024

# RFC-invalid frames that ZSTD_decompress (zstd 1.5.6) accepts and this decoder refuses, on purpose
STRICT = {
    "huf_12_bits": "Huffman codes of 12 bits: RFC 8878 limits Huffman codes to 11 bits (Max_Number_of_Bits); zstd "
                   "1.5.6 decodes up to 12",
    "raw_block_over_128k": "a raw block above 128 KiB (Block_Maximum_Size); the one-shot ZSTD_decompress never "
                           "checks a raw block's size",
    "rle_block_over_128k": "an RLE block above 128 KiB, likewise unchecked by ZSTD_decompress",
    "compressed_output_over_128k": "a compressed block that decodes to more than 128 KiB; ZSTD_decompress does not "
                                   "check how much a block produces",
    "literal_stream_not_used_up": "a Huffman literal stream with bits left over below its last code: zstd 1.5.6's "
                                  "Huffman decoders do not check that a stream is used up exactly",
}


# ------------------------------------------------------------------------------------------------
# the three decoders
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def zemu(emu):
    emu.emu_zstd_decode.restype = C.c_int
    emu.emu_zstd_decode.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    emu.emu_zstd_fail_line.restype = C.c_int
    return emu


@pytest.fixture(scope="module")
def zref(ref_if_built):
    r = ref_if_built
    if r is None or not hasattr(r, "ZSTD_decompress"):
        return None
    r.ZSTD_decompress.restype = C.c_size_t
    r.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    r.ZSTD_isError.restype = C.c_uint
    r.ZSTD_isError.argtypes = [C.c_size_t]
    return r


def emu_decode(emu, frame, cap):
    """(return code, bytes written, canary after cap intact, fail line)"""
    src = np.frombuffer(bytes(frame) + b"\0", np.uint8).copy()
    out = np.full(cap + 64, 0x77, np.uint8)
    r = emu.emu_zstd_decode(ptr(src), len(frame), ptr(out), cap)
    return r, out[:max(r, 0)].tobytes(), bool((out[cap:] == 0x77).all()), emu.emu_zstd_fail_line()


def ref_decode(zref, frame, cap):
    """ZSTD_decompress: the bytes, or None for an error"""
    src = np.frombuffer(bytes(frame) + b"\0", np.uint8).copy()
    out = np.zeros(cap + 64, np.uint8)
    r = zref.ZSTD_decompress(ptr(out), cap, ptr(src), len(frame))
    return None if zref.ZSTD_isError(r) else out[:r].tobytes()


def strict_decode(frame):
    """zstd_frame's verdict: (bytes, infos) or None"""
    try:
        return zf.decode_stream(frame)
    except (zf.ZstdError, IndexError):
        return None


# ------------------------------------------------------------------------------------------------
# description helpers
# ------------------------------------------------------------------------------------------------
def cblk(lit, seqs=(), modes=None, **kw):
    return dict(type="compressed", lit=lit, seqs=list(seqs), modes=modes or {}, **kw)


def raw(data):
    return dict(type="raw", data=bytes(data))


def rle(byte, size):
    return dict(type="rle", byte=byte, size=size)


def L(mode, data, **kw):
    return dict(mode=mode, data=bytes(data), **kw)


def skewed(n, nsym, seed=0):
    """n bytes over nsym symbols with unequal frequencies (a Huffman code of several lengths)"""
    rng = random.Random(seed)
    pool = [s for s in range(nsym) for _ in range(s % 5 + 1)]
    base = bytes(range(nsym))
    return (base + bytes(rng.choice(pool) for _ in range(max(n - nsym, 0))))[:n]


def last_block(infos, k=-1):
    return infos[-1].blocks[k]


ACCEPT = {}           # name -> (frame, content, check(infos))


def accept(name, frame_and_content, check=None):
    assert name not in ACCEPT
    ACCEPT[name] = (frame_and_content[0], frame_and_content[1], check or (lambda infos: None))


def _lit_check(mode, sf, streams=None, regen=None, weights=None, nweights=None):
    def check(infos):
        lit = last_block(infos)["lit"]
        assert lit["type"] == mode and lit["size_format"] == sf, lit["type"]
        if streams is not None:
            assert lit["streams"] == streams
        if regen is not None:
            assert lit["regen"] == regen
        if weights is not None:
            assert lit["weights"] == weights
        if nweights is not None:
            assert sum(1 for x in lit["lengths"] if x) == nweights
    return check


def _build_accept():
    # blocks: raw, RLE, empty ones
    accept("raw_block", zw.frame([raw(b"raw bytes")]), lambda i: [b["type"] for b in i[0].blocks] == ["raw"])
    accept("rle_block", zw.frame([rle(7, 300)]), lambda i: i[0].blocks[0]["type"] == "rle")
    accept("empty_raw_block", zw.frame([raw(b"")]), lambda i: i[0].blocks[0]["size"] == 0)
    accept("empty_rle_block", zw.frame([raw(b"ab"), rle(9, 0), raw(b"c")]), lambda i: i[0].blocks[1]["out"] == 0)
    accept("empty_compressed_block", zw.frame([raw(b"xy"), cblk(L("raw", b""))]), lambda i: i[0].blocks[1]["out"] == 0)
    accept("empty_frame_no_fcs", zw.frame([raw(b"")], fcs=None), lambda i: i[0].fcs is None)
    # literals size formats at their thresholds
    for n in (0, 31, 32, 4095, 4096, 70000):
        accept(f"raw_lits_{n}", zw.frame([cblk(L("raw", skewed(n, 40, n)))]),
               _lit_check("raw", 0 if n < 32 else (1 if n < 4096 else 3), regen=n))
        accept(f"rle_lits_{n}", zw.frame([cblk(L("rle", bytes([5]) * n, byte=5))]),
               _lit_check("rle", 0 if n < 32 else (1 if n < 4096 else 3), regen=n))
    accept("raw_lits_sf2", zw.frame([cblk(L("raw", b"abc", sf=2))]), _lit_check("raw", 0, regen=3))
    for n, st, sf in ((1023, 1, 0), (1023, 4, 1), (1024, 4, 2), (16383, 4, 2), (16384, 4, 3), (BLOCK, 4, 3)):
        accept(f"huf_lits_{n}_{st}", zw.frame([cblk(L("huf", skewed(n, 60, n), streams=st))]),
               _lit_check("compressed", sf, streams=st, regen=n))
    for n in (6, 7, 9, 10):                                   # 6 and 9: the fourth stream is empty
        accept(f"huf_4streams_{n}", zw.frame([cblk(L("huf", skewed(n, 4, n), streams=4, sf=1))]),
               _lit_check("compressed", 1, streams=4, regen=n))
    # Huffman weights: direct and FSE-coded, 1 to 255 explicit weights
    accept("weights_direct_1", zw.frame([cblk(L("huf", b"abab" * 5, wmode="direct"))]),
           _lit_check("compressed", 0, weights="direct", nweights=2))
    accept("weights_direct_128", zw.frame([cblk(L("huf", skewed(600, 129, 3), wmode="direct", streams=4))]),
           _lit_check("compressed", 1, weights="direct", nweights=129))
    for k in (5, 17, 100, 200, 256):
        data = skewed(max(4 * k, 40), k, k)
        accept(f"weights_fse_{k - 1}", zw.frame([cblk(L("huf", data, wmode="fse", streams=4))]),
               _lit_check("compressed", 1 if len(data) < 1024 else 2, weights="fse", nweights=k))
    w = zw.weights_for(skewed(300, 40, 1))
    wl = w[:max(s for s in range(256) if w[s])]
    hist = [wl.count(v) for v in range(13)]
    for log in (5, 6):
        accept(f"weights_fse_log{log}", zw.frame([cblk(L("huf", skewed(300, 40, 1), weights=w, wmode="fse",
                                                          wnorm=(zw.normalize(hist, log), log), streams=4))]),
               lambda i, log=log: last_block(i)["lit"]["weights_log"] == log)
    # treeless literals after a raw block and after an RLE block
    d = skewed(200, 30, 5)
    accept("treeless_after_raw", zw.frame([cblk(L("huf", d, streams=4)), raw(b"r" * 10), cblk(L("treeless", d[:50],
                                                                                                  streams=1))]),
           lambda i: i[0].blocks[2]["lit"]["type"] == "treeless" and i[0].blocks[2]["lit"]["streams"] == 1)
    accept("treeless_4streams_after_rle", zw.frame([cblk(L("huf", d, streams=1)), rle(1, 5),
                                                    cblk(L("treeless", d[::-1], streams=4))]),
           lambda i: i[0].blocks[2]["lit"]["type"] == "treeless" and i[0].blocks[2]["lit"]["streams"] == 4)
    # sequence tables: every mode, repeat across raw / RLE blocks, FSE descriptions at every accuracy log
    lits = skewed(64, 20, 2)
    seqs = [(10, 8, 3 + 5), (6, 20, 3 + 9), (3, 5, 1), (0, 4, 2), (12, 33, 3 + 40)]
    modes_fse = {"ll": ("fse", None, 5), "of": ("fse", None, 5), "ml": ("fse", None, 5)}
    accept("tables_predefined", zw.frame([cblk(L("raw", lits), seqs)]),
           lambda i: set(last_block(i)["seq"]["modes"].values()) == {"predefined"})
    accept("tables_fse", zw.frame([cblk(L("raw", lits), seqs, modes_fse)]),
           lambda i: set(last_block(i)["seq"]["modes"].values()) == {"fse"})
    accept("tables_rle", zw.frame([cblk(L("raw", lits), [(4, 7, 3 + 2), (4, 7, 3 + 3)],
                                        {"ll": ("rle", 4), "of": ("rle", 2), "ml": ("rle", 4)})]),
           lambda i: set(last_block(i)["seq"]["modes"].values()) == {"rle"})
    rep = {"ll": "repeat", "of": "repeat", "ml": "repeat"}
    accept("tables_repeat_across_raw", zw.frame([cblk(L("raw", lits), seqs, modes_fse), raw(b"between"),
                                                 cblk(L("raw", lits[:40]), seqs[:3], rep)]),
           lambda i: set(i[0].blocks[2]["seq"]["modes"].values()) == {"repeat"})
    accept("tables_repeat_predefined_after_rle", zw.frame([cblk(L("raw", lits), seqs), rle(3, 9),
                                                           cblk(L("raw", lits[:40]), seqs[:3], rep)]),
           lambda i: set(i[0].blocks[2]["seq"]["modes"].values()) == {"repeat"})
    accept("tables_repeat_rle", zw.frame([cblk(L("raw", lits), [(4, 7, 3 + 2)], {"ll": ("rle", 4), "of": ("rle", 2),
                                                                                "ml": ("rle", 4)}),
                                          cblk(L("raw", lits), [(4, 7, 3 + 2), (4, 7, 3 + 3)], rep)]),
           lambda i: set(i[0].blocks[1]["seq"]["modes"].values()) == {"repeat"})
    for name, maxlog in (("ll", 9), ("of", 8), ("ml", 9)):
        for log in range(5, maxlog + 1):
            m = {name: ("fse", None, log)}
            accept(f"fse_{name}_log{log}", zw.frame([cblk(L("raw", lits), seqs, m)]),
                   lambda i, name=name, log=log: last_block(i)["seq"]["logs"][name] == log)
    # FSE description corners: zero runs of 3, of 6 (two repeat flags), of 24 and more, "-1" probabilities
    def ll_norm(points, log, minus=()):
        n = [0] * 36
        for k, v in points.items():
            n[k] = v
        for k in minus:
            n[k] = -1
        return n
    # LL codes used: 0, 3, 6, 10, 12 (and 22).  13..16 are a zero and a run of 3; 14..21 a zero and a run of 7
    accept("fse_zero_run_3", zw.frame([cblk(L("raw", lits), seqs, {"ll": ("fse", ll_norm({0: 8, 3: 4, 6: 4, 10: 4,
                                                                                           12: 4, 17: 8}, 5), 5)})]),
           lambda i: 3 in last_block(i)["seq"]["zero_runs"]["ll"])
    seqs_far = [(10, 8, 3 + 5), (6, 20, 3 + 9), (3, 5, 1), (0, 4, 2), (32, 33, 3 + 40)]   # ll code 22
    accept("fse_zero_run_7", zw.frame([cblk(L("raw", lits), seqs_far, {"ll": ("fse", ll_norm({0: 8, 3: 8, 6: 4, 10: 4,
                                                                                               13: 4, 22: 4}, 5), 5)})]),
           lambda i: 7 in last_block(i)["seq"]["zero_runs"]["ll"])
    ml_seqs = [(10, 3, 3 + 5), (6, 4, 3 + 9), (3, 10, 1), (0, 259, 2), (12, 4, 3 + 40)]    # ML codes 0, 1, 7, 44
    mln = [0] * 53
    for c in (0, 1, 7, 44):
        mln[c] = 16
    accept("fse_zero_run_24", zw.frame([cblk(L("raw", lits), ml_seqs, {"ml": ("fse", mln, 6)})]),
           lambda i: max(last_block(i)["seq"]["zero_runs"]["ml"]) >= 24)
    accept("fse_minus_one", zw.frame([cblk(L("raw", lits), seqs, {"ll": ("fse", ll_norm({0: 8, 3: 8, 6: 8, 10: 5},
                                                                                        5, minus=(12, 13, 14)), 5)})]),
           lambda i: last_block(i)["seq"]["modes"]["ll"] == "fse")
    # sequence-count forms
    accept("seq_count_0", zw.frame([cblk(L("raw", b"only literals"))]),
           lambda i: last_block(i)["seq"]["count"] == 0)
    for ns in (1, 127, 128, 0x7EFF, 0x7F00, 0x7F00 + 300):
        m = {"ll": ("rle", 0), "of": ("rle", 2), "ml": ("rle", 0)}
        accept(f"seq_count_{ns}", zw.frame([raw(b"seed1234"), cblk(L("raw", b""), [(0, 3, 4)] * ns, m)]),
               lambda i, ns=ns: last_block(i)["seq"]["count"] == ns and
               last_block(i)["seq"]["count_bytes"] == (1 if ns < 128 else (2 if ns < 0x7F00 else 3)))
    # offsets: the largest code the output allows, every repeat-offset case, rep1 - 1
    big = bytes(random.Random(4).getrandbits(8) for _ in range(BLOCK))
    accept("offset_code_17", zw.frame([raw(big), raw(big[:9000]), cblk(L("raw", b"q"), [(1, 40, 3 + BLOCK + 8000)])]),
           lambda i: last_block(i)["seq"]["seqs"][0][2] == 17)
    accept("offset_code_16", zw.frame([raw(big[:70000]), cblk(L("raw", b"q"), [(1, 40, 3 + 65600)])]),
           lambda i: last_block(i)["seq"]["seqs"][0][2] == 16)
    reps = [(16, 4, 3 + 11), (2, 4, 3 + 5), (1, 4, 1), (1, 4, 2), (1, 4, 3), (0, 4, 1), (0, 4, 2), (0, 4, 3),
            (2, 5, 3 + 7), (0, 4, 3)]
    accept("repeat_offsets", zw.frame([cblk(L("raw", skewed(40, 26, 9)), reps)]),
           lambda i: {s[5] for s in last_block(i)["seq"]["seqs"]} >=
           {"new", "rep1", "rep2", "rep3", "rep2_ll0", "rep3_ll0", "rep1m1_ll0"})
    accept("repeat_offsets_across_blocks", zw.frame([cblk(L("raw", skewed(40, 26, 9)), reps[:2]), raw(b"raw"),
                                                     cblk(L("raw", b"zz"), [(1, 4, 2), (0, 5, 3)])]),
           lambda i: [s[5] for s in i[0].blocks[2]["seq"]["seqs"]] == ["rep2", "rep1m1_ll0"])
    # frame header forms: windows, dictionary IDs, content sizes, checksums
    for wd in range(0, 22 * 8, 1):
        if wd % 8 and wd // 8 not in (0, 7, 21) and wd % 8 not in (7,):
            continue
        accept(f"window_{wd}", zw.frame([cblk(L("raw", b"window!"), [(7, 5, 3 + 7)])], wd=wd),
               lambda i, wd=wd: i[0].window == (1 << ((wd >> 3) + 10)) + ((1 << ((wd >> 3) + 10)) >> 3) * (wd & 7))
    for db in (1, 2, 4):
        accept(f"did_zero_{db}", zw.frame([raw(b"dictionary id 0")], did_bytes=db),
               lambda i, db=db: i[0].did_bytes == db)
    for fb, n in ((1, 200), (2, 256), (2, 65791), (4, 70000), (8, 300)):
        single = fb == 1
        accept(f"fcs_{fb}_{n}", zw.frame([raw(big[:n])], fcs_bytes=fb, single=single),
               lambda i, fb=fb, n=n: i[0].fcs_bytes == fb and i[0].fcs == n)
    accept("single_segment_compressed", zw.frame([cblk(L("raw", big[:300]), [(300, 30, 3 + 100)])], single=True,
                                                 fcs_bytes=2),
           lambda i: i[0].single_segment and i[0].blocks[0]["type"] == "compressed")
    for n in (0, 31, 32, 33, 100):
        accept(f"checksum_{n}", zw.frame([raw(big[:n])], checksum=True),
               lambda i: i[0].checksum)
    accept("checksum_compressed", zw.frame([cblk(L("raw", lits), seqs)], checksum=True, fcs=None),
           lambda i: i[0].checksum and i[0].fcs is None)
    # several frames in one input (ZSTD_decompressMultiFrame)
    f1, c1 = zw.frame([cblk(L("raw", lits), seqs, modes_fse)], checksum=True)
    f2, c2 = zw.frame([cblk(L("huf", skewed(100, 12, 1), streams=4)), rle(2, 30)], fcs=None, checksum=True)
    accept("two_frames", (f1 + f2, c1 + c2), lambda i: len(i) == 2)
    accept("frame_then_skippable", (f1 + zw.skippable(b"skip me"), c1), lambda i: len(i) == 1)
    accept("skippable_then_frames", (zw.skippable(b"", 15) + f2 + f1, c2 + c1), lambda i: len(i) == 2)
    accept("skippable_only", (zw.skippable(b"nothing"), b""), lambda i: len(i) == 0)
    # a compressed block and literals as large as a small window allows
    accept("block_at_window", zw.frame([cblk(L("raw", big[:1021]))], wd=0),
           lambda i: i[0].window == 1024 and i[0].blocks[0]["size"] == 1024)
    accept("block_at_window_mantissa_1", zw.frame([cblk(L("raw", big[:1149]))], wd=1),
           lambda i: i[0].window == 1152 and i[0].blocks[0]["size"] == 1152)
    accept("block_at_window_64k", zw.frame([cblk(L("raw", big[:65532]))], wd=0x30),
           lambda i: i[0].window == 65536 and i[0].blocks[0]["size"] == 65536)
    accept("block_at_window_72k", zw.frame([cblk(L("rle", bytes(73728), byte=0))], wd=0x31),
           lambda i: i[0].window == 73728 and i[0].blocks[0]["lit"]["regen"] == 73728)


_build_accept()


def test_xxh64_published_vectors():
    assert zw.xxh64(b"") == 0xEF46DB3751D8E999
    assert zw.xxh64(b"a") == 0xD24EC4F1A98C6E5B
    assert zw.xxh64(b"abc") == 0x44BC2CF5AD770999
    assert zw.xxh64(b"", 1) == 0xD5AFBA1336A3BE4B


@pytest.mark.parametrize("name", sorted(ACCEPT))
def test_accept_corpus_emu(zemu, zref, name):
    frame, content, check = ACCEPT[name]
    got = strict_decode(frame)
    assert got is not None, "zstd_frame refuses it"
    assert got[0] == content
    assert check(got[1]) is not False, "the frame does not have the structure it is for"
    n = len(content)
    for cap in (n, n + 9):
        r, out, canary, _ = emu_decode(zemu, frame, cap)
        assert r == n and out == content and canary, (cap, r)
    if n > 0:
        r, _, canary, _ = emu_decode(zemu, frame, n - 1)
        assert r == -1 and canary
    if zref is not None:
        assert ref_decode(zref, frame, n) == content
        if n > 0:
            assert ref_decode(zref, frame, n - 1) is None


# ------------------------------------------------------------------------------------------------
# reject corpus: one defect each, and the ZS_FAIL line that must catch it
# ------------------------------------------------------------------------------------------------
def fail_lines():
    """{line number: text} of every `return ZS_FAIL` in dev_zstd.cuh"""
    out = {}
    for i, line in enumerate(open(SRC).read().split("\n"), 1):
        if "ZS_FAIL" in line and "#define" not in line:
            out[i] = line
    return out


def line_of(fragment):
    hits = [k for k, t in fail_lines().items() if fragment in t]
    assert len(hits) == 1, (fragment, hits)
    return hits[0]


REJECT = {}           # name -> (frame, cap, fragment of the refusing line)


def reject(name, frame, fragment, cap=None):
    assert name not in REJECT
    if isinstance(frame, tuple):
        frame, content = frame
        cap = len(content) if cap is None else cap
    REJECT[name] = (bytes(frame), 4096 if cap is None else cap, fragment)


def patch(frame, pos, value):
    b = bytearray(frame)
    b[pos] = value
    return bytes(b)


def _build_reject():
    lits = skewed(64, 20, 2)
    seqs = [(10, 8, 3 + 5), (6, 20, 3 + 9), (3, 5, 1), (0, 4, 2), (12, 33, 3 + 40)]
    good, content = zw.frame([cblk(L("raw", lits), seqs)], fcs=None)
    # frame header
    reject("too_short", good[:4], "csize - ip < 5")
    reject("short_frame", good[:5], "csize < 6")
    reject("bad_magic", patch(good, 0, 0x29), "!= 0xFD2FB528u")
    reject("reserved_fhd_bit", zw.frame([raw(b"abc")], reserved=True), "fhd & 0x08")
    reject("window_above_2g", zw.frame([raw(b"abc")], wd=22 * 8), "> 21) return")
    reject("did_past_end", zw.MAGIC.to_bytes(4, "little") + b"\x03\x00\x00", "ip + did_bytes > csize")
    reject("did_nonzero", zw.frame([raw(b"abc")], did_bytes=2)[0][:6] + b"\x00\x01" +
           zw.frame([raw(b"abc")], did_bytes=2)[0][8:], "if (in[ip + i])")
    reject("fcs_past_end", zw.MAGIC.to_bytes(4, "little") + b"\xc0\x00\x00\x00", "ip + fcs_bytes > csize")
    reject("fcs_above_cap", zw.frame([raw(b"abcdef")]), "fcs > (u64)cap", cap=5)
    reject("fcs_mismatch", zw.frame([raw(b"abcdef")], content=b"abcdefg"), "(u64)op != fcs")
    reject("fcs2_without_256", zw.frame([raw(bytes(300))], fcs_bytes=2)[0][:6] + (300).to_bytes(2, "little") +
           zw.frame([raw(bytes(300))], fcs_bytes=2)[0][8:], "(u64)op != fcs", cap=600)
    # blocks
    reject("no_block_header", good[:7], "ip + 3 > csize")
    reject("reserved_block_type", zw.MAGIC.to_bytes(4, "little") + b"\x00\x00" + bytes([0b111, 0, 0]), "btype == 3")
    reject("raw_past_end", zw.frame([raw(b"abcdef")])[0][:-2], "bsize > ZS_BLOCKMAX || ip + bsize > csize || op")
    reject("rle_past_end", zw.frame([rle(1, 10)])[0][:-1], "bsize > ZS_BLOCKMAX || ip + 1 > csize")
    reject("raw_over_cap", zw.frame([raw(b"abcdef")], fcs=None), "bsize > ZS_BLOCKMAX || ip + bsize > csize || op",
           cap=5)
    reject("compressed_past_end", good[:-1], "bsize > bmax || bsize < 2")
    reject("compressed_size_1", zw.frame([dict(cblk(L("raw", b"")), bsize=1)], fcs=None)[0][:-1],
           "bsize > bmax || bsize < 2")
    big = bytes(random.Random(4).getrandbits(8) for _ in range(3000))
    reject("compressed_above_window", zw.frame([cblk(L("raw", big[:2000]))], wd=0), "bsize > bmax || bsize < 2")
    reject("literals_above_window", zw.frame([cblk(L("rle", bytes(2000), byte=0))], wd=0), "regen > bmax")
    reject("literals_above_window_64k", zw.frame([cblk(L("rle", bytes(70000), byte=0))], wd=0x30), "regen > bmax")
    big70 = bytes(random.Random(5).getrandbits(8) for _ in range(70000))
    reject("compressed_above_window_64k", zw.frame([raw(big70[:100]), cblk(L("raw", big70[:65600]))], wd=0x30),
           "bsize > bmax || bsize < 2")
    reject("compressed_above_single_segment_fcs", zw.frame([cblk(L("raw", big[:90]))], single=True, fcs_bytes=1),
           "bsize > bmax || bsize < 2")
    reject("checksum_missing", zw.frame([raw(b"abc")], checksum=True)[0][:-2], "ip + 4 > csize")
    reject("checksum_wrong", zw.frame([raw(b"abc")], checksum=True, bad_checksum=True), "zs_xxh64(out, op) != want")
    # literals section
    def blk(body, n=None):
        return zw.MAGIC.to_bytes(4, "little") + b"\x00\x00" + (1 | 4 | (len(body) << 3)).to_bytes(3, "little") + body
    reject("raw_lits_sf3_cut", blk(bytes([0b1100, 0])), "if (bend < 3) return ZS_FAIL")
    reject("raw_lits_past_block", blk(bytes([31 << 3]) + b"abc\x00"), "hdr + regen > bend")
    reject("rle_lits_past_block", blk(bytes([1 | (4 << 3)])), "bsize > bmax || bsize < 2")
    reject("huf_header_short", blk(bytes([2 | (3 << 2), 0])), "bend < (sf < 2 ? 3 : sf + 2)")
    reject("huf_comp_past_block", blk((2 | (0 << 2) | (5 << 4) | (60 << 14)).to_bytes(3, "little") + b"\x00"),
           "hdr + comp > bend")
    # a treeless block with no earlier tree: the tree of a first frame does not carry into a second
    d = skewed(40, 6, 1)
    fa, ca = zw.frame([cblk(L("huf", d))])
    st = {"rep": [1, 4, 8]}
    zw.literals_section(L("huf", d), st)
    tl = zw.literals_section(L("treeless", d[:20], streams=1), st) + b"\x00"
    reject("treeless_without_table", (fa + blk(tl), ca + d[:20]), "treeless block without a previous table")
    reject("four_streams_under_6", (blk(zw.literals_section(L("huf", d[:5], streams=4, sf=1),
                                                             {"rep": [1, 4, 8]}) + b"\x00"), d[:5]),
           "regen < 6) return")
    huf1 = zw.literals_section(L("huf", d[:30], streams=1), {"rep": [1, 4, 8]})
    reject("single_stream_no_end_mark", (blk(huf1[:-1] + b"\x00" + b"\x00"), d[:30]), "zs_back_init(L.s[0], q, qlen)")
    reject("huf_tree_bad", (blk(huf1[:3] + b"\x00" + huf1[4:] + b"\x00"), d[:30]), "hb == 0 || used > len")
    # FSE descriptions cut short, and Huffman tree descriptions one defect each
    reject("fse_description_cut", blk(b"\x00\x01\x80" + zw.fse_description([1] * 32, 5)[:4]), "pos > total")
    reject("fse_description_cut_at_byte", blk(b"\x00\x01\x80" + zw.fse_description([1] * 32, 5)[:3]), "avail <= 0")
    reject("fse_zero_flags_cut", blk(b"\x00\x01\x80" + zw.fse_description([1, 0, 0, 0, 0, 31], 5)[:2]),
           "pos + 2 > total")
    reject("huf_comp_0", blk((2 | (10 << 4)).to_bytes(3, "little") + b"\x00"), "no tree description")
    reject("fse_description_missing", blk(b"\x00\x01\x80"), "no description")
    d4 = skewed(60, 9, 3)
    sec = zw.literals_section(L("huf", d4, streams=4, wmode="fse"), {"rep": [1, 4, 8]})
    hb = sec[3]
    h = len(zw.fse_description(*_weights_norm(d4)))
    reject("huf_weights_no_stream", (blk(sec[:3] + bytes([h]) + sec[4:] + b"\x00"), d4), "h < 0 || h >= hb")
    reject("huf_weights_no_end_mark", (blk(patch(sec, 3 + hb, 0) + b"\x00"), d4), "zs_back_init(b, p + 1 + h")
    rnd = random.Random(0)
    wdesc = zw.fse_description([0, 60, 4], 6)             # weight 1 almost always: a weight costs about a bit
    wstream = bytes(rnd.getrandbits(8) for _ in range(39)) + b"\x01"
    wtree = bytes([len(wdesc) + len(wstream)]) + wdesc + wstream + b"\x01"
    reject("huf_weights_over_255", blk((2 | (10 << 4) | (len(wtree) << 14)).to_bytes(3, "little") + wtree + b"\x00"),
           "first state")
    reject("huf_weights_all_zero", blk((2 | (10 << 4) | (3 << 14)).to_bytes(3, "little") + b"\x82\x00\x01\x00"),
           "sum == 0")
    reject("rle_lits_no_byte", blk(bytes([1 | (1 << 2) | (3 << 4), 0])), "hdr + 1 > bend")
    tree = 1 + hb
    comp = tree + 5
    reject("four_streams_no_jump_table", (blk((2 | (1 << 2) | (len(d4) << 4) | (comp << 14)).to_bytes(3, "little") +
                                              sec[3:3 + comp] + b"\x00"), d4), "qlen < 6")
    l1 = sec[3 + tree] | sec[4 + tree] << 8
    reject("stream_no_end_mark", (blk(patch(sec, 3 + tree + 6 + l1 - 1, 0) + b"\x00"), d4), "zs_back_init(L.s[2]")
    # sequences section
    reject("no_sequences_section", blk(bytes([3 << 3]) + b"abc"), "no sequence count")
    reject("count2_cut", blk(bytes([0]) + b"\x80"), "lp + 1 > bend")
    reject("count3_cut", blk(bytes([0]) + b"\xff\x00"), "lp + 2 > bend")
    reject("no_modes_byte", blk(bytes([0]) + b"\x01"), "no modes byte")
    reject("ml_repeat_without_table", (patch(good, 6 + 3 + 2 + 64 + 1, 0x0C), content), "ML table")
    reject("modes_reserved", (patch(good, 6 + 3 + 2 + 64 + 1, 0x01), content), "modes & 3")
    reject("bytes_after_no_sequences", blk(bytes([0]) + b"\x00\x00"), "lp != bend")
    m_rle = {"ll": ("rle", 4), "of": ("rle", 2), "ml": ("rle", 4)}
    fr, c = zw.frame([cblk(L("raw", lits), [(4, 7, 3 + 2)], m_rle)], fcs=None)
    reject("rle_symbol_out_of_range", (patch(fr, 6 + 3 + 2 + 64 + 2, 36), c), "p[0] > maxsym")
    reject("repeat_without_table", (patch(good, 6 + 3 + 2 + 64 + 1, 0x30), content), "OF table")
    fr, c = zw.frame([cblk(L("raw", lits), seqs, {"ml": ("fse", None, 6)})], fcs=None)
    reject("fse_log_too_big", (patch(fr, 6 + 3 + 2 + 64 + 2, 0x0f), c), "alog > maxlog")
    st = {"rep": [1, 4, 8]}
    ls = zw.literals_section(L("raw", lits), st)
    ss = zw.sequences_section(seqs, {}, st)
    reject("seq_stream_cut", (blk(ls + ss[:2] + ss[4:]), content), "        if (sb.pos < 0) return ZS_FAIL;")
    reject("seq_stream_left_over", (blk(ls + ss[:2] + b"\x5a" + ss[2:]), content), "sb.pos != 0")
    reject("offset_before_frame", _bad_offset(), "offset > (u32)op")
    reject("rep1_minus_1_zero", _rep1m1_zero(), "offset == 0")
    reject("sequences_over_cap", zw.frame([cblk(L("raw", lits), seqs)], fcs=None), "(u64)op + ll + ml > (u64)cap",
           cap=20)
    reject("sequences_need_more_literals", _more_literals(), "zs_lit_take(L, huf, out + op, (int)ll)")
    reject("literals_over_cap", zw.frame([cblk(L("raw", lits))], fcs=None), "op + rest > cap", cap=10)
    # skippable frames and trailing bytes
    reject("skippable_short", zw.skippable(b"")[:7] + b"", "csize - ip < 8")
    reject("skippable_past_end", zw.skippable(b"abc")[:-1], "fsz > (u32)(csize - ip - 8)")
    reject("trailing_4_bytes", (good + b"\x28\xb5\x2f\xfd", content), "csize - ip < 5")


def _weights_norm(data):
    """the (norm, log) zstd_write picks for the FSE-coded weights of `data`'s Huffman code"""
    w = zw.weights_for(data)
    explicit = w[:max(s for s in range(256) if w[s])]
    return zw.normalize([explicit.count(v) for v in range(13)], 6), 6


def _bad_offset():
    """a sequence whose offset reaches before the frame; the writer's own range check is bypassed"""
    lit = L("raw", b"ab")
    st = {"rep": [1, 4, 8]}
    body = zw.literals_section(lit, st) + zw.sequences_section([(2, 4, 3 + 9)], {}, st)
    return zw.MAGIC.to_bytes(4, "little") + b"\x00\x00" + (1 | 4 | (len(body) << 3)).to_bytes(3, "little") + body


def _rep1m1_zero():
    """rep1 = 1, then offset value 3 with LL = 0: rep1 - 1 = 0"""
    st = {"rep": [1, 4, 8]}
    body = zw.literals_section(L("raw", b"abcd"), st) + zw.sequences_section([(4, 4, 3 + 1), (0, 4, 3)], {}, st)
    return zw.MAGIC.to_bytes(4, "little") + b"\x00\x00" + (1 | 4 | (len(body) << 3)).to_bytes(3, "little") + body


def _more_literals():
    st = {"rep": [1, 4, 8]}
    body = zw.literals_section(L("raw", b"abcd"), st) + zw.sequences_section([(9, 4, 3 + 1)], {}, st)
    return zw.MAGIC.to_bytes(4, "little") + b"\x00\x00" + (1 | 4 | (len(body) << 3)).to_bytes(3, "little") + body


_build_reject()


@pytest.mark.parametrize("name", sorted(REJECT))
def test_reject_corpus_emu(zemu, zref, name):
    frame, cap, fragment = REJECT[name]
    r, _, canary, line = emu_decode(zemu, frame, cap)
    assert r == -1 and canary
    assert line == line_of(fragment), (line, fail_lines().get(line))
    if zref is not None:
        assert ref_decode(zref, frame, cap) is None, "ZSTD_decompress accepts it"


# ------------------------------------------------------------------------------------------------
# STRICT: RFC-invalid frames that ZSTD_decompress accepts, refused here on purpose
# ------------------------------------------------------------------------------------------------
def _huf12():
    """Huffman weights with a 12-bit code: the weights of 13 symbols 1, 1, 2, 3, ..., 12 (a complete tree)"""
    w = [0] * 256
    for s, x in enumerate([1, 1] + list(range(2, 13))):
        w[s] = x
    data = bytes(s for s in range(13) for _ in range(1 << max(w[s] - 1, 0)))[:1000]
    st = {"rep": [1, 4, 8]}
    tree = zw.huffman_tree(w, "direct")
    codes = {}
    at = 0
    for wt in range(1, 13):
        for s, x in enumerate(w):
            if x == wt:
                codes[s] = (at >> (wt - 1), 13 - wt)
                at += 1 << (wt - 1)
    parts = [zw.huffman_stream(data[k * 250:(k + 1) * 250], codes) for k in range(4)]
    payload = tree + b"".join(len(p).to_bytes(2, "little") for p in parts[:3]) + b"".join(parts)
    hdr = (2 | (2 << 2) | (len(data) << 4) | (len(payload) << 18)).to_bytes(4, "little")
    body = hdr + payload + b"\x00"
    return (zw.MAGIC.to_bytes(4, "little") + b"\x00\x50" + (1 | 4 | (len(body) << 3)).to_bytes(3, "little") + body,
            data)


def strict_frames():
    big = bytes(random.Random(8).getrandbits(8) for _ in range(BLOCK + 1))
    return {
        "huf_12_bits": (_huf12(), "maxbits > ZS_HUFLOG"),
        "raw_block_over_128k": (zw.frame([raw(big)], fcs=None), "bsize > ZS_BLOCKMAX || ip + bsize > csize || op"),
        "rle_block_over_128k": (zw.frame([rle(3, BLOCK + 1)], fcs=None), "bsize > ZS_BLOCKMAX || ip + 1 > csize"),
        "compressed_output_over_128k": (zw.frame([cblk(L("raw", b"z" * 100), [(100, BLOCK - 50, 3 + 1)])], fcs=None),
                                        "op + (int)ll + (int)ml - block_start > ZS_BLOCKMAX"),
        "literal_stream_not_used_up": (_spare_bits(), "L.s[k].pos != 0 || L.quota[k] != 0"),
    }


def _spare_bits():
    """300 Huffman literals in four streams; the second stream has 3 bits to spare below its first code"""
    data = skewed(300, 60, 300)
    w = zw.weights_for(data)
    codes, tree = zw.huffman_codes(w), zw.huffman_tree(w)
    seg = (len(data) + 3) // 4
    parts = []
    for k in range(4):
        items = [codes[b] for b in (data[k * seg:(k + 1) * seg] if k < 3 else data[3 * seg:])]
        parts.append(zw.backward(items + ([(0, 3)] if k == 1 else [])))
    payload = tree + b"".join(len(p).to_bytes(2, "little") for p in parts[:3]) + b"".join(parts)
    body = (2 | (2 << 2) | (len(data) << 4) | (len(payload) << 18)).to_bytes(4, "little") + payload + b"\x00"
    return zw.MAGIC.to_bytes(4, "little") + b"\x00\x00" + (1 | 4 | (len(body) << 3)).to_bytes(3, "little") + body, data


@pytest.mark.parametrize("name", sorted(STRICT))
def test_strict_entries_emu(zemu, zref, name):
    (frame, content), fragment = strict_frames()[name]
    assert strict_decode(frame) is None, "zstd_frame accepts it: the frame is RFC-valid"
    r, _, canary, line = emu_decode(zemu, frame, len(content) + 16)
    assert r == -1 and canary and line == line_of(fragment), (r, fail_lines().get(line))
    if zref is not None:
        assert ref_decode(zref, frame, len(content) + 16) == content, "ZSTD_decompress no longer accepts it"


def test_reference_verdicts_pinned(zemu, zref):
    """The reference's verdict and bytes for the crafted corpus, recorded: accepted frames give their content,
    rejected frames -1 (STRICT frames, which the reference accepts, give the content the writer put in them)."""
    corpus = [(n, f, len(c)) for n, (f, c, _) in sorted(ACCEPT.items())]
    corpus += [(n, f, cap) for n, (f, cap, _) in sorted(REJECT.items())]
    strict = {n: fc for n, ((fc), _) in strict_frames().items()}
    corpus += [(n, fc[0], len(fc[1]) + 16) for n, fc in sorted(strict.items())]

    def rec(name, got):
        return (name, -1, np.zeros(0, np.uint8)) if got is None else (name, len(got), np.frombuffer(got, np.uint8))
    ours = []
    for name, frame, cap in corpus:
        if name in strict:
            ours.append(rec(name, strict[name][1]))
        else:
            r, out, _, _ = emu_decode(zemu, frame, cap)
            ours.append(rec(name, out if r >= 0 else None))
    reference = None if zref is None else [rec(n, ref_decode(zref, f, cap)) for n, f, cap in corpus]
    assert_pinned("zstd_decode_edges", ours, reference)


# ------------------------------------------------------------------------------------------------
# the ledger: every ZS_FAIL line is reached by the reject corpus or by single damage to a small frame
# ------------------------------------------------------------------------------------------------
UNREACHABLE = {
    "if (ip >= csize) return ZS_FAIL;": "a frame is at least 6 bytes (checked first), so its window byte, at 5, is "
                                        "always there",
    "if (h < 0) return ZS_FAIL;": "passes on the failure of zs_fse_header, whose own line is the one recorded",
    "if (used < 0) return ZS_FAIL;": "passes on the failure of zs_huf_table, whose own line is the one recorded",
    "if (bend < 2) return ZS_FAIL": "a compressed block has at least 2 bytes (checked with its size)",
    "regen < 3 * seg": "from 6 literals on (checked before), 3 * ceil(regen / 4) never exceeds regen",
    "oc > 31 || mc > 52 || lc > 35": "no table holds a symbol above its maximum: RLE symbols and FSE descriptions are "
                                     "checked against it when the table is built",
    "second state": "the second state's weight is written at odd n <= 253 (the first state's check has already "
                    "stopped the loop at n = 254), so n >= 254 never holds there",
}


def _damage_corpus():
    """small valid frames, each truncated at every length and with each byte xored with 0x01, 0x40 and 0xff"""
    d = skewed(60, 9, 3)
    lits = skewed(64, 20, 2)
    seqs = [(10, 8, 3 + 5), (6, 20, 3 + 9), (3, 5, 1), (0, 4, 2), (12, 33, 3 + 40)]
    fse = {"ll": ("fse", None, 5), "of": ("fse", None, 5), "ml": ("fse", None, 5)}
    bases = [
        zw.frame([cblk(L("huf", d, streams=4), seqs[:2] and [(10, 8, 3 + 5), (6, 20, 3 + 9)], fse)], checksum=True),
        zw.frame([cblk(L("huf", skewed(40, 30, 1), wmode="fse")), cblk(L("treeless", d[:20]), [(20, 5, 3 + 3)],
                                                                        {"ll": ("rle", 18), "of": ("rle", 2),
                                                                         "ml": ("rle", 2)})], wd=3),
        zw.frame([cblk(L("huf", skewed(30, 8, 5), wmode="direct")), rle(4, 3), raw(b"rawraw")], fcs=None),
        zw.frame([cblk(L("raw", lits), seqs, {"ml": ("fse", None, 6)})], single=True, fcs_bytes=1),
    ]
    for fr, c in bases:
        for n in range(len(fr)):
            yield fr[:n], len(c)
        for pos in range(len(fr)):
            for x in (0x01, 0x40, 0xFF):
                yield patch(fr, pos, fr[pos] ^ x), len(c)


def test_damage_follows_the_rule_and_ledger_emu(zemu, zref):
    reached = {line_of(frag) for _, _, frag in REJECT.values()}
    reached |= {line_of(frag) for _, frag in strict_frames().values()}
    nbad = 0
    for frame, cap in _damage_corpus():
        r, out, canary, line = emu_decode(zemu, frame, cap)
        assert canary
        mine = strict_decode(frame)
        if r < 0:
            reached.add(line)
            nbad += 1
            if mine is not None and len(mine[0]) <= cap:
                pytest.fail(f"an RFC-valid frame is refused at line {line}: {frame.hex()}")
        elif mine is not None:
            assert out == mine[0]
        if zref is not None:
            want = ref_decode(zref, frame, cap)
            if want is None:
                assert r < 0, frame.hex()
            elif r >= 0:
                assert out == want, frame.hex()
            else:
                assert mine is None, frame.hex()          # refused where the reference accepts: RFC-invalid only
    assert nbad > 500
    lines = fail_lines()
    skip = {line_of(f) for f in UNREACHABLE if len([k for k, t in lines.items() if f in t]) == 1}
    missing = {k: lines[k].strip() for k in lines if k not in reached and k not in skip}
    assert not missing, missing


# ------------------------------------------------------------------------------------------------
# random descriptions, written and decoded three ways, then damaged
# ------------------------------------------------------------------------------------------------
def random_description(rng):
    """random blocks: raw, RLE and compressed; literals raw, RLE, Huffman or treeless (over the symbols of the frame's
    last Huffman table); tables predefined, RLE (when the block's codes allow), FSE or repeat (a repeat whose table
    lacks a code is refused by the writer, and the caller draws again)"""
    blocks, out_len, huf_syms, have = [], 0, None, set()
    for _ in range(rng.randint(1, 4)):
        kind = rng.random()
        if kind < 0.15 or out_len == 0 and kind < 0.3:
            n = rng.randint(0, 40)
            blocks.append(raw(bytes(rng.getrandbits(8) for _ in range(n))))
            out_len += n
            continue
        if kind < 0.25:
            n = rng.randint(0, 50)
            blocks.append(rle(rng.getrandbits(8), n))
            out_len += n
            continue
        nlit = rng.randint(0, 120)
        lits = skewed(nlit, rng.randint(2, 40), rng.getrandbits(16))
        mode = rng.choice(["raw", "rle", "huf", "huf", "treeless"])
        if mode == "treeless" and (huf_syms is None or nlit < 6):
            mode = "huf"
        if mode == "treeless":
            lits = bytes(rng.choice(huf_syms) for _ in range(nlit))
        if mode == "rle":
            lits = bytes([lits[0] if lits else 0]) * nlit
        if mode == "huf" and nlit < 6:
            mode = "raw"
        lit = L(mode, lits, byte=lits[0] if lits else 0)
        if mode in ("huf", "treeless"):
            lit.update(streams=rng.choice([1, 4]))
        if mode == "huf":
            lit.update(wmode=rng.choice(["direct", "fse"]))
            if len(set(lits)) < 3 and lit["wmode"] == "fse":
                lit["wmode"] = "direct"
            w = zw.weights_for(lits)
            huf_syms = [b for b in range(256) if w[b]]
        seqs, pos, used = [], out_len, 0
        for _ in range(rng.randint(0, 12)):
            ll = rng.randint(0, nlit - used) if nlit > used else 0
            if pos + ll == 0:
                continue
            ml = rng.choice([3, 4, 5, 17, 40, 300])
            ov = 3 + rng.randint(1, pos + ll) if rng.random() < 0.7 else rng.choice([1, 2, 3])
            seqs.append((ll, ml, ov))
            used += ll
            pos += ll + ml
        codes = {"ll": {zw.ll_code(q[0]) for q in seqs}, "ml": {zw.ml_code(q[1]) for q in seqs},
                 "of": {q[2].bit_length() - 1 for q in seqs}}
        modes = {}
        for name in ("ll", "of", "ml"):
            choice = ["predefined", ("fse", None, rng.randint(5, 6))]
            if len(codes[name]) == 1:
                choice.append(("rle", min(codes[name])))
            if name in have:
                choice.append("repeat")
            modes[name] = rng.choice(choice)
        if seqs:
            have |= {"ll", "of", "ml"}
        blocks.append(cblk(lit, seqs, modes))
        out_len = pos + nlit - used
    return blocks, dict(checksum=rng.random() < 0.3, fcs=rng.choice(["auto", None]))


def _valid_random(rng):
    while True:
        blocks, kw = random_description(rng)
        try:
            return zw.frame(blocks, **kw)
        except AssertionError:
            continue                                   # a repeat offset that reaches before the frame: draw again


def test_random_corpus_emu(zemu, zref):
    rng = random.Random(77)
    forms = set()
    for t in range(300):
        frame, content = _valid_random(rng)
        got = strict_decode(frame)
        assert got is not None and got[0] == content, t
        for b in got[1][0].blocks:
            if b["type"] == "compressed":
                forms.add(b["lit"]["type"])
                forms |= set(b["seq"]["modes"].values())
        r, out, canary, _ = emu_decode(zemu, frame, len(content))
        assert r == len(content) and out == content and canary, t
        if zref is not None:
            assert ref_decode(zref, frame, len(content)) == content, t
        bad = bytearray(frame)
        pos = rng.randrange(len(bad))
        bad[pos] = rng.getrandbits(8) if rng.random() < 0.5 else bad[pos] ^ (1 << rng.randrange(8))
        bad = bytes(bad)
        r, out, canary, _ = emu_decode(zemu, bad, len(content) + 8)
        assert canary
        mine = strict_decode(bad)
        if mine is not None and len(mine[0]) <= len(content) + 8:
            assert r == len(mine[0]) and out == mine[0], (t, pos)
        if zref is not None:
            want = ref_decode(zref, bad, len(content) + 8)
            if want is None:
                assert r == -1, (t, pos)
            elif r >= 0:
                assert out == want, (t, pos)
            else:
                assert mine is None, (t, pos)
    assert forms >= {"raw", "rle", "compressed", "treeless", "predefined", "fse", "repeat"}, forms


# ------------------------------------------------------------------------------------------------
# Blosc chunks of crafted frames, one frame per block
# ------------------------------------------------------------------------------------------------
def zstd_chunk(frames, blocksize, nbytes):
    """an unsplit zstd chunk (flags: one stream per block, codec 4) of the given frames"""
    nblocks = len(frames)
    head = 16 + 4 * nblocks
    bstarts, body, at = [], b"", head
    for f in frames:
        bstarts.append(at)
        body += struct.pack("<i", len(f)) + f
        at += 4 + len(f)
    cb = head + len(body)
    return (bytes([2, 1, 0x10 | (4 << 5), 1]) + struct.pack("<iii", nbytes, blocksize, cb) +
            b"".join(struct.pack("<i", s) for s in bstarts) + body)


def chunk_corpus(damaged=False):
    """(name, chunk, nbytes, kind) with kind "accept", "reject" or "strict": the whole crafted corpus, one frame per
    chunk and the blocksize its content's size (rejected frames get the room they were written for, at least one
    byte), two-block chunks, chunks where only one block is bad and, with damaged=True, every fifth damaged frame.
    Frames as long as their content are left out: such a block reads as stored (copied raw) at the chunk level."""
    out = []
    for n, (f, c, _) in sorted(ACCEPT.items()):
        if c and len(f) != len(c):
            out.append((n, zstd_chunk([f], len(c), len(c)), len(c), "accept"))
    for n, (f, cap, _) in sorted(REJECT.items()):
        if cap and len(f) != cap:
            out.append(("reject_" + n, zstd_chunk([f], cap, cap), cap, "reject"))
    for n, ((f, c), _) in sorted(strict_frames().items()):
        out.append(("strict_" + n, zstd_chunk([f], len(c), len(c)), len(c), "strict"))
    f1, c1 = zw.frame([cblk(L("huf", skewed(300, 20, 1), streams=4), [(30, 200, 3 + 10)])])
    f2, c2 = zw.frame([cblk(L("raw", b"tail"), [(4, 96, 3 + 4)])], checksum=True)
    n2 = len(c1) + len(c2)
    out.append(("two_blocks", zstd_chunk([f1, f2], len(c1), n2), n2, "accept"))
    out.append(("second_block_bad", zstd_chunk([f1, f2[:-1] + bytes([f2[-1] ^ 1])], len(c1), n2), n2, "reject"))
    out.append(("first_block_bad", zstd_chunk([patch(f1, 12, f1[12] ^ 0x10), f2], len(c1), n2), n2, "reject"))
    if damaged:
        for k, (f, cap) in enumerate(_damage_corpus()):
            if k % 5 == 0 and cap and len(f) != cap:
                out.append((f"damaged_{k}", zstd_chunk([f], cap, cap), cap, "damaged"))
    return out


def test_chunks_emu_against_reference(zemu, ref_if_built):
    zemu.blosc_getitem.restype = C.c_int
    for name, ch, n, kind in chunk_corpus():
        c = np.frombuffer(ch, np.uint8).copy()
        out = np.full(n + 32, 0x77, np.uint8)
        r = zemu.blosc_decompress_ctx(ptr(c), ptr(out), sz(n), C.c_int(1))
        assert (r == n) == (kind == "accept"), (name, r)
        assert (out[n:] == 0x77).all()
        item = np.full(n + 8, 0x33, np.uint8)
        g = zemu.blosc_getitem(ptr(c), C.c_int(0), C.c_int(n), ptr(item))
        assert (g == n) == (kind == "accept"), (name, g)
        if ref_if_built is not None:
            o2 = np.zeros(n + 32, np.uint8)
            r2 = ref_if_built.blosc_decompress_ctx(ptr(c), ptr(o2), sz(n), C.c_int(1))
            i2 = np.zeros(n + 8, np.uint8)
            g2 = ref_if_built.blosc_getitem(ptr(c), C.c_int(0), C.c_int(n), ptr(i2))
            if kind == "strict":                      # the reference accepts these frames; they are refused here
                assert r2 == n and g2 == n, (name, r2, g2)
                continue
            assert r2 == r and g2 == g, (name, r, r2, g, g2)
            if r == n:
                assert (out[:n] == o2[:n]).all()


@pytest.mark.gpu
def test_crafted_chunks_gpu(pkg, cuda, zemu):
    """The crafted corpus through the CUDA decoder, from host and device buffers: the emulator's return code and
    bytes, nothing written past destsize."""
    for name, ch, n, _ in chunk_corpus(damaged=True):
        c = np.frombuffer(ch, np.uint8).copy()
        want = np.full(n + 32, 0x77, np.uint8)
        r0 = zemu.blosc_decompress_ctx(ptr(c), ptr(want), sz(n), C.c_int(1))
        out = np.full(n + 32, 0x77, np.uint8)
        r = pkg.decompress_ctx(c, out[:n], n)
        assert r == r0 and (r < 0 or (out[:n] == want[:n]).all()) and (out[n:] == 0x77).all(), (name, r, r0)
        d_c = cuda.from_numpy(c).cuda()
        d_o = cuda.full((n + 32,), 0x77, dtype=cuda.uint8, device="cuda")
        r = pkg.decompress_ctx(d_c, d_o[:n], n)
        o = d_o.cpu().numpy()
        assert r == r0 and (r < 0 or (o[:n] == want[:n]).all()) and (o[n:] == 0x77).all(), (name, r, r0)

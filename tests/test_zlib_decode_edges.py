"""The inflate decoder (csrc/dev_inflate.cuh) branch by branch, on zlib streams written to order.

tests/deflate_write.py writes stored, fixed and dynamic blocks from explicit code lengths and items, so the forms that
Python's zlib never writes are spelled out: 15-bit codes, a lone 1-bit distance code, a block without distance codes,
symbols 286/287 and distances 30/31 in fixed blocks, code 16 at index 0, runs past HLIT + HDIST, HLIT / HDIST above
their maxima, incomplete and over-subscribed codes, length 258 as code 285 and as 284 + 31, distances equal to the
output position and one beyond it, stored blocks with LEN / NLEN mismatch, LEN 0, unaligned starts, and zlib headers
with FDICT, CINFO 8 or a bad FCHECK.  The verdict and the bytes of every stream come from Python's zlib.

Each rejected stream names the INF_FAIL line that must refuse it, and the ledger test fails if any INF_FAIL line of
dev_inflate.cuh goes unreached.  The warp Adler-32 gets its own sizes (lane slices at the 3800-byte run bound, and
0xFF runs long enough that a and b would leave 32 bits inside a slice without the bound)."""
import ctypes as C
import os
import random
import struct
import zlib

import numpy as np
import pytest

import deflate_write as dw
from datagen import ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "c-blosc_b200", "csrc", "dev_inflate.cuh")


@pytest.fixture(scope="module")
def zemu(emu):
    emu.emu_zlib_decode.restype = C.c_int
    emu.emu_zlib_decode.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    emu.emu_zlib_fail_line.restype = C.c_int
    return emu


def zlib_verdict(stream, cap):
    """what uncompress() does with `cap` bytes of room: the bytes, or None"""
    try:
        do = zlib.decompressobj()
        got = do.decompress(stream, cap + 1)
        return got if do.eof and len(got) <= cap else None
    except zlib.error:
        return None


def emu_decode(emu, stream, cap):
    """(return code, bytes, canary after cap intact, fail line)"""
    src = np.frombuffer(bytes(stream) + b"\0", np.uint8).copy()
    out = np.full(cap + 64, 0x77, np.uint8)
    r = emu.emu_zlib_decode(ptr(src), len(stream), ptr(out), cap)
    return r, out[:max(r, 0)].tobytes(), bool((out[cap:] == 0x77).all()), emu.emu_zlib_fail_line()


def fail_lines():
    return {i: t for i, t in enumerate(open(SRC).read().split("\n"), 1) if "INF_FAIL" in t and "#define" not in t}


def line_of(fragment):
    hits = [k for k, t in fail_lines().items() if fragment in t]
    assert len(hits) == 1, (fragment, hits)
    return hits[0]


def flat(symbols, n):
    """code lengths (n entries) of a complete code over `symbols`"""
    symbols = sorted(symbols)
    nb = (len(symbols) - 1).bit_length()
    nshort = (1 << nb) - len(symbols)
    out = [0] * n
    for i, s in enumerate(symbols):
        out[s] = nb - 1 if i < nshort else nb
    return out


def stream(blocks, content=None, **kw):
    """zlib stream of the blocks written by `blocks(w)`; the Adler-32 is of `content`, by default of what the raw
    DEFLATE body decodes to (b"" when it does not decode)"""
    w = dw.Bits()
    blocks(w)
    body = w.bytes()
    if content is None:
        try:
            content = zlib.decompressobj(-15).decompress(body)
        except zlib.error:
            content = b""
    return dw.zlib_stream(body, content, **kw)


ACCEPT, REJECT = {}, {}          # name -> stream ; name -> (stream, cap, fragment)


def _corpus():
    A, R = ACCEPT, REJECT
    txt = b"the quick brown fox jumps over the lazy dog"
    A["fixed_literals"] = stream(lambda w: dw.fixed(w, list(txt), final=True))
    # 15-bit codes and a lone 1-bit distance code: 'a'..'n' take 1..14 bits, 259 and the end code 15 bits
    lit = dw.lit_lengths({**{97 + i: i + 1 for i in range(14)}, 259: 15, 256: 15}, 260)
    items = [97, 98, 110, 110, ("match", 5, 1), 97]
    A["codes_of_15_bits"] = stream(lambda w: dw.dynamic(w, lit, [1], items, final=True))
    # no distance codes at all: fine until a distance is used
    lit2 = flat([120, 121, 256, 257], 258)
    A["no_distance_codes"] = stream(lambda w: dw.dynamic(w, lit2, [0], [120, 121, 120], final=True))
    R["no_distance_codes_used"] = (stream(lambda w: dw.dynamic(w, lit2, [0], [120, ("len", 257, 0), ("bits", 0, 8)],
                                                              final=True)), 100, "ds < 0 || ds >= 30")
    # HLIT and HDIST at their maxima, runs of 16 / 17 / 18 spelling the lengths
    lit3 = flat([65, 66, 256, 285], 286)
    dist3 = flat([0, 29], 30)
    lens = lit3 + dist3
    cl = []
    i = 0
    while i < len(lens):
        j = i
        while j < len(lens) and lens[j] == lens[i]:
            j += 1
        run = j - i
        if lens[i] == 0 and run >= 11:
            k = min(run, 138)
            cl.append((18, k - 11))
        elif lens[i] == 0 and run >= 3:
            k = min(run, 10)
            cl.append((17, k - 3))
        elif lens[i] and run >= 4:
            k = min(run - 1, 6) + 1
            cl += [(lens[i], 0), (16, k - 1 - 3)]
        else:
            k = 1
            cl.append((lens[i], 0))
        i += k
    A["hlit_286_hdist_30_runs"] = stream(lambda w: dw.dynamic(w, lit3, dist3, [65, 66, ("match", 258, 1), 65], final=True,
                                                             cl_items=cl))
    R["hlit_287"] = (stream(lambda w: dw.dynamic(w, lit3 + [0], dist3, [65], final=True)), 100, "nlen > INF_MAXLCODES")
    R["hlit_288"] = (stream(lambda w: dw.dynamic(w, lit3 + [0, 0], dist3, [65], final=True)), 100, "nlen > INF_MAXLCODES")
    R["hdist_31"] = (stream(lambda w: dw.dynamic(w, lit3, dist3 + [0], [65], final=True)), 100, "nlen > INF_MAXLCODES")
    R["hdist_32"] = (stream(lambda w: dw.dynamic(w, lit3, dist3 + [0, 0], [65], final=True)), 100,
                     "nlen > INF_MAXLCODES")
    # code-length code and code-length items
    lit4 = flat([65, 66, 256], 257)
    R["code16_at_index_0"] = (stream(lambda w: dw.dynamic(w, lit4, [1], [65], final=True,
                                                          cl_items=[(16, 0)] + [(x, 0) for x in lit4[3:] + [1]])), 100,
                              "nothing to repeat")
    R["run17_past_end"] = (stream(lambda w: dw.dynamic(w, lit4, [1], [65], final=True,
                                                       cl_items=[(x, 0) for x in lit4] + [(17, 7)])), 100,
                           "idx + rep > nlen + ndist")
    R["run18_past_end"] = (stream(lambda w: dw.dynamic(w, lit4, [1], [65], final=True,
                                                       cl_items=[(x, 0) for x in lit4[:200]] + [(18, 127)])), 100,
                           "idx + rep > nlen + ndist")
    cl_inc = [0] * 19
    cl_inc[0], cl_inc[1], cl_inc[2] = 2, 2, 2                         # three 2-bit codes: incomplete
    R["code_length_code_incomplete"] = (stream(lambda w: dw.dynamic(w, lit4, [1], [65], final=True, cl_lengths=cl_inc,
                                                                    cl_items=[(0, 0)])), 100,
                                        "the code-length code must be complete")
    cl_over = [0] * 19
    cl_over[0], cl_over[1], cl_over[2] = 1, 1, 1
    R["code_length_code_oversubscribed"] = (stream(lambda w: dw.dynamic(w, lit4, [1], [65], final=True,
                                                                        cl_lengths=cl_over, cl_items=[(0, 0)])), 100,
                                            "the code-length code must be complete")
    R["code_length_code_all_zero"] = (stream(lambda w: dw.dynamic(w, lit4, [1], [65], final=True, cl_lengths=[0] * 19,
                                                                  hclen=19, cl_items=[])), 100,
                                      "not a code-length code")
    R["no_end_of_block_code"] = (stream(lambda w: dw.dynamic(w, flat([65, 66, 257], 258), [1], [65], final=True,
                                                             end=False)), 100, "no end-of-block code")
    R["distance_code_incomplete"] = (stream(lambda w: dw.dynamic(w, lit2, [2, 2], [120], final=True)), 100,
                                     "ndist != dcount[0] + dcount[1]")
    R["distance_code_oversubscribed"] = (stream(lambda w: dw.dynamic(w, lit2, [1, 1, 1], [120], final=True)), 100,
                                         "ndist != dcount[0] + dcount[1]")
    R["literal_code_incomplete"] = (stream(lambda w: dw.dynamic(w, dw.lit_lengths({65: 2, 66: 2, 256: 2}), [1], [65],
                                                                final=True)), 100, "nlen != lcount[0] + lcount[1]")
    R["literal_code_oversubscribed"] = (stream(lambda w: dw.dynamic(w, dw.lit_lengths({65: 1, 66: 1, 256: 1}), [1],
                                                                    [65], final=True)), 100,
                                        "nlen != lcount[0] + lcount[1]")
    A["literal_code_single_end"] = stream(lambda w: dw.dynamic(w, dw.lit_lengths({256: 1}), [1], [], final=True))
    # fixed blocks: symbols 286 / 287, distances 30 / 31, length 258 spelled twice, distances at the output position
    for s in (286, 287):
        R[f"fixed_symbol_{s}"] = (stream(lambda w, s=s: dw.fixed(w, [65, ("len", s, 0)], final=True)), 100, "sym >= 29")
    for d in (30, 31):
        R[f"fixed_distance_{d}"] = (stream(lambda w, d=d: dw.fixed(w, [65, ("len", 257, 0), ("dist", d, 0)],
                                                                   final=True)), 100, "ds < 0 || ds >= 30")
    A["length_258_as_285_and_284_31"] = stream(lambda w: dw.fixed(w, [122, ("match", 258, 1), ("len", 284, 31),
                                                                      ("dist", 0, 0)], final=True))
    A["distance_equal_to_position"] = stream(lambda w: dw.fixed(w, [97, 98, 99, 100, ("match", 3, 4)], final=True))
    R["distance_beyond_position"] = (stream(lambda w: dw.fixed(w, [97, 98, 99, 100, ("match", 3, 5)], final=True),
                                            content=b"abcd"), 100, "dist > z.op")
    R["literal_over_cap"] = (A["fixed_literals"], len(txt) - 1, "z.op >= z.oend")
    R["stream_cut_in_a_symbol"] = (A["fixed_literals"][:12], 100, "not a literal/length code")
    R["reserved_block_type"] = (stream(lambda w: w.put(7, 3)) + b"\0", 100, "type == 3")
    # stored blocks
    A["stored_len_0_then_final"] = stream(lambda w: (dw.stored(w, b""), dw.stored(w, b"tail", final=True)))
    A["stored_unaligned_after_fixed"] = stream(lambda w: (dw.fixed(w, [65, 66, 67]),
                                                         dw.stored(w, b"stored bytes", final=True)))
    A["stored_then_fixed_then_dynamic"] = stream(lambda w: (dw.stored(w, b"xyz"), dw.fixed(w, [97, ("match", 4, 1)]),
                                                           dw.dynamic(w, lit2, [1], [120, 121], final=True)))
    R["stored_len_nlen_mismatch"] = (stream(lambda w: dw.stored(w, b"abc", final=True, nlength=0x1234)), 100,
                                     "len != (~nlen & 0xffffu)")
    R["stored_past_end"] = (stream(lambda w: dw.stored(w, b"abc", final=True, length=200)), 300,
                            "z.ip + (int)len > z.iend")
    R["stored_header_cut"] = (bytes([0x78, 0x01, 0x01, 0x05, 0x00]) + b"\0", 100, "z.ip + 4 > z.iend")
    R["no_block_header"] = (bytes([0x78, 0x01, 0x00, 0x00, 0x00, 0xff, 0xff]), 100, "no block header")
    w = dw.Bits()
    dw.stored(w, b"")
    dw.dynamic(w, lit4, [1], [65], final=True)
    R["code_length_code_cut"] = (bytes([0x78, 0x01]) + w.bytes()[:8], 100, "code-length code cut")
    # zlib header and trailer
    R["cinfo_8"] = (stream(lambda w: dw.fixed(w, [65], final=True), cmf=0x88), 100, "(cmf >> 4) > 7u")
    R["method_not_deflate"] = (stream(lambda w: dw.fixed(w, [65], final=True), cmf=0x79), 100, "(cmf >> 4) > 7u")
    R["bad_fcheck"] = (stream(lambda w: dw.fixed(w, [65], final=True), flg=0x02), 100, "FCHECK")
    R["fdict"] = (stream(lambda w: dw.fixed(w, [65], final=True), fdict=True), 100, "FDICT")
    R["too_short"] = (bytes([0x78, 0x01, 0x03, 0x00, 0x00]), 100, "csize < 2 + 4")
    R["adler_cut"] = (A["fixed_literals"][:-2], 100, "endpos + 4 > csize")
    R["adler_wrong"] = (stream(lambda w: dw.fixed(w, list(txt), final=True), content=txt + b"!"), 100,
                        "((tb << 16) | ta) != want")


_corpus()


def adler_streams():
    """(name, stream, content): stored blocks of the sizes where the warp Adler-32 changes path"""
    rng = random.Random(3)
    out = []
    for n, fill in ((0, None), (1, None), (31, None), (32, None), (33, None), (32 * 3799, None), (32 * 3800, 0xFF),
                    (32 * 3801, 0xFF), (32 * 3800 + 1, None), (32 * 6001, 0xFF), (32 * 7000 + 5, 0xFF)):
        data = bytes([fill]) * n if fill is not None else bytes(rng.getrandbits(8) for _ in range(n))

        def blocks(w, data=data):
            parts = [data[i:i + 65535] for i in range(0, len(data), 65535)] or [b""]
            for k, p in enumerate(parts):
                dw.stored(w, p, final=k == len(parts) - 1)
        out.append((f"adler_{n}_{'ff' if fill else 'rand'}", stream(blocks, content=data), data))
    return out


@pytest.mark.parametrize("name", sorted(ACCEPT))
def test_accept_corpus_emu(zemu, name):
    st = ACCEPT[name]
    want = zlib_verdict(st, 1 << 20)
    assert want is not None, "zlib refuses it"
    n = len(want)
    for cap in (n, n + 7):
        r, out, canary, _ = emu_decode(zemu, st, cap)
        assert r == n and out == want and canary, (cap, r)
    if n:
        r, _, canary, _ = emu_decode(zemu, st, n - 1)
        assert r == -1 and canary and zlib_verdict(st, n - 1) is None


@pytest.mark.parametrize("name", sorted(REJECT))
def test_reject_corpus_emu(zemu, name):
    st, cap, fragment = REJECT[name]
    assert zlib_verdict(st, cap) is None, "zlib accepts it"
    r, _, canary, line = emu_decode(zemu, st, cap)
    assert r == -1 and canary and line == line_of(fragment), (line, fail_lines().get(line))


def test_warp_adler32_sizes_emu(zemu):
    for name, st, data in adler_streams():
        assert zlib_verdict(st, len(data)) == data, name
        r, out, canary, _ = emu_decode(zemu, st, len(data))
        assert r == len(data) and out == data and canary, name
        bad = st[:-4] + ((zlib.adler32(data) ^ 0x10000) & 0xFFFFFFFF).to_bytes(4, "big")
        r, _, _, line = emu_decode(zemu, bad, len(data))
        assert r == -1 and line == line_of("((tb << 16) | ta) != want"), name


UNREACHABLE = {
    "the input ended inside the last symbol": "every read that can run out of input is checked where it happens "
                                              "(block header, stored header, code lengths, extra bits, symbols)",
}


def _damage_corpus():
    """small valid streams, each truncated at every length and with each byte xored with 0x01, 0x20 and 0xff"""
    for name in ("fixed_literals", "codes_of_15_bits", "hlit_286_hdist_30_runs", "stored_then_fixed_then_dynamic",
                 "no_distance_codes"):
        st = ACCEPT[name]
        n = len(zlib_verdict(st, 1 << 20))
        for k in range(len(st)):
            yield st[:k], n
        for pos in range(len(st)):
            for x in (0x01, 0x20, 0xFF):
                b = bytearray(st)
                b[pos] ^= x
                yield bytes(b), n


def test_damage_follows_zlib_and_ledger_emu(zemu):
    reached = {line_of(f) for _, _, f in REJECT.values()}
    nbad = 0
    for st, cap in _damage_corpus():
        r, out, canary, line = emu_decode(zemu, st, cap)
        want = zlib_verdict(st, cap)
        assert canary
        if want is None:
            assert r == -1, st.hex()
            reached.add(line)
            nbad += 1
        else:
            assert r == len(want) and out == want, st.hex()
    assert nbad > 300
    lines = fail_lines()
    skip = {line_of(f) for f in UNREACHABLE}
    missing = {k: lines[k].strip() for k in lines if k not in reached and k not in skip}
    assert not missing, missing


# ------------------------------------------------------------------------------------------------
# Blosc chunks of the crafted streams, one stream per block
# ------------------------------------------------------------------------------------------------
def zlib_chunk(st, n):
    """an unsplit one-block zlib chunk (codec 3) holding `st` for n bytes"""
    return (bytes([2, 1, 0x10 | (3 << 5), 1]) + struct.pack("<iii", n, n, 16 + 4 + 4 + len(st)) +
            struct.pack("<ii", 20, len(st)) + st)


def chunk_corpus():
    """(name, chunk, nbytes) for every crafted stream whose size differs from its block's (an equal size would read
    as a stored block); rejected streams get the room zlib was given, at least one byte"""
    out = []
    for name, st in sorted(ACCEPT.items()):
        n = len(zlib_verdict(st, 1 << 20))
        if n and n != len(st):
            out.append((name, zlib_chunk(st, n), n))
    for name, (st, cap, _) in sorted(REJECT.items()):
        if cap and cap != len(st):
            out.append(("reject_" + name, zlib_chunk(st, cap), cap))
    for name, st, data in adler_streams():
        if data:
            out.append((name, zlib_chunk(st, len(data)), len(data)))
            bad = st[:-1] + bytes([st[-1] ^ 1])
            out.append((name + "_bad", zlib_chunk(bad, len(data)), len(data)))
    return out


def test_chunks_emu(zemu):
    zemu.blosc_getitem.restype = C.c_int
    for name, ch, n in chunk_corpus():
        c = np.frombuffer(ch, np.uint8).copy()
        out = np.full(n + 32, 0x77, np.uint8)
        r = zemu.blosc_decompress_ctx(ptr(c), ptr(out), sz(n), C.c_int(1))
        st = ch[24:]
        want = zlib_verdict(st, n)
        if want is not None and len(want) == n:
            assert r == n and out[:n].tobytes() == want, name
        else:
            assert r < 0, (name, r)
        assert (out[n:] == 0x77).all(), name


@pytest.mark.gpu
def test_crafted_chunks_gpu(pkg, cuda, zemu):
    """The crafted streams through the CUDA decoder, from host and device buffers: the emulator's return code and
    bytes, nothing written past destsize."""
    for name, ch, n in chunk_corpus():
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

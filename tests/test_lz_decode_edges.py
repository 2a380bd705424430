"""The LZ4 and BloscLZ decoders (csrc/dev_lz4.cuh, dev_lz4dpair.cuh, dev_blosclz.cuh) tier by tier, on streams
written to order.

lz4_decode_warp has five tiers -- dense, lone long match, batch, single sequence, general -- each with its own entry
condition and its own rule for reading a match from the 16 KiB shared-memory ring that mirrors recent output or from
global memory (offset thresholds 13696 / 15872 / 16000 / 16320 / 14272, and `ring_lo`, which moves after a literal run
longer than 16320 bytes, after a match longer than 2048 bytes and after an offset-0 fill).  lz4_pair_parse /
lz4_pair_copier restate all of it across two warps.  Real encoder output almost never reaches these boundaries, and a
wrong threshold or a missing `ring_lo` update gives plausible wrong bytes rather than a crash.

tests/lz_write.py writes blocks from explicit sequences.  Accept corpus: one scenario per tier x source x boundary,
each decoded by emu_lz4_decode, emu_lz4_decode_pair, the oracle and (when oracle/_ref is built) LZ4_decompress_safe,
at cap = n and n + 9 with a canary after cap; each asserts the branch ids (LZ4D_H_*) it was written to reach, in both
decoders.  Reject corpus: one defect each, naming the LZ4D_FAIL / BLZ_FAIL line that must refuse it.  Ledgers fail if a
fail line or a branch id goes unreached.  The reference's verdicts for the crafted corpus are pinned in
tests/golden/reference_results.json."""
import ctypes as C
import os
import random
import struct

import numpy as np
import pytest

import lz_write as lw
from lz_write import seq
from datagen import assert_pinned, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "c-blosc_b200", "csrc")
SRC_WARP = os.path.join(CSRC, "dev_lz4.cuh")
SRC_PAIR = os.path.join(CSRC, "dev_lz4dpair.cuh")
SRC_BLZ = os.path.join(CSRC, "dev_blosclz.cuh")
CANARY = 0x77

# branch ids: the order of the enums in dev_lz4.cuh and dev_blosclz.cuh
H = ["DENSE_SHIFT%d" % s for s in range(9)] + [
    "DENSE_LONGCAP", "DENSE_BAD", "DENSE_BAD0", "DENSE_FEW", "DENSE_RING", "DENSE_GLOBAL",
    "LONE_RING", "LONE_GLOBAL", "LONE_PERIOD", "BATCH_FAST", "BATCH_WALK", "BATCH_RING", "BATCH_GLOBAL",
    "SINGLE_RING", "SINGLE_GLOBAL", "GEN_LITBUMP", "GEN_OFF0", "GEN_RING", "GEN_GLOBAL", "GEN_LONG", "GEN_LAST"]
BH = ["DENSE", "DENSE_FEW", "DENSE_BAD", "FAR", "LENEXT", "LITERAL", "DROPPED"]


def _enum_names(path, first, last):
    """the enum's names, in order, as the source declares them (checks H / BH against the code)"""
    text = open(path).read()
    body = text[text.index(first):text.index(last)]
    return [w.strip() for w in body.replace("\n", " ").split(",") if w.strip()]


def test_branch_id_tables_match_source():
    names = []
    text = open(SRC_WARP).read()
    body = text[text.index("LZ4D_H_DENSE_SHIFT = 0"):text.index("LZ4D_NHIT")]
    for line in body.split("\n"):
        line = line.split("/*")[0]
        names += [w.split("=")[0].strip() for w in line.split(",") if w.strip()]
    assert names[0] == "LZ4D_H_DENSE_SHIFT" and names[1] == "LZ4D_H_DENSE_LONGCAP"
    assert ["LZ4D_H_" + h for h in H[9:]] == names[1:]
    assert ["BLZ_H_" + h for h in BH] == _enum_names(SRC_BLZ, "BLZ_H_DENSE,", "BLZ_NHIT")


# ------------------------------------------------------------------------------------------------
# the decoders
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lemu(emu):
    for f in ("emu_lz4_decode", "emu_lz4_decode_pair", "emu_blz_decode"):
        getattr(emu, f).restype = C.c_int
        getattr(emu, f).argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    for f in ("emu_lz4d_fail_line", "emu_blz_fail_line"):
        getattr(emu, f).restype = C.c_int
    emu.emu_lz4d_hits.restype = C.c_int
    emu.emu_lz4d_hits.argtypes = [C.c_void_p]
    emu.emu_blz_hits.restype = C.c_int
    emu.emu_blz_hits.argtypes = [C.c_void_p]
    emu.emu_lz4_decode_list.restype = None
    hits(emu)
    bhits(emu)
    return emu


@pytest.fixture(scope="module")
def lref(ref_if_built):
    r = ref_if_built
    if r is None:
        return None
    r.LZ4_decompress_safe.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    r.blosclz_decompress.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    return r


@pytest.fixture(scope="module")
def lorc(orc):
    orc.orc_lz4_decompress_safe.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    orc.orc_blosclz_decompress.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    return orc


def hits(emu):
    h = (C.c_longlong * 64)()
    n = emu.emu_lz4d_hits(h)
    assert n == len(H)
    return {H[i] for i in range(n) if h[i]}


def bhits(emu):
    h = (C.c_longlong * 16)()
    n = emu.emu_blz_hits(h)
    assert n == len(BH)
    return {BH[i] for i in range(n) if h[i]}


def _src(stream):
    return np.frombuffer(bytes(stream) + b"\0", np.uint8).copy()


def emu_lz4(emu, stream, cap, pair=False):
    """(return code, bytes written, canary after cap intact, fail line, branch ids reached)"""
    src = _src(stream)
    out = np.full(cap + 64, CANARY, np.uint8)
    f = emu.emu_lz4_decode_pair if pair else emu.emu_lz4_decode
    r = f(ptr(src), len(stream), ptr(out), cap)
    return r, out[:max(r, 0)].tobytes(), bool((out[cap:] == CANARY).all()), emu.emu_lz4d_fail_line(), hits(emu)


def emu_blz(emu, stream, cap):
    src = _src(stream)
    out = np.full(cap + 64, CANARY, np.uint8)
    r = emu.emu_blz_decode(ptr(src), len(stream), ptr(out), cap)
    return r, out[:max(r, 0)].tobytes(), bool((out[cap:] == CANARY).all()), emu.emu_blz_fail_line(), bhits(emu)


def c_lz4(lib, fname, stream, cap):
    """LZ4_decompress_safe (or the oracle's): the bytes, or None for an error; and the canary"""
    src = _src(stream)
    out = np.full(cap + 64, CANARY, np.uint8)
    r = getattr(lib, fname)(ptr(src), ptr(out), len(stream), cap)
    return (None if r < 0 else out[:r].tobytes()), bool((out[cap:] == CANARY).all())


def c_blz(lib, fname, stream, cap):
    src = _src(stream)
    out = np.full(cap + 64, CANARY, np.uint8)
    r = getattr(lib, fname)(ptr(src), len(stream), ptr(out), cap)
    return (None if r <= 0 else out[:r].tobytes()), bool((out[cap:] == CANARY).all())


def lz4_all(lemu, lorc, lref, stream, cap):
    """every LZ4 decoder's verdict; asserts the canaries and that they all agree.  Returns (bytes or None, fail line
    of the warp decoder, fail line of the pair, hits of the warp decoder, hits of the pair)"""
    r1, o1, k1, l1, h1 = emu_lz4(lemu, stream, cap)
    r2, o2, k2, l2, h2 = emu_lz4(lemu, stream, cap, pair=True)
    assert k1 and k2, "written past cap"
    v1, v2 = (o1 if r1 >= 0 else None), (o2 if r2 >= 0 else None)
    assert v1 == v2, ("warp and pair differ", r1, r2)
    vo, ko = c_lz4(lorc, "orc_lz4_decompress_safe", stream, cap)
    assert ko and vo == v1, ("oracle differs", r1, None if vo is None else len(vo))
    if lref is not None:
        vr, kr = c_lz4(lref, "LZ4_decompress_safe", stream, cap)
        assert kr and vr == v1, ("LZ4_decompress_safe differs", r1, None if vr is None else len(vr))
    return v1, l1, l2, h1, h2


def blz_all(lemu, lorc, lref, stream, cap):
    r, o, k, line, h = emu_blz(lemu, stream, cap)
    assert k, "written past cap"
    v = o if r > 0 else None
    vo, ko = c_blz(lorc, "orc_blosclz_decompress", stream, cap)
    assert ko and vo == v, ("oracle differs", r)
    if lref is not None:
        vr, kr = c_blz(lref, "blosclz_decompress", stream, cap)
        assert kr and vr == v, ("blosclz_decompress differs", r)
    return v, line, h


# ------------------------------------------------------------------------------------------------
# building blocks of the LZ4 scenarios
# ------------------------------------------------------------------------------------------------
def rnd(n, seed=0):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def lead(L, fill=True, seed=1):
    """L random literals (+ a 4-byte match), then, with fill, one 10-literal sequence.  Both go down the general path,
    and the dense tier's back-off (one skipped round after the literal run) is used up by the filler, so that the
    sequence after it is offered to every tier."""
    s = [seq(rnd(L, seed), 7, 4)]
    if fill:
        s.append(seq(rnd(10, seed + 1), 5, 4))
    return s


def dseq(off, ml=8):
    """a dense-form sequence: no literals, a 4..18-byte match"""
    assert 4 <= ml <= 18
    return seq(b"", off, ml)


def lseq(off, ml):
    """a dense-form long match: no literals, token 0x0F and one length byte (ml = 19 + byte)"""
    return seq(b"", off, ml)


def _tailbytes(m):
    return 3 + (len(lw.length_bytes(m - 4)) if m - 4 >= 15 else 0)


def _lastbytes(k):
    return 1 + k + (len(lw.length_bytes(k)) if k >= 15 else 0)


def tuned(before, tier, need_in=None, need_out=None, seed=9):
    """block = before + tier + a literal-free match at offset 1 + final literals, with the tail chosen so that at
    the first sequence of `tier` exactly need_in input bytes are left (iend - ip) and need_out output bytes
    (oend - op, cap = the block's output).  Without room for that match, the final literals alone make the tail."""
    t_in = len(lw.lz4_block(tier, end=False)[0])
    t_out = sum(len(s["lits"]) + s["ml"] for s in tier)
    ip = len(lw.lz4_block(before, end=False)[0])
    for k in range(5, 4000):
        for m in (3000 if need_out is None else need_out - t_out - k, 0):
            if m < 0 or 0 < m < 19 or m == 0 and need_out is not None and t_out + k != need_out:
                continue
            tb = _tailbytes(m) if m else 0
            if need_in is None and k == (200 if need_out is None else 60 if t_out + 60 < need_out else k) or \
                    need_in is not None and t_in + tb + _lastbytes(k) == need_in:
                blk, out = lw.lz4_block(before + tier + ([seq(b"", 1, m)] if m else []), rnd(k, seed))
                assert need_in is None or len(blk) - ip == need_in
                return blk, out
    raise AssertionError("no tail fits")


ACCEPT = {}           # name -> (block, content, cap list, hits required, hits forbidden)


def accept(name, block_content, need=(), forbid=(), caps=None, exact=False):
    """exact: an entry condition at equality -- decoded at cap = n only (more room changes the tier)"""
    assert name not in ACCEPT
    blk, out = block_content
    assert out is not None
    if exact:
        caps = [len(out)]
    ACCEPT[name] = (blk, out, caps, set(need), set(forbid))


def _build_accept():
    # ---- dense tier: ring threshold 13696, every segment shift, the long-match cap, runs of 3 and 4 ----
    for off, src in ((13696, "RING"), (13697, "GLOBAL")):
        accept(f"dense_off_{off}", tuned(lead(14000), [dseq(off)] * 32), ["DENSE_SHIFT0", "DENSE_" + src],
               ["DENSE_" + ("GLOBAL" if src == "RING" else "RING")])
    accept("dense_match_0", tuned(lead(200), [dseq(218 + 8 * k, 8) for k in range(32)]),
           ["DENSE_SHIFT0", "DENSE_RING"])
    for s in range(9):                       # s long matches, each after three short ones
        tier = []
        for j in range(s):
            tier += [dseq(2900 + j), dseq(2800 + j, 12), dseq(2700, 18), lseq(2600 + j, 19 + 30 * j)]
        tier += [dseq(800, 6)] * (32 - len(tier))
        accept(f"dense_shift_{s}", tuned(lead(3000), tier), ["DENSE_SHIFT%d" % s])
    tier = []
    for j in range(9):                       # a ninth long match in one step: the step stops in front of it
        tier += [dseq(2000 + j), dseq(2100 + j), lseq(2200 + j, 200 + j)]
    tier += [dseq(2500)] * 5
    accept("dense_ninth_long", tuned(lead(4000), tier), ["DENSE_SHIFT8", "DENSE_LONGCAP"])
    accept("dense_long_at_lane_31", tuned(lead(3000), [dseq(1500, 9)] * 31 + [lseq(2900, 273)] + [dseq(600)] * 4),
           ["DENSE_SHIFT1"])
    # far offsets in full steps with long matches: the ring slots of sources > 13696 back are overwritten by the step
    for off in (14000, 16000, 16320, 16321, 40000):
        tier = []
        for j in range(8):
            tier += [dseq(off, 18), dseq(off - j, 17), dseq(off, 16), lseq(off - 3 * j, 273 - j)]
        accept(f"dense_far_{off}", tuned(lead(41000), tier), ["DENSE_SHIFT8", "DENSE_GLOBAL"], ["DENSE_RING"])
    accept("dense_ext_254", tuned(lead(3000), [dseq(1000)] * 6 + [lseq(2000, 19 + 254)] + [dseq(700)] * 25),
           ["DENSE_SHIFT1"])
    accept("dense_ext_255", tuned(lead(3000), [dseq(1000)] * 6 + [lseq(2000, 19 + 255 + 7)] + [dseq(700)] * 25),
           ["DENSE_SHIFT0"])
    accept("dense_run_3", tuned(lead(3000), [dseq(1000)] * 3 + [seq(b"abc", 900, 8)] + [seq(b"q" * 10, 5, 4)] * 3),
           ["DENSE_FEW"], ["DENSE_SHIFT0"])
    accept("dense_run_4", tuned(lead(3000), [dseq(1000)] * 4 + [seq(b"abc", 900, 8)] + [seq(b"q" * 10, 5, 4)] * 3),
           ["DENSE_SHIFT0"])
    # a sequence that reads the step's own output ends the run: exactly at the 8-byte slack, and one past it
    accept("dense_bad_slack", tuned(lead(3000), [dseq(1000)] * 5 + [dseq(5 * 8 + 8 + 7, 8)] + [dseq(1000)] * 26),
           ["DENSE_BAD", "DENSE_SHIFT0"])
    accept("dense_slack_ok", tuned(lead(3000), [dseq(1000)] * 5 + [dseq(5 * 8 + 8 + 8, 8)] + [dseq(1000)] * 26),
           ["DENSE_SHIFT0"], ["DENSE_BAD"])
    accept("dense_bad_lane0", tuned(lead(3000), [dseq(4, 8)] + [dseq(1000)] * 31), ["DENSE_BAD0"])
    # dense data resuming after a back-off
    accept("dense_after_backoff", tuned(lead(3000), [seq(b"x" * 10, 900, 4)] * 4 + [dseq(1000, 9)] * 40 +
                                        [seq(b"y" * 10, 800, 4)] * 9 + [dseq(1100, 10)] * 64),
           ["DENSE_SHIFT0"])
    # ---- lone long match: period copies; the ring unless ring_lo says the source is not mirrored ----
    for off in (1, 2, 3, 7, 18, 19, 31, 32, 33, 200, 280):
        accept(f"lone_off_{off}", tuned(lead(3000), [lseq(off, 19 + 254)]), ["LONE_RING"] +
               (["LONE_PERIOD"] if off < 273 else []))
    accept("lone_after_long_copy", tuned(lead(20000, fill=False), [seq(rnd(10, 3), 5, 3000), lseq(3, 119)]),
           ["GEN_LONG", "LONE_GLOBAL", "LONE_PERIOD"], ["LONE_RING"])
    accept("lone_after_off0", tuned(lead(20000, fill=False), [seq(rnd(10, 3), 0, 100), lseq(3, 119)]),
           ["GEN_OFF0", "LONE_GLOBAL"], ["LONE_RING"])
    # ---- batch: eligibility 319 / 320, ring threshold 16000, fast chain and walk, lit 9 / 10, mln 14 / 15 ----
    for off, src in ((16000, "RING"), (16001, "GLOBAL")):
        accept(f"batch_fast_off_{off}", tuned(lead(17000), [dseq(off)] * 11, need_in=80),
               ["BATCH_FAST", "BATCH_" + src], ["BATCH_" + ("GLOBAL" if src == "RING" else "RING")])
        accept(f"batch_walk_off_{off}", tuned(lead(17000), [seq(b"ab", off, 8), seq(b"c" * 9, off, 18)] * 3),
               ["BATCH_WALK", "BATCH_" + src], ["BATCH_" + ("GLOBAL" if src == "RING" else "RING")])
    accept("batch_off_319", tuned(lead(3000), [seq(b"ab", 319, 8)]), ["SINGLE_RING"], ["BATCH_WALK", "BATCH_FAST"])
    accept("batch_off_320", tuned(lead(3000), [seq(b"ab", 320, 8)]), ["BATCH_WALK"])
    accept("batch_match_0", tuned([seq(rnd(696, 5), 7, 4)], [dseq(700, 4)] + [dseq(600)] * 10, need_in=80),
           ["BATCH_FAST"])
    accept("batch_lit_9", tuned(lead(3000), [seq(b"L" * 9, 500, 8)]), ["BATCH_WALK"])
    accept("batch_lit_10", tuned(lead(3000), [seq(b"L" * 10, 500, 8)]), ["GEN_RING"], ["BATCH_WALK", "SINGLE_RING"])
    accept("batch_mln_14", tuned(lead(3000), [seq(b"L", 500, 18)]), ["BATCH_WALK"])
    accept("batch_mln_15", tuned(lead(3000), [seq(b"L", 500, 19)]), ["GEN_RING"], ["BATCH_WALK", "SINGLE_RING"])
    for need_in, taken in ((49, True), (48, False)):
        accept(f"batch_entry_in_{need_in}", tuned(lead(3000), [seq(b"ab", 400, 8)], need_in=need_in),
               ["BATCH_WALK" if taken else "SINGLE_RING"], [] if taken else ["BATCH_WALK"])
    for need_out, taken in ((332, True), (331, False)):
        accept(f"batch_entry_out_{need_out}", tuned(lead(3000), [seq(b"ab", 400, 8)], need_out=need_out),
               ["BATCH_WALK" if taken else "SINGLE_RING"], [] if taken else ["BATCH_WALK"], exact=True)
    # ---- single sequence: ring threshold 16320, entry ip + 20 and op + total <= oend - 12, self-overlap ----
    for off, src in ((16320, "RING"), (16321, "GLOBAL")):
        accept(f"single_off_{off}", tuned(lead(17000), [seq(b"ab", off, 8)], need_in=30),
               ["SINGLE_" + src], ["SINGLE_" + ("GLOBAL" if src == "RING" else "RING")])
    for need_in, taken in ((20, True), (19, False)):
        accept(f"single_entry_in_{need_in}", tuned(lead(3000), [seq(b"ab", 100, 8)], need_in=need_in),
               ["SINGLE_RING" if taken else "GEN_RING"], [] if taken else ["SINGLE_RING"])
    for need_out, taken in ((25, True), (24, False)):
        accept(f"single_entry_out_{need_out}", tuned(lead(3000), [seq(b"L" * 9, 100, 4)], need_out=need_out),
               ["SINGLE_RING" if taken else "GEN_RING"], [] if taken else ["SINGLE_RING"], exact=True)
    accept("single_match_0", tuned([seq(rnd(40, 5), 7, 4)], [seq(b"ab", 46, 8)], need_in=30), ["SINGLE_RING"])
    accept("single_self_overlap", tuned(lead(3000), [seq(b"ab", 9, 8)], need_in=30), ["GEN_RING"], ["SINGLE_RING"])
    # ---- general path: ring threshold 14272, 2048 / 2049-byte matches, long literal runs, offset 0 ----
    for off, src in ((14272, "RING"), (14273, "GLOBAL")):
        accept(f"general_off_{off}", tuned([], [seq(rnd(15000, 4), off, 100)]),
               ["GEN_" + src], ["GEN_" + ("GLOBAL" if src == "RING" else "RING")])
    accept("general_match_0", tuned([seq(rnd(200, 5), 7, 4)], [seq(b"L" * 10, 214, 100)]), ["GEN_RING"])
    for off in (1, 2, 3, 7, 31, 32, 33, 65535):
        for ml in (2048, 2049):
            accept(f"general_ml_{ml}_off_{off}", tuned(lead(66000 if off > 3000 else 3000), [seq(b"L" * 10, off, ml)]),
                   ["GEN_LONG"] if ml > 2048 else ["GEN_GLOBAL" if off > 14272 else "GEN_RING"])
    for n in (16320, 16321, 20000):
        bump = ["GEN_LITBUMP"] if n > 16320 else []
        accept(f"literal_run_{n}_single", tuned([seq(rnd(n, 6), 16300, 8)], [seq(b"ab", 16310, 8)], need_in=30),
               bump + ["SINGLE_RING"], [] if bump else ["GEN_LITBUMP"])
        accept(f"literal_run_{n}_dense", tuned([seq(rnd(n, 6), 13000, 8), seq(b"f" * 10, 9, 4)],
                                               [dseq(13600 - 40 * k, 18) for k in range(32)]),
               bump + ["DENSE_SHIFT0", "DENSE_RING"])
    accept("off0_then_single", tuned(lead(20000, fill=False), [seq(rnd(10, 3), 0, 100), seq(b"ab", 50, 8)],
                                     need_in=60), ["GEN_OFF0", "SINGLE_GLOBAL"], ["SINGLE_RING"])
    accept("off0_then_batch", tuned(lead(20000, fill=False), [seq(rnd(10, 3), 0, 1000)] + [dseq(900)] * 11,
                                    need_in=90), ["GEN_OFF0", "BATCH_GLOBAL"], ["BATCH_RING"])
    accept("off0_then_dense", tuned(lead(20000, fill=False), [seq(rnd(10, 3), 0, 2000), seq(b"f" * 10, 9, 4)] +
                                    [dseq(1900 - 40 * k, 18) for k in range(32)]),
           ["GEN_OFF0", "DENSE_GLOBAL"], ["DENSE_RING"])
    accept("off0_then_general", tuned([], [seq(rnd(20000, 3), 0, 500), seq(b"L" * 10, 300, 100)]),
           ["GEN_OFF0", "GEN_GLOBAL"], ["GEN_RING"])
    accept("long_copy_then_single", tuned(lead(20000, fill=False), [seq(rnd(10, 3), 7, 3000), seq(b"ab", 50, 8)],
                                          need_in=60), ["GEN_LONG", "SINGLE_GLOBAL"], ["SINGLE_RING"])
    accept("long_copy_then_batch", tuned(lead(20000, fill=False), [seq(rnd(10, 3), 7, 3000)] + [dseq(900)] * 11,
                                         need_in=90), ["GEN_LONG", "BATCH_GLOBAL"], ["BATCH_RING"])
    accept("long_copy_then_dense", tuned(lead(20000, fill=False), [seq(rnd(10, 3), 7, 3000), seq(b"f" * 10, 9, 4)] +
                                         [dseq(2900 - 40 * k, 18) for k in range(32)]),
           ["GEN_LONG", "DENSE_GLOBAL"], ["DENSE_RING"])
    # ---- the end of the block ----
    accept("last_literals_to_iend", lw.lz4_block([seq(rnd(20, 7), 10, 7)], rnd(5, 8)), ["GEN_LAST"])
    accept("match_ends_at_oend_5", lw.lz4_block([seq(rnd(20, 7), 10, 12)], rnd(5, 8)), ["GEN_LAST"])
    accept("literals_end_at_iend_8", lw.lz4_block([seq(rnd(20, 7), 10, 8)], rnd(5, 8)), ["GEN_LAST"])
    accept("only_literals", lw.lz4_block([], rnd(300, 9)), ["GEN_LAST"])
    accept("empty_output", (b"\x00", b""), caps=[0, 9])
    accept("lit_len_15", lw.lz4_block([seq(rnd(15, 7), 10, 19)], rnd(15, 8)), ["GEN_LAST"])
    accept("lit_len_270", lw.lz4_block([seq(rnd(270, 7), 10, 4 + 15 + 255)], rnd(270, 8)), ["GEN_LAST"])
    accept("chain_255_x40", lw.lz4_block([seq(rnd(15 + 255 * 40, 7), 3, 4 + 15 + 255 * 40)], rnd(20, 8)),
           ["GEN_LAST"])


_build_accept()


@pytest.mark.parametrize("name", sorted(ACCEPT))
def test_lz4_accept_corpus_emu(lemu, lorc, lref, name):
    blk, content, caps, need, forbid = ACCEPT[name]
    n = len(content)
    for cap in caps or (n, n + 9):
        got, _, _, h1, h2 = lz4_all(lemu, lorc, lref, blk, cap)
        assert got == content, (cap, None if got is None else len(got))
        for h in (h1, h2):
            assert need <= h, ("branch not reached", sorted(need - h))
            assert not (forbid & h), ("branch reached", sorted(forbid & h))
    if n > 0 and caps is None:
        got, _, _, _, _ = lz4_all(lemu, lorc, lref, blk, n - 1)
        assert got is None


# ------------------------------------------------------------------------------------------------
# reject corpus: one defect each, and the LZ4D_FAIL line that must catch it (in each decoder)
# ------------------------------------------------------------------------------------------------
def fail_lines(path, macro):
    """{line number: text} of every line of `path` that uses `macro` (not its definition)"""
    return {i: t for i, t in enumerate(open(path).read().split("\n"), 1) if macro in t and "#define" not in t}


def line_of(path, macro, fragment):
    hits_ = [k for k, t in fail_lines(path, macro).items() if fragment in t]
    assert len(hits_) == 1, (fragment, hits_)
    return hits_[0]


# site -> (fragment in dev_lz4.cuh, fragment in dev_lz4dpair.cuh)
SITES = {
    "cap0": ("(csize == 1 && in[0] == 0) ? 0 : LZ4D_FAIL", "(csize == 1 && in[0] == 0) ? 0 : LZ4D_FAIL"),
    "csize0": ("if (csize == 0) return LZ4D_FAIL", "if (csize == 0) return LZ4D_FAIL"),
    "batch_match": ("my_rank >= 0 && match < 0)) return LZ4D_FAIL", "my_rank >= 0 && match < 0)) { result = LZ4D_FAIL"),
    "single_match": ("if (match < 0) return LZ4D_FAIL;                     /* lz4.c:2356 (off",
                     "if (match < 0) { result = LZ4D_FAIL; break; }       /* lz4.c:2356 */"),
    "litlen_start": ("if (ip >= iend - 15) return LZ4D_FAIL", "if (ip >= iend - 15) { result = LZ4D_FAIL"),
    "litlen_bytes": ("if (ip > iend - 15) return LZ4D_FAIL", "if (ip > iend - 15) { result = LZ4D_FAIL"),
    "litlen_oend": ("if (len > oend) return LZ4D_FAIL;                     /* same", "if (len > oend) { result = LZ4D_FAIL"),
    "last": ("if (last && (ip + len != iend || cpy > oend)) return LZ4D_FAIL",
             "if (last && (ip + len != iend || cpy > oend)) { result = LZ4D_FAIL"),
    "mlen_bytes": ("if (ip > iend - LZ4_LASTLITERALS + 1) return LZ4D_FAIL",
                   "if (ip > iend - LZ4_LASTLITERALS + 1) { result = LZ4D_FAIL"),
    "mlen_oend": ("if (len > oend) return LZ4D_FAIL;                     /* keeps", "if (mlen > oend) { result = LZ4D_FAIL"),
    "general_match": ("if (match < 0) return LZ4D_FAIL;                          /* lz4.c:2356 */",
                      "if (match < 0) { ok = false; LZ4D_FAIL_NOTE(); }"),
    "match_oend": ("if (cpy > oend - LZ4_LASTLITERALS) return LZ4D_FAIL", "cpy > oend - LZ4_LASTLITERALS) { ok = false"),
}
REJECT = {}           # name -> (block, cap, site)


def reject(name, block, site, cap=None):
    assert name not in REJECT and site in SITES
    blk, out = block if isinstance(block, tuple) else (block, None)
    REJECT[name] = (bytes(blk), (len(out) if out is not None else 4096) if cap is None else cap, site)


def _build_reject():
    reject("cap0_not_empty_token", b"\x10a", "cap0", cap=0)
    reject("cap0_two_bytes", b"\x00\x00", "cap0", cap=0)
    reject("empty_input", b"", "csize0", cap=10)
    # match == -1 (one byte before the block) in every tier that checks it
    reject("batch_fast_match_minus_1", tuned([seq(rnd(400, 5), 7, 4)], [dseq(405)] + [dseq(400)] * 10,
                                             need_in=80)[0], "batch_match", cap=5000)
    reject("batch_walk_match_minus_1", tuned([seq(rnd(400, 5), 7, 4)], [seq(b"ab", 407, 8)])[0], "batch_match",
           cap=5000)
    reject("single_match_minus_1", tuned([seq(rnd(40, 5), 7, 4)], [seq(b"ab", 47, 8)], need_in=30)[0],
           "single_match", cap=4000)
    reject("general_match_minus_1", tuned([seq(rnd(200, 5), 7, 4)], [seq(b"L" * 10, 215, 100)])[0],
           "general_match", cap=4000)
    reject("general_match_far", tuned([seq(rnd(200, 5), 7, 4)], [seq(b"L" * 10, 65535, 100)])[0],
           "general_match", cap=4000)
    reject("first_match_offset_1", lw.lz4_block([seq(b"", 1, 20)], rnd(12, 3))[0], "general_match", cap=100)
    # literal lengths: the first extension byte at iend - 15, a chain that runs into iend - 15, longer than cap
    reject("litlen_ext_at_iend_15", bytes([0xF0]) + bytes(14), "litlen_start", cap=100)
    reject("litlen_chain_to_iend_15", bytes([0xF0]) + bytes([255] * 40) + bytes(14), "litlen_bytes", cap=100000)
    reject("litlen_above_cap", bytes([0xF0]) + bytes([255] * 40) + bytes(40), "litlen_oend", cap=1000)
    # last literals: short of iend, past iend, past cap; a match too close to the end
    reject("last_short_of_iend", lw.lz4_block([], rnd(20, 1))[0] + b"\x00", "last", cap=100)
    reject("last_past_iend", lw.lz4_block([], rnd(20, 1))[0][:-1], "last", cap=100)
    reject("litlen_20_past_cap", lw.lz4_block([], rnd(20, 1))[0], "litlen_oend", cap=19)
    reject("last_past_cap", lw.lz4_block([], rnd(10, 1))[0], "last", cap=9)
    reject("literals_end_inside_iend_8", lw.lz4_block([seq(rnd(20, 7), 10, 8)], rnd(4, 8)), "last", cap=60)
    reject("mflimit_one_short", lw.lz4_block([seq(rnd(20, 7), 10, 6)], rnd(5, 8)), "last")
    reject("match_ends_at_oend_4", lw.lz4_block([seq(rnd(20, 7), 10, 12)], rnd(5, 8))[0], "match_oend", cap=36)
    reject("match_past_cap", lw.lz4_block([seq(rnd(20, 7), 10, 40)], rnd(5, 8))[0], "match_oend", cap=60)
    reject("no_final_literals", lw.lz4_block([seq(rnd(20, 7), 10, 8)] * 3, end=False), "last", cap=200)
    # match lengths: the chain runs into iend - 4, longer than cap
    reject("mlen_chain_to_iend_4", bytes([0x1F]) + b"a" + b"\x01\x00" + bytes([255] * 30) + bytes(4), "mlen_bytes",
           cap=100000)
    reject("mlen_above_cap", bytes([0x1F]) + b"a" + b"\x01\x00" + bytes([255] * 30) + bytes([0]) + bytes([0x50]) +
           b"abcde", "mlen_oend", cap=5000)


_build_reject()


@pytest.mark.parametrize("name", sorted(REJECT))
def test_lz4_reject_corpus_emu(lemu, lorc, lref, name):
    blk, cap, site = REJECT[name]
    got, l1, l2, _, _ = lz4_all(lemu, lorc, lref, blk, cap)
    assert got is None
    assert l1 == line_of(SRC_WARP, "LZ4D_FAIL", SITES[site][0]), (l1, fail_lines(SRC_WARP, "LZ4D_FAIL").get(l1))
    assert l2 == line_of(SRC_PAIR, "LZ4D_FAIL", SITES[site][1]), (l2, fail_lines(SRC_PAIR, "LZ4D_FAIL").get(l2))


# ------------------------------------------------------------------------------------------------
# BloscLZ
# ------------------------------------------------------------------------------------------------
lit_, m_ = lw.blz_lit, lw.blz_match
BACCEPT = {}          # name -> (stream, content, cap, hits required, hits forbidden)
BREJECT = {}          # name -> (stream, cap, fragment)


def baccept(name, sc, need=(), forbid=(), room=0):
    st, out = sc
    assert name not in BACCEPT and out is not None
    BACCEPT[name] = (st, out, len(out) + room, set(need), set(forbid))


def breject(name, st, fragment, cap):
    assert name not in BREJECT
    BREJECT[name] = (bytes(st[0] if isinstance(st, tuple) else st), cap, fragment)


def _blz_lead(n=200, seed=3):
    data = rnd(n, seed)
    return [lit_(data[k:k + 32]) for k in range(0, n, 32)]


def _build_blz():
    for n in (1, 2, 31, 32):
        baccept(f"literal_run_{n}", lw.blz_stream([lit_(rnd(n, n))]), ["LITERAL"])
    baccept("literal_runs", lw.blz_stream([lit_(rnd(k, k)) for k in range(1, 33)]), ["LITERAL"])
    for ml in range(3, 9):
        baccept(f"short_match_{ml}", lw.blz_stream(_blz_lead() + [m_(100, ml), lit_(b"end")]))
    for d in (1, 2, 7, 8, 255, 256, 8190, 8191):
        baccept(f"near_dist_{d}", lw.blz_stream(_blz_lead(9000) + [m_(d, 8), m_(d, 40), lit_(b"end")]))
    for ext in ([0], [254], [255, 0], [255, 255, 3]):
        baccept(f"length_bytes_{'_'.join(map(str, ext))}",
                lw.blz_stream(_blz_lead() + [m_(3, 9 + sum(ext), ext=ext), lit_(b"e")]), ["LENEXT"])
    for d in (8192, 8193, 9000, 8192 + 0xFFFF):
        baccept(f"far_dist_{d}", lw.blz_stream(_blz_lead(8192 + 0xFFFF + 10) + [m_(d, 5), m_(d, 30), lit_(b"e")]),
                ["FAR"])
    # the last match dropped when its bytes end the input (length bytes or the far form), with room for it
    baccept("dropped_ext_match", lw.blz_stream(_blz_lead() + [m_(5, 12)]), ["DROPPED", "LENEXT"], room=12)
    baccept("dropped_far_match", lw.blz_stream(_blz_lead(8300) + [m_(8200, 4)]), ["DROPPED", "FAR"], room=4)
    # dense path: chains of 2-byte near matches, a back-off, a run that resumes, a length-byte token inside a run
    dense = [m_(150 + (k % 7), 3 + k % 6) for k in range(100)]
    baccept("dense_chain", lw.blz_stream(_blz_lead(300) + dense + [lit_(b"end")]), ["DENSE"])
    baccept("dense_chain_len_byte", lw.blz_stream(_blz_lead(2100) + dense[:10] + [m_(2000, 9, ext=[0])] + dense[10:] +
                                                  [lit_(b"end")]), ["DENSE", "LENEXT"])
    baccept("dense_chain_far", lw.blz_stream(_blz_lead(9000) + dense[:10] + [m_(8500, 5)] + dense[10:] +
                                             [lit_(b"end")]), ["DENSE", "FAR"])
    baccept("dense_few", lw.blz_stream(_blz_lead(300) + dense[:3] + [lit_(b"x")] + dense[:50] + [lit_(b"end")]),
            ["DENSE_FEW", "DENSE"])
    baccept("dense_bad", lw.blz_stream(_blz_lead(300) + dense[:5] + [m_(1, 8)] + dense[:60] + [lit_(b"end")]),
            ["DENSE", "DENSE_BAD"])
    baccept("dense_bad_lane0", lw.blz_stream(_blz_lead(300) + [m_(2, 8)] + dense[:60] + [lit_(b"end")]),
            ["DENSE"])
    baccept("dense_ref_0", lw.blz_stream([lit_(rnd(30, 1))] + [m_(30 + 3 * k, 3) for k in range(40)] + _blz_lead(320)),
            ["DENSE"])
    # reject corpus
    lead = _blz_lead()
    breject("empty", b"", "if (length == 0) return BLZ_FAIL", 10)
    breject("length_bytes_cut", lw.blz_stream(lead + [m_(3, 9 + 255 + 255, ext=[255, 255, 0])])[0][:-2],
            "length bytes run into the end", 4000)
    breject("code_missing", lw.blz_stream(lead + [m_(3, 5)])[0][:-1], "} else if (ip + 1 >= length)", 4000)
    breject("short_match_last", lw.blz_stream(lead + [m_(3, 5)]), "} else if (ip + 1 >= length)", 4000)
    breject("far_cut", lw.blz_stream(_blz_lead(8300) + [m_(8200, 4)])[0][:-1], "no room for the 16-bit", 9000)
    st, out = lw.blz_stream(lead + [m_(3, 40), lit_(b"end")])
    breject("match_past_cap", st, "if (op + len > maxout)", len(out) - 4)
    breject("dropped_match_past_cap", lw.blz_stream(lead + [m_(5, 12)]), "if (op + len > maxout)", 200)
    breject("ref_minus_1", lw.blz_stream(lead + [m_(201, 5), lit_(b"end")]), "if (ref - 1 < 0)", 4000)
    breject("far_ref_minus_1", lw.blz_stream(lead + [m_(8192, 5, far=True), lit_(b"end")]), "if (ref - 1 < 0)", 4000)
    breject("dense_ref_minus_1", lw.blz_stream([lit_(rnd(30, 1))] + [m_(30 + 3 * k + (k == 20), 3) for k in range(40)] +
                                               [lit_(b"e")]), "if (ref - 1 < 0)", 4000)
    st, out = lw.blz_stream(lead + [lit_(b"abcdef")])
    breject("literal_past_cap", st, "if ((long long)op + ctrl > maxout)", len(out) - 1)
    breject("literal_past_input", st[:-1], "if ((long long)ip + ctrl > length)", 4000)


_build_blz()


@pytest.mark.parametrize("name", sorted(BACCEPT))
def test_blz_accept_corpus_emu(lemu, lorc, lref, name):
    st, content, cap, need, forbid = BACCEPT[name]
    for c in (cap, cap + 9):
        got, _, h = blz_all(lemu, lorc, lref, st, c)
        assert got == content, (c, None if got is None else len(got))
        assert need <= h, ("branch not reached", sorted(need - h))
        assert not (forbid & h), ("branch reached", sorted(forbid & h))
    got, _, _ = blz_all(lemu, lorc, lref, st, cap - 1)
    assert got is None


@pytest.mark.parametrize("name", sorted(BREJECT))
def test_blz_reject_corpus_emu(lemu, lorc, lref, name):
    st, cap, fragment = BREJECT[name]
    got, line, _ = blz_all(lemu, lorc, lref, st, cap)
    assert got is None
    assert line == line_of(SRC_BLZ, "BLZ_FAIL", fragment), (line, fail_lines(SRC_BLZ, "BLZ_FAIL").get(line))


def test_reference_verdicts_pinned(lemu, lorc, lref):
    """LZ4_decompress_safe's and blosclz_decompress's verdicts and bytes for the crafted corpus, recorded"""
    corpus = [("lz4", n, b, cap) for n, (b, c, caps, _, _) in sorted(ACCEPT.items()) for cap in (caps or [len(c)])]
    corpus += [("lz4", n, b, cap) for n, (b, cap, _) in sorted(REJECT.items())]
    corpus += [("blz", n, s, cap) for n, (s, _, cap, _, _) in sorted(BACCEPT.items())]
    corpus += [("blz", n, s, cap) for n, (s, cap, _) in sorted(BREJECT.items())]

    def rec(name, got):
        return (name, -1, np.zeros(0, np.uint8)) if got is None else (name, len(got), np.frombuffer(got, np.uint8))

    def run(lib, names):
        out = []
        for kind, name, st, cap in corpus:
            got = (c_lz4 if kind == "lz4" else c_blz)(lib, names[kind], st, cap)[0]
            out.append(rec(name, got))
        return out
    ours = run(lorc, {"lz4": "orc_lz4_decompress_safe", "blz": "orc_blosclz_decompress"})
    reference = None if lref is None else run(lref, {"lz4": "LZ4_decompress_safe", "blz": "blosclz_decompress"})
    assert_pinned("lz_decode_edges", ours, reference)


# ------------------------------------------------------------------------------------------------
# the ledgers: every fail line and every branch id is reached
# ------------------------------------------------------------------------------------------------
# branch ids no stream can reach, with the reason (none at present).  Not an id: the lone tier's ring threshold
# (offset <= 15872) cannot be crossed, because that tier only takes a long match whose offset is below its length + 8
# (<= 280); any farther one is a dense step.
LZ4_UNREACHED_HITS = {}


def _damaged(blk, rng, k):
    b = bytearray(blk)
    for _ in range(k):
        pos = rng.randrange(len(b))
        b[pos] = rng.getrandbits(8) if rng.random() < 0.5 else b[pos] ^ (1 << rng.randrange(8))
    return bytes(b)


def test_lz4_ledger(lemu, lorc, lref):
    reached_w = {line_of(SRC_WARP, "LZ4D_FAIL", SITES[s][0]) for _, _, s in REJECT.values()}
    reached_p = {line_of(SRC_PAIR, "LZ4D_FAIL", SITES[s][1]) for _, _, s in REJECT.values()}
    seen = set()
    for blk, content, caps, _, _ in ACCEPT.values():
        for cap in caps or (len(content),):
            _, _, _, h1, h2 = lz4_all(lemu, lorc, lref, blk, cap)
            seen |= h1 | h2
    missing_w = {k: t.strip() for k, t in fail_lines(SRC_WARP, "LZ4D_FAIL").items() if k not in reached_w}
    missing_p = {k: t.strip() for k, t in fail_lines(SRC_PAIR, "LZ4D_FAIL").items() if k not in reached_p}
    assert not missing_w and not missing_p, (missing_w, missing_p)
    assert set(H) - seen == set(LZ4_UNREACHED_HITS), sorted(set(H) - seen)


def test_blz_ledger(lemu, lorc, lref):
    reached = {line_of(SRC_BLZ, "BLZ_FAIL", f) for _, _, f in BREJECT.values()}
    seen = set()
    for st, _, cap, _, _ in BACCEPT.values():
        seen |= blz_all(lemu, lorc, lref, st, cap)[2]
    missing = {k: t.strip() for k, t in fail_lines(SRC_BLZ, "BLZ_FAIL").items() if k not in reached}
    assert not missing, missing
    assert set(BH) - seen == set(), sorted(set(BH) - seen)


# ------------------------------------------------------------------------------------------------
# ring reuse: a CTA that draws several tickets does not clear the ring between streams
# ------------------------------------------------------------------------------------------------
def decode_list(emu, streams, caps, pair):
    """the streams one after another through one warp (or one parser / copier pair) in one launch: [(rc, bytes,
    canary intact, fail line)]"""
    n = len(streams)
    srcs = [_src(s) for s in streams]
    outs = [np.full(c + 64, CANARY, np.uint8) for c in caps]
    res, lines = (C.c_int * n)(), (C.c_int * n)()
    emu.emu_lz4_decode_list((C.c_void_p * n)(*[s.ctypes.data for s in srcs]), (C.c_int * n)(*[len(s) for s in streams]),
                            (C.c_void_p * n)(*[o.ctypes.data for o in outs]), (C.c_int * n)(*caps), n, int(pair), res,
                            lines)
    return [(res[i], outs[i][:max(res[i], 0)].tobytes(), bool((outs[i][caps[i]:] == CANARY).all()), lines[i])
            for i in range(n)]


def ring_pairs():
    """(name, stream A, stream B): A leaves a distinctive pattern in the whole ring; B then reads, within 16 KiB,
    output it wrote by a path that does not mirror into the ring (a long match, an offset-0 fill, a literal run
    longer than the ring), so only ring_lo keeps B from reading A's bytes"""
    pat = bytes((i * 7 + 0xAB) & 255 for i in range(20000))
    a = lw.lz4_block([], pat)
    lit = rnd(12, 4)
    readers = {
        "single": [seq(b"ab", 50, 8)],
        "batch": [dseq(900)] * 11,
        "general": [seq(b"L" * 10, 300, 100)],
        "lone": [lseq(3, 119)],
        "dense": [seq(b"f" * 10, 9, 4)] + [dseq(1900 - 40 * k, 18) for k in range(32)],
    }
    out = []
    for wname, writer in (("off0", seq(lit, 0, 3000)), ("long_copy", seq(lit, 5, 3000)),
                          ("long_copy_2049", seq(lit, 1, 2049))):
        for rname, reader in readers.items():
            need_in = {"single": 30, "batch": 90}.get(rname)
            out.append((f"{wname}_then_{rname}", a, tuned([writer], reader, need_in=need_in)))
    big = rnd(20000, 8)
    out.append(("literal_run_then_single", a, tuned([seq(big, 16310, 8)], [seq(b"ab", 16300, 8)], need_in=30)))
    return out


@pytest.mark.parametrize("pair", [False, True])
def test_ring_reuse_across_streams_emu(lemu, pair):
    for name, a, (b, want) in ring_pairs():
        res = decode_list(lemu, [a[0], b, a[0], b], [len(a[1]), len(want), len(a[1]), len(want)], pair)
        for (r, got, canary, _), exp in zip(res, [a[1], want, a[1], want]):
            assert r == len(exp) and got == exp and canary, (name, r)
    # a rejected stream in the middle leaves the next one unharmed
    bad = REJECT["general_match_far"]
    a, (b, want) = ring_pairs()[0][1:]
    res = decode_list(lemu, [a[0], bad[0], b], [len(a[1]), bad[1], len(want)], pair)
    assert res[1][0] == -1 and res[2][0] == len(want) and res[2][1] == want


# ------------------------------------------------------------------------------------------------
# random structured streams, drawn to straddle the thresholds, then damaged
# ------------------------------------------------------------------------------------------------
OFFS = [1, 2, 3, 7, 8, 18, 19, 31, 32, 33, 280, 281, 319, 320, 13696, 13697, 14272, 14273, 15872, 15873, 16000,
        16001, 16320, 16321, 65535]
MLS = list(range(4, 19)) * 3 + [19, 20, 272, 273, 274, 2048, 2049, 3000]


def random_block(rng):
    seqs = []
    n = rng.choice([20, 400, 3000, 14000, 16330, 17000])
    seqs.append(seq(rnd(n, rng.getrandbits(16)), rng.choice([1, 7, 20]), rng.choice([4, 8, 100, 2049])))
    n += seqs[0]["ml"]
    for _ in range(rng.randint(1, 120)):
        u = rng.random()
        lits = 0 if u < 0.5 else rng.randint(1, 9) if u < 0.8 else rng.randint(10, 20) if u < 0.97 else \
            rng.choice([16320, 16321])
        reach = n + lits
        offs = [o for o in OFFS if o <= reach] + [rng.randint(1, min(reach, 65535))]
        off = 0 if rng.random() < 0.02 else rng.choice(offs)
        ml = rng.choice(MLS)
        seqs.append(seq(rnd(lits, rng.getrandbits(16)), off, ml))
        n += lits + ml
    return lw.lz4_block(seqs, rnd(rng.randint(5, 300), rng.getrandbits(16)))


def test_random_streams_emu(lemu, lorc, lref):
    rng = random.Random(1234)
    seen = set()
    for t in range(300):
        blk, want = random_block(rng)
        got, _, _, h1, h2 = lz4_all(lemu, lorc, lref, blk, len(want))
        assert got == want, t
        seen |= h1 | h2
        for k in (1, 3):
            bad = _damaged(blk, rng, k)
            lz4_all(lemu, lorc, lref, bad, len(want) + rng.choice([0, 0, 7]))
    assert len(seen) >= 20, sorted(set(H) - seen)


def random_blz(rng):
    items = [lw.blz_lit(rnd(rng.randint(1, 32), rng.getrandbits(16)))]
    n = len(items[0]["data"])
    for _ in range(rng.randint(1, 200)):
        u = rng.random()
        if u < 0.25:
            d = rnd(rng.randint(1, 32), rng.getrandbits(16))
            items.append(lw.blz_lit(d))
            n += len(d)
            continue
        dist = rng.choice([1, 2, 3, 8, 100, 8191, rng.randint(1, n)])
        if n > 8192 and rng.random() < 0.2:
            dist = rng.randint(8192, min(n, 8192 + 0xFFFF))
        dist = min(dist, n)
        ml = rng.choice([3, 4, 5, 6, 7, 8, 9, 10, 40, 264, 300])
        items.append(lw.blz_match(dist, ml))
        n += ml
    items.append(lw.blz_lit(b"end"))
    return lw.blz_stream(items)


def test_random_blz_streams_emu(lemu, lorc, lref):
    rng = random.Random(99)
    seen = set()
    for t in range(300):
        st, want = random_blz(rng)
        got, _, h = blz_all(lemu, lorc, lref, st, len(want))
        assert got == want, t
        seen |= h
        bad = _damaged(st, rng, rng.choice([1, 2]))
        blz_all(lemu, lorc, lref, bad, len(want) + rng.choice([0, 5]))
    assert seen >= {"DENSE", "FAR", "LENEXT", "LITERAL"}, seen


# ------------------------------------------------------------------------------------------------
# Blosc chunks of crafted streams: unsplit single-stream blocks, and typesize-4 blocks of four streams
# ------------------------------------------------------------------------------------------------
def lz_chunk(streams, neblock, codec, split):
    """a one-block chunk: unsplit (flags DONT_SPLIT, one stream) or split (typesize 4, four streams of neblock bytes
    each).  A stream given as ("raw", data) is stored (its size equals neblock)."""
    payload = b""
    for s in streams:
        payload += struct.pack("<i", len(s)) + s
    nbytes = neblock * len(streams)
    flags = (codec << 5) | (0 if split else 0x10)
    head = bytes([2, 1, flags, 4 if split else 1]) + struct.pack("<iii", nbytes, nbytes, 16 + 4 + len(payload))
    return head + struct.pack("<i", 20) + payload, nbytes


def chunk_corpus():
    """(name, chunk, nbytes): every crafted LZ4 and BloscLZ stream whose size differs from its output (a block as
    long as its output reads as stored) in an unsplit chunk, and each accepted LZ4 stream of 128 bytes or more in a
    split chunk next to a stored stream"""
    out = []
    for n, (b, c, caps, _, _) in sorted(ACCEPT.items()):
        cap = (caps or [len(c)])[0]
        if cap and len(b) != cap:
            out.append(("lz4_" + n,) + lz_chunk([b], cap, 1, False))
        if len(c) >= 128 and len(b) != len(c) and caps is None:
            raw = rnd(len(c), 11)
            out.append(("lz4_split_" + n,) + lz_chunk([b, raw, b, b], len(c), 1, True))
    for n, (b, cap, _) in sorted(REJECT.items()):
        if cap and len(b) != cap:
            out.append(("lz4_reject_" + n,) + lz_chunk([b], cap, 1, False))
    b, c = ACCEPT["dense_off_13696"][:2]
    out.append(("lz4_split_one_bad",) + lz_chunk([b, b, b[:-1] + bytes([b[-1] ^ 1]), b], len(c), 1, True))
    for n, (s, c, cap, _, _) in sorted(BACCEPT.items()):
        if len(s) != cap:
            out.append(("blz_" + n,) + lz_chunk([s], cap, 0, False))
    for n, (s, cap, _) in sorted(BREJECT.items()):
        if cap and len(s) != cap:
            out.append(("blz_reject_" + n,) + lz_chunk([s], cap, 0, False))
    return out


def _chunk_decode(lib, fn, ch, n):
    c = np.frombuffer(ch, np.uint8).copy()
    out = np.full(n + 32, CANARY, np.uint8)
    r = getattr(lib, fn)(ptr(c), ptr(out), sz(n), C.c_int(1))
    assert (out[n:] == CANARY).all()
    item = np.full(n + 8, 0x33, np.uint8)
    ts = ch[3]                                                # getitem counts items of `typesize` bytes
    g = getattr(lib, fn.replace("decompress_ctx", "getitem"))(ptr(c), C.c_int(0), C.c_int(n // ts), ptr(item))
    return r, out[:n].tobytes(), g, item[:n].tobytes()


def test_chunks_emu_against_reference(lemu, lorc, ref_if_built):
    lemu.blosc_getitem.restype = C.c_int
    lorc.orc_getitem.restype = C.c_int
    nok = 0
    for pair in (1, 0):
        lemu.emu_set_lz4d_pair(pair)
        try:
            for name, ch, n in chunk_corpus():
                r, o, g, i = _chunk_decode(lemu, "blosc_decompress_ctx", ch, n)
                r2, o2, g2, i2 = _chunk_decode(lorc, "orc_decompress_ctx", ch, n)
                assert (r, g) == (r2, g2) and (r != n or o == o2) and (g != n or i == i2), (name, r, r2, g, g2)
                if ref_if_built is not None:
                    r3, o3, g3, i3 = _chunk_decode(ref_if_built, "blosc_decompress_ctx", ch, n)
                    assert (r, g) == (r3, g3) and (r != n or o == o3), (name, r, r3, g, g3)
                nok += r == n
        finally:
            lemu.emu_set_lz4d_pair(1)
    assert nok > 200


@pytest.mark.gpu
def test_crafted_chunks_gpu(pkg, cuda, lemu):
    """The crafted chunks through the CUDA library, from host and device buffers, in both shapes (unsplit blocks go to
    decode_kernel, four-stream blocks to decode_pair_kernel): the emulator's return code and bytes, nothing written
    past destsize."""
    for name, ch, n in chunk_corpus():
        c = np.frombuffer(ch, np.uint8).copy()
        want = np.full(n + 32, CANARY, np.uint8)
        r0 = lemu.blosc_decompress_ctx(ptr(c), ptr(want), sz(n), C.c_int(1))
        out = np.full(n + 32, CANARY, np.uint8)
        r = pkg.decompress_ctx(c, out[:n], n)
        assert r == r0 and (r < 0 or (out[:n] == want[:n]).all()) and (out[n:] == CANARY).all(), (name, r, r0)
        d_c = cuda.from_numpy(c).cuda()
        d_o = cuda.full((n + 32,), CANARY, dtype=cuda.uint8, device="cuda")
        r = pkg.decompress_ctx(d_c, d_o[:n], n)
        o = d_o.cpu().numpy()
        assert r == r0 and (r < 0 or (o[:n] == want[:n]).all()) and (o[n:] == CANARY).all(), (name, r, r0)

"""The one-warp LZ4 encoder (lz4_encode_stream without TEAM, csrc/dev_lz4.cuh) and the BloscLZ encoder
(blz_encode_warp, csrc/dev_blosclz.cuh) branch by branch, on inputs built to order (tests/lz_encode_write.py).

Generated data seldom reaches the branches where an encoder that replays the reference can go subtly wrong: the
65535-distance rule, the skip schedule past 64 probes, catch-ups of 32 bytes and more, 270+ matches leaving the
chain, BloscLZ's far-distance and MAX_FARDISTANCE rules, the entropy probe's threshold per clevel, bit 16 of the
packed tables.  Each scenario here is built for some of them and asserts the branch ids (LZ4E_H_* / BLZE_H_*, counted
by emulator builds only) it reaches at the acceleration or clevel it was built for.  Every scenario then runs at
every acceleration 1..9 (LZ4, in the table flavours it applies to) or clevel 1..9 and split 0 / 1 (BloscLZ), at full
capacity, at its exact fit and at fit - 1; return code, bytes and the smallest accepted capacity (emu_last_need)
must be the oracle's, and the oracle must decode the output back to the source.  Where oracle/_ref is built the same
calls go to LZ4_compress_fast / blosclz_compress; their results are pinned in tests/golden/reference_results.json.
Ledgers fail if an id goes unreached.  The scenarios wrapped into Blosc chunks run through the emulator's chunk path
(encode_kernel, and the team encoder, pack on and off) and, with -m gpu, through the CUDA library."""
import ctypes as C
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

import lz_encode_write as ew
from datagen import assert_pinned, bench_words, ci, compress, gen, ptr
from lz_encode_write import Stream, probe_offset
from test_lz4_team import chains_and_gaps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "c-blosc_b200", "csrc")
SRC_LZ4 = os.path.join(CSRC, "dev_lz4.cuh")
SRC_BLZ = os.path.join(CSRC, "dev_blosclz.cuh")

# branch ids: the order of the enums in dev_lz4.cuh and dev_blosclz.cuh
LH = ["WIN_PREFETCHED", "WIN_BLOCKING", "WIN_PB_OFF", "WIN_FLUSH", "CH_MISS", "CH_D65535", "CH_D65536",
      "CH_LEN_REG", "CH_LEN_X3", "CH_LEN_X4", "CH_TAIL_BALLOT", "CH_TAIL_LOOP", "CH_HUGE", "CH_EXT",
      "CH_END_LAST", "CH_END_PROBE",
      "POST_WIDE", "POST_NARROW", "POST_HIT", "POST_MISS", "POST_D65535", "POST_D65536",
      "SP_HIT0", "SP_HIT1", "SP_HIT2", "SP_HIT3", "SP_ENDED", "SP_D65535", "SP_D65536",
      "R_HIT", "R_FWD_HIT", "R_FWD_MISS", "R_PARTIAL", "R_STEP64", "R_STEP128", "R_STEP192",
      "CU_NONE", "CU_SHORT", "CU_LONG", "CU_ANCHOR", "CU_ZERO",
      "ML_NEXT", "ML_X0", "ML_X1", "ML_X2", "ML_TAIL", "ML_ROOM20", "ML_ROOM4", "ML_CLAMP", "ML_NARROW",
      "EM_COMPACT", "EM_LIT_FF0", "EM_LIT_FF1", "EM_LIT_FF2", "EM_ML_FF0", "EM_ML_FF1", "EM_ML_FF2", "EM_IMM", "EM_LITS",
      "LIM_FLUSH", "LIM_FIRST", "LIM_COMPACT", "LIM_LONG", "LIM_LAST",
      "LAST_SHORT", "LAST_FF0", "LAST_FF1", "LAST_NOPARSE",
      "TAB_U16", "TAB_U32", "TAB_PACK", "PACK_HI"]
BH = ["PROBE_BELOW", "PROBE_EQUAL", "PROBE_ABOVE", "PROBE_EXT", "SHIFT3_NOSPLIT", "SHIFT3_LOWRATIO", "SHIFT4",
      "REF_SHORT", "REF_MAXOUT", "TAB_HL12", "TAB_HL13", "TAB_HL14", "TAB_17", "TAB_32", "TAB17_HI",
      "R_LANE0", "R_LANE31", "R_NONE", "R_FWD", "R_PARTIAL", "R_MINLEN3", "R_BELOW3", "R_MINLEN4", "R_BELOW4",
      "EXT_MISMATCH", "EXT_BOUND", "FAR5", "FAR6", "MAXFAR_M1", "MAXFAR",
      "P1_HIT", "P1_DIST", "P1_BYTES", "P1_LEN", "NEAR8190", "FAR8191", "SHORT_NEAR", "SHORT_FAR",
      "LONG_NEAR0", "LONG_NEAR1", "LONG_NEAR2", "LONG_FAR0", "LONG_FAR1", "LONG_FAR2", "COPY0", "LIT_CROSS",
      "L9_STORE", "LIM_LIT", "LIM_SHORT", "LIM_LONG", "LIM_CTRL", "LIM_LEFT"]

# ids no input can reach, with the reason
LZ4_UNREACHED = {
    "ML_ROOM4": "room <= 4 needs ip + 13 >= n, but have_next (the only way into that branch) needs ip + 14 <= n "
                "(post-match probe) or ip + 16 <= n (scalar probe)",
    "ML_CLAMP": "every count is bounded by matchlimit, so mc never exceeds room when room > 4",
}
# Not an id: PACK's clearing atomicAnd.  A stream's positions only grow and its table is zeroed first, so no store
# clears a bit that is set; the packed scenarios check that bit 16 is read (PACK_HI) and set by two lanes of a round.


def test_branch_id_tables_match_source():
    text = open(SRC_LZ4).read()
    body = text[text.index("LZ4E_H_WIN_PREFETCHED"):text.index("LZ4E_NHIT\n")]
    names = []
    for line in body.split("\n"):
        line = line.split("/*")[0]
        names += [w.split("=")[0].strip() for w in line.split(",") if w.strip()]
    # LZ4E_H_SP_ENDED = LZ4E_H_SP_HIT0 + 4: the three ids between are SP_HIT0 + 1..3
    i = names.index("LZ4E_H_SP_HIT0")
    names[i + 1:i + 1] = ["LZ4E_H_SP_HIT1", "LZ4E_H_SP_HIT2", "LZ4E_H_SP_HIT3"]
    assert ["LZ4E_H_" + h for h in LH] == names
    text = open(SRC_BLZ).read()
    body = text[text.index("BLZE_H_PROBE_BELOW"):text.index("BLZE_NHIT\n")]
    names = []
    for line in body.split("\n"):
        line = line.split("/*")[0]
        names += [w.strip() for w in line.split(",") if w.strip()]
    assert ["BLZE_H_" + h for h in BH] == names


# ------------------------------------------------------------------------------------------------
# fixtures and the calls
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eemu(emu):
    emu.emu_lz4_encode.restype = C.c_int
    emu.emu_lz4_encode.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    emu.emu_blz_encode.restype = C.c_int
    emu.emu_blz_encode.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    emu.emu_last_need.restype = C.c_int
    for f in ("emu_lz4e_hits", "emu_blze_hits"):
        getattr(emu, f).restype = C.c_int
        getattr(emu, f).argtypes = [C.c_void_p]
    lhits(emu)
    bhits(emu)
    return emu


@pytest.fixture(scope="module")
def eorc(orc):
    orc.orc_lz4_compress_fast.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    orc.orc_blosclz_compress.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    orc.orc_lz4_decompress_safe.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    orc.orc_blosclz_decompress.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    return orc


@pytest.fixture(scope="module")
def eref(ref_if_built):
    r = ref_if_built
    if r is not None:
        r.LZ4_compress_fast.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        r.blosclz_compress.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    return r


def lhits(emu):
    h = (C.c_longlong * 128)()
    n = emu.emu_lz4e_hits(h)
    assert n == len(LH)
    return {LH[i] for i in range(n) if h[i]}


def bhits(emu):
    h = (C.c_longlong * 128)()
    n = emu.emu_blze_hits(h)
    assert n == len(BH)
    return {BH[i] for i in range(n) if h[i]}


FILL = 0xA5


def lz4_call(lib, fname, src, cap, accel):
    out = np.full(cap + 64, FILL, np.uint8)
    r = getattr(lib, fname)(ptr(src), ptr(out), len(src), cap, accel)
    assert (out[cap:] == FILL).all(), "written past the capacity"
    return r, out[:max(r, 0)].copy()


def blz_call(lib, fname, src, cap, clevel, split):
    out = np.full(cap + 64, FILL, np.uint8)
    r = getattr(lib, fname)(clevel, ptr(src), len(src), ptr(out), cap, split)
    assert (out[cap:] == FILL).all(), "written past the capacity"
    return r, out[:max(r, 0)].copy()


def emu_lz4(emu, src, cap, accel):
    out = np.full(cap + 64, FILL, np.uint8)
    r = emu.emu_lz4_encode(ptr(src), len(src), ptr(out), cap, accel)
    assert (out[cap:] == FILL).all(), "written past the capacity"
    return r, out[:max(r, 0)].copy(), emu.emu_last_need(), lhits(emu)


def emu_blz(emu, src, cap, clevel, split):
    out = np.full(cap + 64, FILL, np.uint8)
    r = emu.emu_blz_encode(clevel, ptr(src), len(src), ptr(out), cap, split)
    assert (out[cap:] == FILL).all(), "written past the capacity"
    return r, out[:max(r, 0)].copy(), emu.emu_last_need(), bhits(emu)


def _min_cap(accepts, hi):
    if not accepts(hi):
        return None
    lo = 0
    while lo < hi:
        mid = (lo + hi) // 2
        if accepts(mid):
            hi = mid
        else:
            lo = mid + 1
    return lo


def lz4_full(n):
    return n + n // 255 + 16                    # LZ4_compressBound: not limited (lz4.c:1388)


def check_lz4(eemu, eorc, src, accel, extra_caps=()):
    """the emulator against the oracle at full capacity, at the oracle's exact fit and at fit - 1 (and extra_caps):
    return code, bytes, need; the oracle decodes its output back to the source.  Returns the ids reached at full
    capacity and the union over the capacities."""
    n = len(src)
    full = lz4_full(n)
    r, o, need, h0 = emu_lz4(eemu, src, full, accel)
    ro, oo = lz4_call(eorc, "orc_lz4_compress_fast", src, full, accel)
    assert r == ro > 0 and np.array_equal(o, oo), (n, accel, r, ro)
    back = np.zeros(n + 64, np.uint8)
    assert eorc.orc_lz4_decompress_safe(ptr(oo), ptr(back), ro, n) == n and np.array_equal(back[:n], src)
    fit = _min_cap(lambda c: lz4_call(eorc, "orc_lz4_compress_fast", src, c, accel)[0] > 0, full)
    assert need == fit, (n, accel, need, fit)
    seen = set(h0)
    for cap in sorted({fit, fit - 1, *extra_caps}):
        if cap < 0:
            continue
        rc, oc, _, h = emu_lz4(eemu, src, cap, accel)
        rr, orr = lz4_call(eorc, "orc_lz4_compress_fast", src, cap, accel)
        assert rc == rr and np.array_equal(oc, orr), (n, accel, cap, rc, rr)
        assert (rc > 0) == (cap >= fit)
        seen |= h
    return h0, seen


def check_blz(eemu, eorc, src, clevel, split, extra_caps=()):
    n = len(src)
    r, o, need, h0 = emu_blz(eemu, src, n, clevel, split)
    ro, oo = blz_call(eorc, "orc_blosclz_compress", src, n, clevel, split)
    assert r == ro and np.array_equal(o, oo), (n, clevel, split, r, ro)
    seen = set(h0)
    if ro > 0:
        back = np.zeros(n + 64, np.uint8)
        assert eorc.orc_blosclz_decompress(ptr(oo), ro, ptr(back), n) == n and np.array_equal(back[:n], src)
        fit = _min_cap(lambda c: blz_call(eorc, "orc_blosclz_compress", src, c, clevel, split)[0] > 0, n)
        assert need == fit, (n, clevel, split, need, fit)
        caps = {fit, fit - 1, *extra_caps}
    else:
        caps = set(extra_caps)
    for cap in sorted(caps):
        if cap < 0:
            continue
        rc, oc, _, h = emu_blz(eemu, src, cap, clevel, split)
        rr, orr = blz_call(eorc, "orc_blosclz_compress", src, cap, clevel, split)
        assert rc == rr and np.array_equal(oc, orr), (n, clevel, split, cap, rc, rr)
        seen |= h
    return h0, seen


# ------------------------------------------------------------------------------------------------
# LZ4 scenarios: name -> (source, acceleration it was built for, ids it must reach there, packed table wanted)
# ------------------------------------------------------------------------------------------------
def _periodic_to(st, end, unit=64):
    """noise of `unit` bytes repeated up to position `end`: one long match (found by the search, general emission)
    that ends exactly at `end` (the caller's next bytes must differ from those `unit` back)"""
    st.noise(unit)
    st.repeat(unit, end - len(st))
    return st


def _key_at(dist, tail, seed):
    """key at 0, a long periodic match up to `dist`, the key again at `dist`, then `tail` bytes of noise: the probe
    at `dist` finds the key at distance exactly `dist` (its bucket was never stored)"""
    st = Stream(seed)
    st.put(ew.rnd(16, seed))
    _periodic_to(st, dist)
    key = bytearray(st.b[:8])
    if key[0] == st.b[dist - 64]:
        key[0] ^= 0x80
        st.b[0] = key[0]
    st.put(key)
    st.noise(tail)
    return st


def lz4_scenarios():
    sc = {}
    for d in (65535, 65536):
        sc[f"post_dist_{d}"] = (_key_at(d, 12, 3).array(), 1, {"POST_WIDE", f"POST_D{d}", "TAB_U32"}, False)
        sc[f"chain_dist_{d}"] = (_key_at(d, 200, 5).array(), 1, {f"CH_D{d}", "TAB_U32"}, False)
        for k in ((0, 1, 2, 3) if d == 65535 else (0, 2)):
            st = Stream(10 + k)
            st.put(ew.rnd(16, 10 + k))
            e0 = d - 1 - probe_offset(k, 1)
            _periodic_to(st, e0)
            st.noise_to(d, ends=64)
            st.put(st.b[:8])
            st.noise(150)
            want = {f"SP_D{d}", "CH_MISS"} | ({f"SP_HIT{k}"} if d == 65535 else set())
            sc[f"probe{k}_dist_{d}"] = (st.array(), 1, want, False)
    for it, ids in ((10, {"R_HIT"}), (70, {"R_HIT", "R_STEP64"}), (140, {"R_HIT", "R_STEP128"}),
                    (200, {"R_HIT", "R_STEP192"})):
        st = Stream(20 + it)
        st.put(ew.rnd(16, 20 + it))
        _periodic_to(st, 5000)
        st.noise_to(5001 + probe_offset(it, 1), ends=64)
        st.put(st.b[:8])
        st.noise_to(20000)
        sc[f"round_it{it}"] = (st.array(), 1, ids | {"TAB_U16"}, False)
    for lit in (14, 15, 269, 270, 524, 525):
        for mc in (14, 15, 269, 270, 524, 525):
            if lit not in (14, 525) and mc not in (14, 525) and lit != mc:
                continue
            st = Stream(1000 * lit + mc)
            st.noise(lit)
            st.repeat(lit, mc + 4)
            st.noise(300, ends=lit)
            # from 270 literals on the first probe that hits lands past the repeat's start: caught up to position 0
            ids = {"EM_LITS"} | ({"CU_ZERO"} if lit >= 270 else set())
            ids |= {"EM_COMPACT"} if lit < 15 and mc < 15 else set()
            ids |= {"EM_LIT_FF%d" % ((lit - 15) // 255)} if lit >= 15 else set()
            ids |= {"EM_ML_FF%d" % ((mc - 15) // 255)} if mc >= 15 else set()
            sc[f"lit{lit}_ml{mc}"] = (st.array(), 1, ids, False)
    for last in list(range(5, 16)) + [269, 270, 400]:
        st = Stream(300 + last)
        st.noise(40)
        st.repeat(40, 200)
        st.noise(last, ends=40)
        ids = {"LAST_SHORT" if last < 15 else "LAST_FF0" if last < 270 else "LAST_FF1"}
        sc[f"last{last}"] = (st.array(), 1, ids, False)
    for n in range(0, 13):
        sc[f"tiny{n}"] = (np.frombuffer(bytes(ew.rnd(n, n)), np.uint8).copy(), 1, {"LAST_NOPARSE", "LAST_SHORT"}, False)
    for k in (14, 20, 29):
        # the post-match probe at e finds position 2 (a scalar probe stored it) with k - 9 bytes of room
        st = Stream(400 + k)
        st.noise(30)
        st.repeat(30, 30)
        st.put(st.b[2:2 + k])
        sc[f"near_end{k}"] = (st.array(), 1, {"ML_ROOM20", "POST_HIT"}, False)
    for k in (12, 14):
        st = Stream(410 + k)
        st.noise(30)
        st.repeat(30, k)
        sc[f"narrow_end{k}"] = (st.array(), 1, {"ML_NARROW"}, False)
    # a chained record whose match runs to matchlimit: the chain ends with ip >= mfl1, and its parked records are
    # the last thing checked before 5 last literals (at fit - 1 the flush refuses)
    st = Stream(450)
    st.noise(40)
    st.repeat(40, 300)
    st.put(st.b[2:102])
    sc["chain_to_end"] = (st.array(), 1, {"CH_END_LAST"}, False)
    # a compact sequence, then the 5 last literals: at fit - 1 the compact-sequence check refuses
    st = Stream(460)
    st.noise(10)
    st.repeat(10, 18)
    st.noise(5, ends=10)
    sc["compact_then_end"] = (st.array(), 1, {"EM_COMPACT", "LAST_SHORT"}, False)
    # two lanes of one round with one hash: the second finds the first (forwarded), or its twin with other bytes
    for same in (True, False):
        st = Stream(500 + same)
        st.put(ew.rnd(16, 500))
        _periodic_to(st, 3000)
        st.noise_to(3010, ends=64)
        y = bytes(ew.rnd(4, 501))
        st.put(y)
        st.noise_to(3020)
        st.put(y if same else ew.hash_twin(y, lambda b: ew.hash_u16(b, 0), 7))
        st.noise_to(8000)
        sc[f"round_shared_hash_{'hit' if same else 'miss'}"] = (st.array(), 1,
                                                               {"R_FWD_HIT" if same else "R_FWD_MISS"}, False)
    # bit 16 of the packed table: a repeat whose candidate lies past 65536
    st = Stream(600)
    st.put(ew.rnd(16, 600))
    _periodic_to(st, 70000)
    st.noise(40, ends=64)
    st.repeat(40, 300)
    st.noise_to(80000, ends=40)
    sc["pack_bit16"] = (st.array(), 1, {"TAB_PACK", "PACK_HI"}, True)
    # generated and structured data: chains on the lane-cached window, catch-ups, long rounds
    sc["chains_and_gaps"] = (chains_and_gaps(40000, seed=41), 1, {"WIN_PREFETCHED", "CH_LEN_REG"}, False)
    sc["chains_and_gaps_u32"] = (chains_and_gaps(100000, seed=43), 5, {"TAB_U32"}, False)
    w = bench_words(4 * 30000)
    sc["bench_plane1"] = (np.ascontiguousarray(w.reshape(-1, 4)[:, 1]), 1, {"WIN_PREFETCHED", "WIN_FLUSH"}, False)
    sc["bench_plane2"] = (np.ascontiguousarray(w.reshape(-1, 4)[:, 2]), 9, set(), False)
    sc["random"] = (np.frombuffer(bytes(ew.rnd(5000, 77)), np.uint8).copy(), 1, {"R_PARTIAL", "LAST_FF1"}, False)
    return sc


LZ4_SC = lz4_scenarios()


_LZ4_SEEN = set()                   # ids the scenario tests reached, for the ledgers
_BLZ_SEEN = set()


@pytest.mark.parametrize("name", sorted(LZ4_SC))
def test_lz4_scenario_emu(eemu, eorc, name):
    """at the acceleration it was built for, the scenario reaches its ids; at every acceleration, full capacity, exact
    fit and fit - 1 (and for short streams every capacity up to the fit), the emulator gives the oracle's results"""
    src, accel, want, pack = LZ4_SC[name]
    seen = set()
    for p in ([True, False] if pack else [False]):
        eemu.emu_set_lz4_pack(C.c_int(p))
        try:
            for a in range(1, 10):
                sweep = range(0, lz4_full(len(src))) if len(src) <= 1400 and a == accel else ()
                h0, s = check_lz4(eemu, eorc, src, a, sweep)
                if a == accel and p == pack:
                    assert want <= h0, (name, sorted(want - h0))
                seen |= s
        finally:
            eemu.emu_set_lz4_pack(C.c_int(0))
    _LZ4_SEEN.update(seen)


# ------------------------------------------------------------------------------------------------
# BloscLZ scenarios: name -> (source, clevel and split it was built for, ids it must reach there, packed table)
# ------------------------------------------------------------------------------------------------
THRESHOLDS = {1: Fraction(2), 2: Fraction(3, 2), 5: Fraction(6, 5), 7: Fraction(23, 20), 8: Fraction(11, 10), 9: Fraction(1)}
BLZ_MAXFAR = 65535 + 8191 - 1


def _blz_repeat(dist, m, seed, total):
    """noise with m bytes Y at p0, a periodic gap (one long match: its positions are never stored, so Y's bucket
    keeps p0), Y again at p0 + dist followed by noise: a match of exactly m equal bytes at distance dist"""
    st = Stream(seed)
    st.noise(100)
    p0 = len(st)
    st.noise(m)
    st.noise(20, ends=0)
    _periodic_to(st, p0 + dist - 40)
    st.noise_to(p0 + dist, ends=64)
    st.put(st.b[p0:p0 + m])
    st.noise(200, ends=dist)
    st.noise_to(total)
    return st


def _compressible_window(st):
    """zeros where the entropy probe looks (the 4096 bytes from three quarters of the stream on), so that it passes"""
    s = 3 * len(st) // 4
    st.b[s:s + 4096] = bytes(len(st.b[s:s + 4096]))


def blz_scenarios():
    sc = {}
    for clevel, want in THRESHOLDS.items():
        for which in ("below", "equal", "above"):
            w = ew.probe_window(want, which, seed=clevel)
            src = np.frombuffer(w * 4, np.uint8).copy()           # the probe reads the last quarter
            sc[f"probe_{clevel}_{which}"] = (src, clevel, 1, {"PROBE_" + which.upper()}, True)
    sc["shift4"] = (np.zeros(20000, np.uint8), 5, 1, {"SHIFT4", "EXT_BOUND"}, True)
    sc["shift3_nosplit"] = (np.zeros(20000, np.uint8), 5, 0, {"SHIFT3_NOSPLIT"}, True)
    sc["text"] = (gen("text", 30000, seed=3), 5, 1, {"SHIFT3_LOWRATIO", "P1_HIT", "P1_BYTES", "P1_LEN", "COPY0",
                                                      "R_LANE0", "LIT_CROSS", "SHORT_NEAR", "TAB_HL14", "TAB_17"}, True)
    sc["ramp_hl12"] = (gen("ramp", 30000), 1, 1, {"TAB_HL12"}, True)
    sc["ramp_hl13"] = (gen("ramp", 30000), 2, 1, {"TAB_HL13"}, True)
    sc["text_tab32"] = (gen("text", 30000, seed=6), 5, 1, {"TAB_32"}, False)
    sc["text_l9"] = (gen("text", 30000, seed=7), 9, 1, {"L9_STORE"}, True)
    sc["short"] = (np.zeros(15, np.uint8), 0, 1, {"REF_SHORT"}, True)
    sc["zeros_maxout"] = (np.zeros(3000, np.uint8), 5, 1, set(), True)
    # exact match lengths: m equal bytes give len = m + 1 - ipshift (ipshift 3 unsplit, 4 split with cratio >= 4)
    for m, split, ids in ((5, 0, {"R_MINLEN3"}), (4, 0, {"R_BELOW3"}), (7, 1, {"R_MINLEN4"}), (6, 1, {"R_BELOW4"})):
        st = _blz_repeat(3000, m, 700 + m, total=20000)
        _compressible_window(st)                                   # a probe window that compresses 4:1 and more
        sc[f"len_m{m}_split{split}"] = (st.array(), 5, split, ids, True)
    for dist, m, ids in ((8191, 40, {"NEAR8190", "LONG_NEAR0"}), (8192, 40, {"FAR8191", "LONG_FAR0"}),
                         (8192, 7, {"FAR5"}), (8192, 8, {"FAR6", "SHORT_FAR"}),
                         (BLZ_MAXFAR - 1, 40, {"MAXFAR_M1"}), (BLZ_MAXFAR, 40, {"MAXFAR"}),
                         (3000, 20, {"LONG_NEAR0"}), (3000, 600, {"LONG_NEAR2", "EXT_MISMATCH"}),
                         (9000, 20, {"LONG_FAR0"}), (9000, 300, {"LONG_FAR1"}), (9000, 600, {"LONG_FAR2"})):
        st = _blz_repeat(dist, m, dist + m, total=max(dist + 2000, 20000))
        _compressible_window(st)
        sc[f"dist{dist}_m{m}"] = (st.array(), 5, 0, ids, True)
    # bit 16 of the packed table: a repeat whose source lies past 65536
    st = Stream(800)
    _periodic_to(st, 66000)
    st.noise(100, ends=64)
    st.repeat(100, 300)
    st.noise(10, ends=100)
    _periodic_to(st, 100000)
    sc["tab17_bit16"] = (st.array(), 5, 1, {"TAB17_HI"}, True)
    # a lower lane with the same bytes supplies the candidate; the round's last lane accepts
    st = Stream(810)
    st.noise(100)
    y = bytes(st.b[10:18])
    st.noise(5, ends=0)
    st.put(y)
    st.noise(31)
    st.put(y)
    st.noise(200)
    st.put(bytes(8000))
    sc["round_lanes"] = (st.array(), 5, 0, {"R_FWD", "R_NONE"}, True)
    # literals, a match, literals, a run to the end: at each capacity up to the fit, one of the five checks refuses
    st = Stream(820)
    st.noise(100)
    st.put(bytes(300))
    st.noise(50)
    st.put(bytes(1050))
    sc["lit_run_lit_run"] = (st.array(), 5, 1, {"LIT_CROSS", "LONG_NEAR1"}, True)
    return sc


BLZ_SC = blz_scenarios()


@pytest.mark.parametrize("name", sorted(BLZ_SC))
def test_blz_scenario_emu(eemu, eorc, name):
    src, clevel, split, want, pack = BLZ_SC[name]
    seen = set()
    for p in (True, False):
        eemu.emu_set_blz_pack(C.c_int(p))
        try:
            for cl in sorted({clevel, *range(1, 10)}):
                for sp in (0, 1):
                    sweep = range(0, len(src) + 1) if len(src) <= 3000 and cl == clevel and sp == split else (65, 66)
                    h0, s = check_blz(eemu, eorc, src, cl, sp, sweep)
                    if cl == clevel and sp == split and p == pack:
                        assert want <= h0, (name, sorted(want - h0))
                    seen |= s
        finally:
            eemu.emu_set_blz_pack(C.c_int(1))
    _BLZ_SEEN.update(seen)


# ------------------------------------------------------------------------------------------------
# the ledgers
# ------------------------------------------------------------------------------------------------
def test_lz4_ledger(eemu, eorc):
    """every LZ4E_H_* id is reached by some scenario (the scenario tests collect them; run alone, this test runs
    them itself)"""
    if set(LH) - _LZ4_SEEN - set(LZ4_UNREACHED):
        for name in sorted(LZ4_SC):
            test_lz4_scenario_emu(eemu, eorc, name)
    assert set(LH) - _LZ4_SEEN == set(LZ4_UNREACHED), sorted(set(LH) - _LZ4_SEEN)


def test_blz_ledger(eemu, eorc):
    if set(BH) - _BLZ_SEEN:
        for name in sorted(BLZ_SC):
            test_blz_scenario_emu(eemu, eorc, name)
    assert set(BH) - _BLZ_SEEN == set(), sorted(set(BH) - _BLZ_SEEN)


# ------------------------------------------------------------------------------------------------
# the reference: the same calls into LZ4_compress_fast / blosclz_compress, pinned
# ------------------------------------------------------------------------------------------------
def _ref_records(lib, lz4_name, blz_name, fits):
    out = []
    for name in sorted(LZ4_SC):
        src, accel = LZ4_SC[name][:2]
        for cap in (lz4_full(len(src)), fits[name] - 1):
            r, o = lz4_call(lib, lz4_name, src, max(cap, 0), accel)
            out.append((name, cap, r, o))
    for name in sorted(BLZ_SC):
        src, clevel, split = BLZ_SC[name][:3]
        for cap in (len(src), fits[name] - 1):
            r, o = blz_call(lib, blz_name, src, max(cap, 0), clevel, split)
            out.append((name, cap, r, o))
    return out


def test_reference_results_pinned(eorc, eref):
    """the oracle's results for every scenario at its own acceleration / clevel, at full capacity and at fit - 1,
    equal LZ4_compress_fast's and blosclz_compress's (live where oracle/_ref is built, else as recorded)"""
    fits = {}
    for name, (src, accel, *_) in LZ4_SC.items():
        fits[name] = _min_cap(lambda c: lz4_call(eorc, "orc_lz4_compress_fast", src, c, accel)[0] > 0, lz4_full(len(src)))
    for name, (src, clevel, split, *_) in BLZ_SC.items():
        f = _min_cap(lambda c: blz_call(eorc, "orc_blosclz_compress", src, c, clevel, split)[0] > 0, len(src))
        fits[name] = 0 if f is None else f
    ours = _ref_records(eorc, "orc_lz4_compress_fast", "orc_blosclz_compress", fits)
    reference = None if eref is None else _ref_records(eref, "LZ4_compress_fast", "blosclz_compress", fits)
    assert_pinned("lz_encode_edges", ours, reference)


# ------------------------------------------------------------------------------------------------
# Blosc chunks of the scenarios
# ------------------------------------------------------------------------------------------------
def chunk_corpus():
    """(name, source, typesize, shuffle, compressor, clevel, blocksize): every scenario as one block of typesize 1
    without shuffle (one stream), and at typesize 2 and 8 with shuffle, each byte repeated typesize times, so that
    every byte-plane stream is the scenario itself.  LZ4 at clevel 10 - acceleration."""
    out = []
    for comp, table in (("lz4", LZ4_SC), ("blosclz", BLZ_SC)):
        for name in sorted(table):
            src = table[name][0]
            clevel = 10 - table[name][1] if comp == "lz4" else max(table[name][1], 1)
            if len(src) < 16:
                continue
            for ts, shuf in ((1, 0), (2, 1), (8, 1)):
                if ts > 1 and len(src) * ts > 400000:
                    continue
                x = np.repeat(src, ts)
                out.append((f"{comp}_{name}_ts{ts}", x, ts, shuf, comp, clevel, len(x)))
    return out


def _chunk(lib, fn, x, ts, shuf, comp, clevel, bs):
    r, d = compress(lib, fn, clevel, shuf, ts, x, len(x) + 16, comp, bs)
    return r, d[:max(r, 0)].copy()


def _pack_source():
    """two blocks of 131072 bytes (one stream each at typesize 1): the packed-table scenario, then the one whose
    rounds pass 192 probes, padded with noise -- every stream long enough for the packed LZ4 table"""
    a = np.concatenate([LZ4_SC["pack_bit16"][0], LZ4_SC["round_it200"][0], LZ4_SC["chains_and_gaps"][0]])
    pad = np.frombuffer(bytes(ew.rnd(262144, 9)), np.uint8)
    return np.concatenate([a, pad[:262144 - len(a)]])


@pytest.mark.parametrize("team", [0, 1])
def test_chunks_emu(eemu, orc, team):
    """every chunk of the corpus through the emulator's chunk path -- LZ4 through encode_kernel as on the GPU
    (team 0) and through the team encoder, BloscLZ with the packed table and without -- equals the oracle's"""
    eemu.emu_set_all_device(0)
    eemu.emu_set_lz4_team(team)
    try:
        for blz_pack in ((1, 0) if team else (1,)):
            eemu.emu_set_blz_pack(blz_pack)
            for name, x, ts, shuf, comp, clevel, bs in chunk_corpus():
                if comp == "blosclz" and blz_pack == 0 and ts > 1:
                    continue
                ra, a = _chunk(orc, "orc_compress_ctx", x, ts, shuf, comp, clevel, bs)
                rb, b = _chunk(eemu, "blosc_compress_ctx", x, ts, shuf, comp, clevel, bs)
                assert ra == rb and np.array_equal(a, b), (name, team, blz_pack, ra, rb)
    finally:
        eemu.emu_set_lz4_team(1)
        eemu.emu_set_blz_pack(1)


def test_pack_chunk_emu(eemu, orc, monkeypatch):
    """BLOSC_B200_LZ4_PACK=1: streams of 65547..131072 bytes take the packed table (PACK) in encode_kernel; the chunk
    equals the oracle's, and bit 16 was read"""
    monkeypatch.setenv("BLOSC_B200_LZ4_PACK", "1")
    eemu.emu_set_all_device(0)
    eemu.emu_set_lz4_team(0)
    try:
        x = _pack_source()
        lhits(eemu)
        for clevel in (9, 5, 1):
            ra, a = _chunk(orc, "orc_compress_ctx", x, 1, 0, "lz4", clevel, 131072)
            rb, b = _chunk(eemu, "blosc_compress_ctx", x, 1, 0, "lz4", clevel, 131072)
            assert ra == rb > 0 and np.array_equal(a, b), (clevel, ra, rb)
            if clevel == 9:
                assert {"TAB_PACK", "PACK_HI"} <= lhits(eemu)
    finally:
        eemu.emu_set_lz4_team(1)


@pytest.mark.gpu
def test_chunks_gpu(pkg, cuda, orc):
    """the corpus through the CUDA library from host buffers and from device buffers of exactly nbytes (typesize 1,
    2 and 8: encode_kernel): the oracle's chunks byte for byte"""
    for name, x, ts, shuf, comp, clevel, bs in chunk_corpus():
        ra, a = _chunk(orc, "orc_compress_ctx", x, ts, shuf, comp, clevel, bs)
        out = np.zeros(len(x) + 16, np.uint8)
        rb = pkg.compress_ctx(clevel, shuf, ts, len(x), x, out, len(x) + 16, comp, bs)
        assert ra == rb and np.array_equal(a, out[:max(rb, 0)]), (name, ra, rb)
        d_x = cuda.from_numpy(x.copy()).cuda()
        d_out = cuda.zeros(len(x) + 16, dtype=cuda.uint8, device="cuda")
        rc = pkg.compress_ctx(clevel, shuf, ts, len(x), d_x, d_out, len(x) + 16, comp, bs)
        assert ra == rc and np.array_equal(a, d_out[:max(rc, 0)].cpu().numpy()), (name, ra, rc)


_FRAME_CHILD = """
import json, sys
import numpy as np, torch
sys.path.insert(0, %r); sys.path.insert(0, %r)
import __graft_entry__ as g
import test_lz_encode_edges as T
pkg = g.load_package()
x = np.concatenate([np.repeat(s, 4) for s in (T._pack_source(), T.LZ4_SC["chains_and_gaps_u32"][0])])
out = {}
for clevel in (9, 5):
    for dev in (0, 1):
        src = torch.from_numpy(x).cuda() if dev else x
        cap = pkg.frame_bound(len(x), 4, 524288)
        fr = torch.zeros(cap, dtype=torch.uint8, device="cuda") if dev else np.zeros(cap, np.uint8)
        fb = pkg.frame_compress(clevel, 1, 4, len(x), src, fr, cap, "lz4", 131072 * 4, 524288)
        f = fr[:fb].cpu().numpy() if dev else fr[:fb]
        chunks = []
        for i in range((len(x) + 524287) // 524288):
            off, clen = pkg.frame_chunk(f, fb, i)
            chunks.append(f[off:off + clen].tobytes().hex())
        out["%%d_%%d" %% (clevel, dev)] = chunks
print(json.dumps(out))
"""


@pytest.mark.gpu
@pytest.mark.parametrize("pack", ["0", "1"])
def test_frame_chunks_gpu(pkg, cuda, orc, pack):
    """typesize 4 through frame_compress, several chunks in flight (encode_kernel, not the team encoder), with and
    without BLOSC_B200_LZ4_PACK=1 (read by the library at each call; a child process keeps it from other tests):
    every chunk equals the oracle's chunk of its slice"""
    code = _FRAME_CHILD % (ROOT, os.path.join(ROOT, "tests"))
    env = dict(os.environ, BLOSC_B200_LZ4_PACK=pack)
    res = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stderr[-3000:]
    got = __import__("json").loads(res.stdout.strip().splitlines()[-1])
    x = np.concatenate([np.repeat(s, 4) for s in (_pack_source(), LZ4_SC["chains_and_gaps_u32"][0])])
    for key, chunks in got.items():
        clevel = int(key.split("_")[0])
        for i, ch in enumerate(chunks):
            piece = x[i * 524288:(i + 1) * 524288].copy()
            r, a = _chunk(orc, "orc_compress_ctx", piece, 4, 1, "lz4", clevel, 131072 * 4)
            assert bytes.fromhex(ch) == a.tobytes(), (key, i, r, len(ch) // 2)

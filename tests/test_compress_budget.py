"""Compression at every destination size near the fit.

The return code of blosc_compress_ctx depends on destsize through two give-up rules of the reference (blosc.c):
  - serial_blosc (nthreads 1, or at most one block, :908-913) hands each split's codec call
    maxout = min(neblock, room left in dest) (:646-651).  A clamped call fails when its stream needs more than that
    room, and a raw split needs the whole neblock (:705-711);
  - the pool (t_blosc) never clamps; it gives up only when the running total passes destsize (:1845-1850).
The library encodes every split at once with maxout = neblock and replays those rules afterwards from each stream's
`need`, the smallest maxout its codec would still have accepted (dev_chunk.cuh scan_place).  A `need` one byte off,
or a split's room counted wrong, turns a chunk into 0 or the other way round while every byte stays right, so no
round trip notices.  These tests look at the return code where it can flip:
  - the oracle against the reference (recorded results), in that window, under both rules;
  - `need` of every exact stream encoder against the oracle's stream encoders (bisection), and hand-built streams
    whose `need - cbytes` gap follows from lz4.c / blosclz.c;
  - the emulated library and the CUDA library against the oracle, with a sentinel past destsize.
"""
import numpy as np
import pytest

from datagen import assert_pinned, ci, compress, decompress, gen, ptr, sz

KINDS = ["bench", "text", "mixed", "i32", "lowent"]
ORC = {"cctx": "orc_compress_ctx", "dctx": "orc_decompress_ctx"}
REF = {"cctx": "blosc_compress_ctx", "dctx": "blosc_decompress_ctx"}
FILL = 0xAA


def _i32(a, o):
    return int.from_bytes(bytes(a[o:o + 4]), "little", signed=True)


# ------------------------------------------------------------------------------------------------ oracle-side geometry
def _splits(chunk):
    """(prefix position, compressed size, length, block, split) of every split of a compressed chunk, in chunk order"""
    flags, ts = int(chunk[2]), int(chunk[3])
    nbytes, bs = _i32(chunk, 4), _i32(chunk, 8)
    out = []
    for b in range((nbytes + bs - 1) // bs):
        bsize = min(bs, nbytes - b * bs)
        ns = ts if not flags & 0x10 and bsize == bs else 1          # blosc.c:628-634
        pos = _i32(chunk, 16 + 4 * b)
        for s in range(ns):
            c = _i32(chunk, pos)
            out.append((pos, c, bsize // ns, b, s))
            pos += 4 + c
    return out


def _split_input(orc, src, chunk, b, s, neblock):
    """the bytes the codec saw for split s of block b: the block, filtered as blosc_c does (blosc.c:607-622)"""
    flags, ts, bs = int(chunk[2]), int(chunk[3]), _i32(chunk, 8)
    blk = np.ascontiguousarray(src[b * bs:(b + 1) * bs])
    if flags & 1 and ts > 1:
        f = np.zeros(len(blk) + 1, np.uint8)
        orc.orc_shuffle(sz(ts), sz(len(blk)), ptr(blk), ptr(f))
        blk = f[:len(blk)]
    elif flags & 4 and len(blk) >= ts:
        f = np.zeros(len(blk) + 1, np.uint8)
        orc.orc_bitshuffle(sz(ts), sz(len(blk)), ptr(blk), ptr(f))
        blk = f[:len(blk)]
    return np.ascontiguousarray(blk[s * neblock:(s + 1) * neblock])


def _orc_stream(orc, comp, clevel, split, x, cap):
    out = np.zeros(cap + 64, np.uint8)
    if comp == "lz4":
        r = orc.orc_lz4_compress_fast(ptr(x), ptr(out), ci(len(x)), ci(cap), ci(10 - clevel))
    else:
        r = orc.orc_blosclz_compress(ci(clevel), ptr(x), ci(len(x)), ptr(out), ci(cap), ci(split))
    return r, out


def _min_cap(accepts, hi):
    """the smallest cap in [0, hi] that `accepts` (monotone), or None"""
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


def _orc_need(orc, comp, clevel, split, x):
    hi = len(x) + len(x) // 255 + 16
    return _min_cap(lambda cap: _orc_stream(orc, comp, clevel, split, x, cap)[0] > 0, hi)


def _window(orc, src, comp, ts, shuf, clevel, bs):
    """The destsizes where the return code can flip: fit-3 ... fit+48, n+15, n+16, and for every split whose room can
    fall below its length there, the sizes where that room crosses the stream's need and its length, each +-1.
    `fit` is the size of the compressed chunk (n + 16 if there is none)."""
    n = len(src)
    fit, chunk = n + 16, None
    for nt in (2, 1):
        r, a = compress(orc, ORC["cctx"], clevel, shuf, ts, src, n + 16, comp, bs, nt)
        if r > 0 and not a[2] & 2:
            fit, chunk = r, a[:r].copy()
            break
    ds = set(range(fit - 3, fit + 49)) | {n + 15, n + 16}
    if chunk is not None:
        split = int(not chunk[2] & 0x10)
        for pos, c, neblock, b, s in _splits(chunk):
            if pos + 4 + neblock < fit - 3:
                continue
            edges = [neblock]
            if c < neblock:
                need = _orc_need(orc, comp, clevel, split, _split_input(orc, src, chunk, b, s, neblock))
                assert need is not None and c <= need, (comp, ts, shuf, clevel, bs, b, s)
                edges.append(need)
            for e in edges:
                ds |= {pos + 4 + e - 1, pos + 4 + e, pos + 4 + e + 1}
    return sorted(d for d in ds if d >= 0), fit


# ------------------------------------------------------------------------------------------------ oracle vs reference
def _configs(comp):
    """every typesize / filter / clevel / forced blocksize for one codec; data kind and size rotate through the cases.
    A forced blocksize of a splitting codec grows to at least 64 KiB (blosc.c:1032-1047), so the larger sizes are what
    give such chunks several blocks; 70001 is one full block plus a leftover."""
    i = 0
    for ts in (1, 2, 3, 4, 8, 16):
        for shuf in (0, 1, 2):
            for clevel in range(10):
                for bs in (100, 1000, 4096):
                    yield ts, shuf, clevel, bs, KINDS[i % len(KINDS)], (3001, 20011, 70001, 3001, 20011, 140001)[(i // len(KINDS)) % 6]
                    i += 1


def _edge_configs():
    """one full block plus a leftover (the pool's nbytes / blocksize <= 1: serial even with nthreads 2), a leftover of
    fewer than 16 bytes (BloscLZ refuses it: stored raw), and all-raw chunks"""
    for comp in ("blosclz", "lz4"):
        for ts, shuf, clevel, bs, kind, n in ((16, 1, 5, 1000, "bench", 1500), (8, 2, 9, 1000, "text", 1999),
                                              (4, 1, 5, 4096, "mixed", 65536 + 20000), (16, 1, 5, 1000, "bench", 5 * 992 + 10),
                                              (16, 0, 9, 1000, "text", 7 * 992 + 15), (2, 1, 5, 4096, "bench", 2 * 65536 + 10),
                                              (16, 0, 5, 1000, "rand", 9000), (2, 1, 5, 1000, "rand", 9000)):
            yield comp, ts, shuf, clevel, bs, kind, n


def _budget_records(comp, nt):
    """nt 1: return code and chunk bytes.  nt 2: return code, cbytes and the decoded buffer -- the reference's block
    order under threads is not deterministic, so its chunk bytes are not compared."""
    def records(orc):
        def run(lib, fn):
            for ts, shuf, clevel, bs, kind, n in _configs(comp):
                src = gen(kind, n, seed=n + ts + clevel)
                ds, _ = _window(orc, src, comp, ts, shuf, clevel, bs)
                for d in ds:
                    case = (n, kind, ts, shuf, clevel, bs, d)
                    r, a = compress(lib, fn["cctx"], clevel, shuf, ts, src, d, comp, bs, nt)
                    assert (a[d:] == FILL).all(), case
                    if nt == 1:
                        yield case, r, a[:max(r, 0)]
                    elif r <= 0:
                        yield case, r
                    else:
                        k, o = decompress(lib, fn["dctx"], a, n)
                        yield case, r, _i32(a, 12), k, o[:n]
        return run
    return records


def _edge_records(orc):
    def run(lib, fn):
        for comp, ts, shuf, clevel, bs, kind, n in _edge_configs():
            src = gen(kind, n, seed=n)
            ds, _ = _window(orc, src, comp, ts, shuf, clevel, bs)
            for d in ds:
                for nt in (1, 2):
                    case = (comp, n, kind, ts, shuf, clevel, bs, d, nt)
                    r, a = compress(lib, fn["cctx"], clevel, shuf, ts, src, d, comp, bs, nt)
                    assert (a[d:] == FILL).all(), case
                    serial = nt == 1 or n // _i32(a, 8) <= 1         # blosc.c:910: serial_blosc even with threads
                    yield (case, r, a[:max(r, 0)]) if serial else (case, r, _i32(a, 12) if r > 0 else 0)
    return run


@pytest.mark.parametrize("comp", ["blosclz", "lz4"])
@pytest.mark.parametrize("nt", [1, 2])
def test_oracle_budget_window(orc, ref_if_built, comp, nt):
    """The oracle's serial (nt 1) and pool (nt 2) give-up rules against the reference at every destsize of the window"""
    run = _budget_records(comp, nt)(orc)
    assert_pinned(f"budget_window[{comp}-nt{nt}]", run(orc, ORC), None if ref_if_built is None else run(ref_if_built, REF))


def test_oracle_budget_edges(orc, ref_if_built):
    run = _edge_records(orc)
    assert_pinned("budget_edges", run(orc, ORC), None if ref_if_built is None else run(ref_if_built, REF))


def test_oracle_rules_differ_in_the_window(orc):
    """The two rules do give different answers: on bench data, typesize 8, shuffle, clevel 1, blocksize 4096, the serial
    rule gives up at destsize == fit, where the pool's chunk fits"""
    n = 300001
    src = gen("bench", n)
    fit, a = compress(orc, ORC["cctx"], 1, 1, 8, src, n + 16, "blosclz", 4096, 2)
    assert 0 < fit < n and not a[2] & 2
    assert compress(orc, ORC["cctx"], 1, 1, 8, src, fit, "blosclz", 4096, 2)[0] == fit
    assert compress(orc, ORC["cctx"], 1, 1, 8, src, fit, "blosclz", 4096, 1)[0] == 0
    assert compress(orc, ORC["cctx"], 1, 1, 8, src, fit - 1, "blosclz", 4096, 2)[0] == 0
    # the pool path validates nthreads, the serial one does not (blosc.c:910, :1975-1986)
    assert compress(orc, ORC["cctx"], 5, 1, 8, src, n + 16, "lz4", 4096, 0)[0] == -1
    assert compress(orc, ORC["cctx"], 5, 1, 8, src, n + 16, "lz4", 4096, 257)[0] == -1
    assert compress(orc, ORC["cctx"], 5, 1, 8, src[:6000], 6016, "lz4", 4096, 0)[0] > 0


# ------------------------------------------------------------------------------------------------ stream level, emulator
def _emu_stream(emu, enc, x, cap):
    out = np.full(cap + 64, FILL, np.uint8)
    r = enc(x, out, cap)
    assert (out[max(cap, 0):] == FILL).all(), "stream encoder wrote past its capacity"
    return r, out, emu.emu_last_need()


def _check_need(emu, orc, enc, comp, clevel, split, x, caps=()):
    """`need` of the encoder `enc` equals the oracle's smallest accepted capacity; at cap = need the bytes are the
    oracle's, at need - 1 the stream is refused; at every cap of `caps`, the oracle's verdict.  Returns (need, cbytes)."""
    n = len(x)
    r, out, need = _emu_stream(emu, enc, x, n)
    ro, _ = _orc_stream(orc, comp, clevel, split, x, n)
    assert r == ro, (n, r, ro)
    if r <= 0:
        return None, r
    want = _orc_need(orc, comp, clevel, split, x)
    assert need == want, (n, need, want, r)
    for cap in sorted({need, need - 1, *caps}):
        if cap < 0:
            continue
        rc, oc, _ = _emu_stream(emu, enc, x, cap)
        ro, oo = _orc_stream(orc, comp, clevel, split, x, cap)
        assert rc == ro == (r if cap >= need else 0), (n, cap, need, rc, ro)
        assert (oc[:max(rc, 0)] == oo[:max(ro, 0)]).all(), (n, cap)
    return need, r


def _lz4(emu, accel):
    return lambda x, out, cap: emu.emu_lz4_encode(ptr(x), ci(len(x)), ptr(out), ci(cap), ci(accel))


def _lz4_team(emu, accel, walker):
    return lambda x, out, cap: emu.emu_lz4_encode_team(ptr(x), ci(len(x)), ptr(out), ci(cap), ci(accel), ci(walker))


def _blz(emu, clevel, split):
    return lambda x, out, cap: emu.emu_blz_encode(ci(clevel), ptr(x), ci(len(x)), ptr(out), ci(cap), ci(split))


STREAM_KINDS = ["bench", "mixed", "lowent", "i32", "zeros", "text", "rand"]


@pytest.mark.parametrize("path", ["u16", "u32", "pack", "team0", "team1", "team2", "team3"])
def test_lz4_stream_need(emu, orc, path):
    """byU16 (n < 65547) and byU32 warp encoders, the packed 17-bit table, the team encoder at each walker warp"""
    sizes = {"u16": [16, 300, 4096, 40000], "u32": [65547, 100000, 140000], "pack": [65547, 100000, 131072]}.get(path, [5000, 70000])
    emu.emu_set_lz4_pack(int(path == "pack"))
    try:
        for i, n in enumerate(sizes):
            for accel in (1, 5):
                kind = STREAM_KINDS[(i * 2 + accel) % len(STREAM_KINDS)]
                x = gen(kind, n, seed=n + accel)
                enc = _lz4_team(emu, accel, int(path[4])) if path.startswith("team") else _lz4(emu, accel)
                need, r = _check_need(emu, orc, enc, "lz4", 10 - accel, 0, x)
                assert need is None or need == r          # see test_lz4_need_gap_is_zero
    finally:
        emu.emu_set_lz4_pack(0)


@pytest.mark.parametrize("table", ["pack", "plain"])
@pytest.mark.parametrize("clevel", range(1, 10))
def test_blosclz_stream_need(emu, orc, table, clevel):
    """BloscLZ with the packed 17-bit table and with the plain 64 KiB table (the only one for streams over 128 KiB)"""
    emu.emu_set_blz_pack(int(table == "pack"))
    try:
        sizes = [16, 17, 100, 5000, 40000] if table == "pack" else [5000, 140000]
        for i, n in enumerate(sizes):
            for split in (0, 1):
                kind = STREAM_KINDS[(i + clevel + split) % 5]          # the kinds BloscLZ's probe lets through
                x = gen(kind, n, seed=n + clevel)
                need, r = _check_need(emu, orc, _blz(emu, clevel, split), "blosclz", clevel, split, x)
                assert need is None or need == max(66, r + 1), (n, need, r)
    finally:
        emu.emu_set_blz_pack(1)


def _rnd(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _cat(*parts):
    return np.ascontiguousarray(np.concatenate([np.asarray(p, np.uint8) for p in parts]))


def test_lz4_need_gap_is_zero(emu, orc):
    """Hand-built LZ4 streams that make each output check of lz4.c binding.  Every match ends at least LASTLITERALS
    before the end (matchlimit, lz4.c:1183), so the last-literals check (lz4.c:1305-1306, the bytes of the last run
    exactly) is never below any other, and ties with the literal check (op + lit + 2 + 1 + LASTLITERALS + lit / 255,
    :1114-1115) and the match check (op + 1 + LASTLITERALS + (mc + 240) / 255, :1187-1188) when the last run is
    LASTLITERALS long: need - cbytes is 0."""
    cases = []
    for lit in (1, 14, 15, 16, 254, 255, 256, 269, 270, 509, 510):      # a literal run before a run of zeros
        cases.append(_cat(_rnd(lit, lit) | 1, np.zeros(300, np.uint8)))
    for m in (8, 18, 19, 20, 270, 273, 274, 530):                        # a match of each length-code size
        cases.append(_cat(_rnd(6, m) | 1, np.zeros(m, np.uint8), _rnd(5, m + 1) | 1))
    for last in (5, 14, 15, 16, 269, 270, 271, 600):                     # last literals of < 15, >= 15 and >= 270 bytes
        cases.append(_cat(np.zeros(200, np.uint8), _rnd(last, last) | 1))
    cases.append(_cat(*([_rnd(9, 7) | 1, np.zeros(30, np.uint8)] * 40)))  # sequence after sequence
    fits = 0
    for accel in (1, 5):
        for x in cases:
            for enc in (_lz4(emu, accel), _lz4_team(emu, accel, 0)):
                n = len(x)
                need, r = _check_need(emu, orc, enc, "lz4", 10 - accel, 0, x, caps=range(max(0, n // 2), n + 2, 7))
                assert need is None or need == r, (len(x), need, r)
                fits += need is not None
    assert fits >= 4 * len(cases) - 8         # all but the shortest match cases compress


def test_blosclz_need_gap(emu, orc):
    """Hand-built BloscLZ streams.  A stream always ends in literals (a match stops short of ip_bound by ipshift,
    blosclz.c:530), so the binding check is the last literal's op + 2 > op_limit (:591): need = cbytes + 1, also when
    that literal completes a run of 32 and the control byte it opened is taken back by `op--` (:600-604) -- unless the
    maxout < 66 floor (:473-475) is higher."""
    cases = [(np.zeros(n, np.uint8), "floor") for n in (16, 17, 40, 100)]                        # cbytes < 65
    cases += [(_cat(np.zeros(1000, np.uint8), _rnd(k, k) | 1), "tail") for k in range(28, 72, 3)]   # run of 32 at the end
    cases += [(_cat(np.zeros(255 * k + 40, np.uint8), _rnd(20, k) | 1), "long") for k in (1, 2, 5)]  # MATCH_LONG, 255s
    far = _rnd(300, 9) | 1                                                                         # matches past 8191
    filler = (np.arange(9000) // 7 % 200).astype(np.uint8) + 50
    cases += [(_cat(far, filler, far, filler[:600], _rnd(20, 3) | 1), "far"), (_cat(far, filler, far[:40]), "far")]
    cases += [(_cat(*([_rnd(6, 5) | 1, np.zeros(12, np.uint8)] * 60)), "ctrl")]                   # match, control byte, literal
    for x, what in cases:
        for clevel, split in ((1, 0), (5, 1), (9, 0), (9, 1)):
            n = len(x)
            need, r = _check_need(emu, orc, _blz(emu, clevel, split), "blosclz", clevel, split, x,
                                  caps=[65, 66, 67, *range(max(0, n // 3), n + 2, 11 if n < 2000 else n // 40)])
            if need is not None:
                assert need == max(66, r + 1), (what, n, clevel, split, need, r)
                if what == "floor":
                    assert r < 65 and need == 66


# ------------------------------------------------------------------------------------------------ chunk level
CHUNK_CONFIGS = [  # comp, ts, shuf, clevel, bs, kind, n
    ("lz4", 4, 1, 5, 4096, "bench", 140001),       # typesize 4 LZ4: the team encoder; 64 KiB blocks of 4 splits
    ("lz4", 2, 1, 9, 4096, "i32", 140001),         # typesize 2 and 8: the warp encoder
    ("lz4", 8, 1, 1, 4096, "bench", 140001),
    ("lz4", 8, 2, 5, 1000, "mixed", 20011),        # 1000 / 8 < 128: unsplit 1000-byte blocks
    ("lz4", 16, 1, 3, 1000, "i32", 20000),
    ("blosclz", 8, 1, 1, 4096, "bench", 140001),
    ("blosclz", 4, 2, 5, 1000, "text", 9000),      # a single block
    ("blosclz", 2, 1, 9, 100, "mixed", 3001),      # 128-byte blocks
    ("blosclz", 16, 1, 7, 1000, "i32", 20000),
    ("blosclz", 16, 1, 5, 1000, "bench", 5 * 992 + 10),  # leftover < 16 bytes: stored raw
    ("blosclz", 16, 1, 5, 1000, "bench", 1500),    # one block + leftover: serial under nt 2
    ("lz4", 8, 1, 5, 1000, "rand", 5000),          # all raw
]
BIG_BLZ = ("blosclz", 1, 0, 9, 200000, "text", 400003)    # BloscLZ streams over 128 KiB: the plain 64 KiB table


def _chunk_check(lib_compress, orc, cfg, ds, what):
    comp, ts, shuf, clevel, bs, kind, n = cfg
    src = gen(kind, n, seed=n)
    for d in ds:
        for nt in (1, 2):
            ra, a = compress(orc, ORC["cctx"], clevel, shuf, ts, src, d, comp, bs, nt)
            rb, b = lib_compress(clevel, shuf, ts, src, d, comp, bs, nt)
            assert ra == rb, (what, cfg, d, nt, ra, rb)
            if ra > 0:
                assert (a[:ra] == b[:ra]).all(), (what, cfg, d, nt)
            assert (b[d:] == FILL).all(), ("wrote at or past destsize", what, cfg, d, nt)


def _big_window(orc, cfg):
    """a few sizes of the window (the streams are long, so every size is a full encode)"""
    comp, ts, shuf, clevel, bs, kind, n = cfg
    ds, fit = _window(orc, gen(kind, n, seed=n), comp, ts, shuf, clevel, bs)
    return sorted(set(ds[::9]) | {fit - 1, fit, fit + 1, n + 15, n + 16} | {d for d in ds if d > fit + 48})


def _emu_sizes(ds, fit, n):
    """the emulator is slow: every size within 4 of the fit and every split crossing outside fit-3 ... fit+48, a
    sample of the rest"""
    return sorted({d for d in ds if abs(d - fit) <= 4 or not fit - 3 <= d <= fit + 48} | set(ds[::6]) | {n + 15, n + 16})


@pytest.mark.parametrize("cfg", CHUNK_CONFIGS, ids=lambda c: "-".join(map(str, c)))
def test_emu_library_budget_window(emu, orc, cfg):
    comp, ts, shuf, clevel, bs, kind, n = cfg
    ds, fit = _window(orc, gen(kind, n, seed=n), comp, ts, shuf, clevel, bs)
    ds = _emu_sizes(ds, fit, n)
    teams = (1, 0) if comp == "lz4" and ts == 4 else (1,)      # the warp encoder as well where the GPU picks the team
    for team in teams:
        emu.emu_set_lz4_team(team)
        try:
            _chunk_check(lambda *a: compress(emu, "blosc_compress_ctx", *a), orc, cfg, ds, f"emu team={team}")
        finally:
            emu.emu_set_lz4_team(1)


def test_emu_library_budget_big_streams(emu, orc):
    _chunk_check(lambda *a: compress(emu, "blosc_compress_ctx", *a), orc, BIG_BLZ, _big_window(orc, BIG_BLZ), "emu big")


def _many_blocks_sizes(orc, comp, clevel, src):
    n = len(src)
    fit, _ = compress(orc, ORC["cctx"], clevel, 1, 4, src, n + 16, comp, 128, 2)
    assert 0 < fit < n
    return fit, [fit - 1, fit, fit + 1, fit + 3, fit + 40, fit + 140]


def _emu_many_sizes(fit):
    return [fit, fit + 3]            # fit - 1 and n + 16: test_emu_kernels.py::test_block_scan_of_more_than_65536_blocks


def test_emu_library_budget_many_blocks(emu, orc):
    """More than 65536 blocks: the scan runs in its own scan_kernel launch"""
    n = 128 * 65536 + 4100
    cfg = ("blosclz", 4, 1, 1, 128, "bench", n)
    fit, _ = _many_blocks_sizes(orc, "blosclz", 1, gen("bench", n, seed=n))
    ds = _emu_many_sizes(fit)
    _chunk_check(lambda *a: compress(emu, "blosc_compress_ctx", *a), orc, cfg, ds, "emu many blocks")


OPT_IN = [("snappy", "BLOSC_B200_SNAPPY", "1"), ("zlib", "BLOSC_B200_ZLIB", "1"), ("zstd", "BLOSC_B200_ZSTD", "1"),
          ("lz4", "BLOSC_B200_PARSE", "fast"), ("lz4hc", None, None)]


def _opt_in_check(lib_compress, lib_decompress, comp, cfgs):
    """Codecs whose bytes are not the reference's have need == cbytes: below one threshold the result is 0, at or above
    it the same chunk, which decodes; nothing is written past destsize.  (Serial snappy is the exception: blosc_c asks
    for snappy_max_compressed_length of room, more than the split, and stores a split raw where that room is short
    (blosc.c:640-651, :705-711), so above its threshold the chunk may still change -- it must still decode.)"""
    for ts, shuf, clevel, bs, kind, n in cfgs:
        src = gen(kind, n, seed=n)
        for nt in (1, 2):
            fit, ref_chunk = lib_compress(clevel, shuf, ts, src, n + 16, comp, bs, nt)
            assert fit > 0, (comp, n, nt)
            if ref_chunk[2] & 2:
                continue                     # stored: nothing to sweep
            ref_chunk = ref_chunk[:fit].copy()
            thr, same = None, not (comp == "snappy" and (nt == 1 or n // _i32(ref_chunk, 8) <= 1))   # blosc.c:910
            for d in sorted(set(range(fit - 4, fit + 12)) | {n + 15}):
                if d > n + 15 or d < 16:
                    continue
                r, a = lib_compress(clevel, shuf, ts, src, d, comp, bs, nt)
                assert (a[d:] == FILL).all(), (comp, n, nt, d)
                if r == 0:
                    assert thr is None, (comp, n, nt, d, "0 above the threshold")
                    continue
                thr = d if thr is None else thr
                assert not same or (r == fit and (a[:r] == ref_chunk).all()), (comp, n, nt, d, r, fit)
                k, o = lib_decompress(a, n)
                assert k == n and (o[:n] == src).all(), (comp, n, nt, d)
            assert thr == fit or not same and thr is not None, (comp, n, nt, thr, fit)


OPT_IN_CFGS = [(4, 1, 5, 4096, "bench", 20011), (1, 0, 9, 1000, "text", 9000), (8, 2, 3, 0, "mixed", 30000)]


@pytest.mark.parametrize("comp,var,val", OPT_IN, ids=[c[0] + ("-" + c[2] if c[2] == "fast" else "") for c in OPT_IN])
def test_emu_library_budget_opt_in_codecs(emu, comp, var, val, monkeypatch):
    if var:
        monkeypatch.setenv(var, val)
    _opt_in_check(lambda *a: compress(emu, "blosc_compress_ctx", *a), lambda c, n: decompress(emu, "blosc_decompress_ctx", c, n),
                  comp, OPT_IN_CFGS)


# ------------------------------------------------------------------------------------------------ chunk level, GPU
def _gpu_compress_into(pkg, cuda, device):
    def run(clevel, shuf, ts, src, destsize, comp, bs=0, nt=1):
        if not device:
            dest = np.full(destsize + 64, FILL, np.uint8)
            r = pkg.compress_ctx(clevel, shuf, ts, len(src), src, dest, destsize, comp, bs, nt)
            return r, dest
        torch = cuda
        dest = torch.full((destsize + 64,), FILL, dtype=torch.uint8, device="cuda")
        r = pkg.compress_ctx(clevel, shuf, ts, len(src), torch.from_numpy(src).cuda(), dest, destsize, comp, bs, nt)
        return r, dest.cpu().numpy()
    return run


def _gpu_decompress(pkg):
    def run(chunk, n):
        dest = np.zeros(n + 64, np.uint8)
        return pkg.decompress_ctx(np.ascontiguousarray(chunk), dest, n), dest
    return run


@pytest.mark.gpu
@pytest.mark.parametrize("device", [0, 1], ids=["host-dest", "device-dest"])
def test_gpu_budget_window(pkg, orc, cuda, device):
    for cfg in CHUNK_CONFIGS:
        comp, ts, shuf, clevel, bs, kind, n = cfg
        ds, _ = _window(orc, gen(kind, n, seed=n), comp, ts, shuf, clevel, bs)
        _chunk_check(_gpu_compress_into(pkg, cuda, device), orc, cfg, ds, f"gpu device={device}")
    _chunk_check(_gpu_compress_into(pkg, cuda, device), orc, BIG_BLZ, _big_window(orc, BIG_BLZ), f"gpu big device={device}")


@pytest.mark.gpu
def test_gpu_budget_many_blocks(pkg, orc, cuda):
    n = 128 * 65536 + 4100
    src = gen("bench", n, seed=n)
    for comp, clevel in (("blosclz", 1), ("lz4", 5)):
        _, ds = _many_blocks_sizes(orc, comp, clevel, src)
        for device in (0, 1):
            _chunk_check(_gpu_compress_into(pkg, cuda, device), orc, (comp, 4, 1, clevel, 128, "bench", n), ds,
                         f"gpu many blocks device={device}")


@pytest.mark.gpu
@pytest.mark.parametrize("comp,var,val", OPT_IN, ids=[c[0] + ("-" + c[2] if c[2] == "fast" else "") for c in OPT_IN])
def test_gpu_budget_opt_in_codecs(pkg, cuda, comp, var, val, monkeypatch):
    if var:
        monkeypatch.setenv(var, val)
    for device in (0, 1):
        _opt_in_check(_gpu_compress_into(pkg, cuda, device), _gpu_decompress(pkg), comp, OPT_IN_CFGS)

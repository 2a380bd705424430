"""The LZ4 team encoder (dev_lz4.cuh, team mode) in the SIMT emulator: a walker and three preparers must give
LZ4_compress_fast's bytes whatever the preparers' timing.  Each stream runs once per walker warp (0..3) and is
compared with the oracle at the same acceleration and capacity.  The emulator's branch counters
(emu_lz4t_counters, totals since the library was loaded: the tests take differences) show that the stale-verdict re-probe, the chain start on prepared tiles and the re-base of
the preparers were all reached."""
import ctypes as C

import numpy as np
import pytest

from datagen import bench_words, ci, compress, ptr

U16_MAX = 65536 + 12 - 1          # shorter streams use the byU16 table (lz4.c:710,1389)
# emu_lz4t_counters: chains, chained sequences, stale verdicts, then LZ4T_LONG, 270+ match, re-base,
# chain start on prepared tiles (dev_lz4.cuh, g_dbg_lz4t_x[0..3])
CHAINS, SEQS, STALE, LONG, HUGE, REBASE, RESUME = range(7)
_seen = np.zeros(7, np.int64)


def counters(emu):
    """what the counters gained since the previous call"""
    global _seen
    c = (C.c_longlong * 7)()
    emu.emu_lz4t_counters(c)
    now = np.array(c[:], np.int64)
    d, _seen = now - _seen, now
    return d


def hash_u32(b, p):
    """lz4.c LZ4_hash5 (byU32 table, 4096 entries) of the five bytes at p"""
    seq = int.from_bytes(bytes(b[p:p + 5]), "little")
    return (((seq << 24) * 889523592379) & (2 ** 64 - 1)) >> 52


def hash_u16(b, p):
    """lz4.c LZ4_hash4 (byU16 table, 8192 entries) of the four bytes at p"""
    return ((int.from_bytes(bytes(b[p:p + 4]), "little") * 2654435761) & 0xffffffff) >> 19


def chains_and_gaps(n, seed):
    """Runs of chained matches separated by incompressible gaps of 40 .. 1500 bytes (chain starts inside, at the
    edge of and past the preparers' run-ahead), a few repeats of 300+ bytes and a repeat that ends 20 bytes
    before the end of the stream"""
    rng = np.random.default_rng(seed)
    out = bytearray(rng.integers(0, 256, 600, dtype=np.uint8).tobytes())
    while len(out) < n - 400:
        kind = rng.integers(0, 8)
        if kind == 0:                                   # long repeat
            src = int(rng.integers(0, len(out) - 350))
            out += out[src:src + int(rng.integers(300, 700))]
        elif kind <= 2:                                 # gap
            out += rng.integers(0, 256, int(rng.choice([40, 200, 260, 290, 400, 1500])), dtype=np.uint8).tobytes()
        else:                                           # chain: a copy from a few hundred bytes back with a byte changed every 8..24
            src = len(out) - int(rng.integers(64, 2000))
            piece = bytearray(out[max(src, 0):max(src, 0) + int(rng.integers(64, 600))])
            k = 0
            while k < len(piece):
                k += int(rng.integers(8, 24))
                if k < len(piece):
                    piece[k] ^= 0x5a
            out += piece
    tail = n - len(out)
    src = len(out) - 3000
    out += out[src:src + tail - 20] + rng.integers(0, 256, 20, dtype=np.uint8).tobytes()
    return np.frombuffer(bytes(out[:n]), np.uint8).copy()


def colliding(n, u16, seed):
    """chains_and_gaps data in which more than 50 pairs of different sequences 64 .. 160 bytes (2 .. 5 tiles) apart
    share a hash: the table entry a preparer read for the later one can be overwritten by the walker's store of
    the earlier one before the walker reaches it"""
    hf = hash_u16 if u16 else hash_u32
    base = chains_and_gaps(n, seed)
    by_hash = {}
    for p in range(0, n - 8):
        by_hash.setdefault(hf(base, p), []).append(p)
    pairs = []
    for ps in by_hash.values():
        for a, b in zip(ps, ps[1:]):
            if 64 <= b - a <= 160 and bytes(base[a:a + 4]) != bytes(base[b:b + 4]):
                pairs.append((a, b))
    assert len(pairs) > 50                              # the data has the collisions the test is about
    return base


def check(emu, orc, src, accel, cap=None, walkers=range(4)):
    n = len(src)
    cap = n if cap is None else cap
    a = np.zeros(cap + 64, np.uint8)
    ra = orc.orc_lz4_compress_fast(ptr(src), ptr(a), ci(n), ci(cap), ci(accel))
    total = np.zeros(7, np.int64)
    for w in walkers:
        b = np.zeros(cap + 64, np.uint8)
        rb = emu.emu_lz4_encode_team(ptr(src), ci(n), ptr(b), ci(cap), ci(accel), ci(w))
        assert ra == rb, (n, accel, cap, w, ra, rb)
        if ra > 0:
            assert (a[:ra] == b[:ra]).all(), (n, accel, cap, w)
            assert (b[ra:] == 0).all()
        total += counters(emu)
    return ra, total


@pytest.fixture(scope="module")
def team(emu):
    emu.emu_lz4_encode_team.restype = C.c_int
    counters(emu)                                       # start counting from here
    return emu


@pytest.mark.parametrize("n", [40000, U16_MAX - 1, U16_MAX, 100000, 131072])
def test_team_chains_and_gaps(team, orc, n):
    src = chains_and_gaps(n, seed=n)
    for accel in (5, 1):
        ra, c = check(team, orc, src, accel)
        assert ra > 0
        assert c[SEQS] > 0 and c[STALE] > 0 and c[RESUME] > 0 and c[REBASE] > 0 and c[LONG] > 0 and c[HUGE] > 0, c


@pytest.mark.parametrize("u16", [True, False])
def test_team_colliding_hashes(team, orc, u16):
    n = 50000 if u16 else 120000
    src = colliding(n, u16, seed=7)
    _, c = check(team, orc, src, 5)
    assert c[STALE] > 0, c


@pytest.mark.parametrize("n", [30000, 131072])
def test_team_byte_planes(team, orc, n):
    """The cfg 2 planes of one block: byte-plane k of 32-bit words"""
    w = bench_words(4 * n)
    for k in range(4):
        src = np.ascontiguousarray(w.view(np.uint8).reshape(-1, 4)[:, k])
        ra, c = check(team, orc, src, 5, walkers=(k,))
        assert ra != 0 or k == 0


@pytest.mark.parametrize("n", [20000, 100000])
def test_team_limited_output(team, orc, n):
    src = chains_and_gaps(n, seed=3 * n)
    full, _ = check(team, orc, src, 5, walkers=(1,))
    assert full > 0
    for cap in (full - 1, full, full // 2):
        ra, _ = check(team, orc, src, 5, cap=cap, walkers=(0, 2))
        assert (ra > 0) == (cap >= full)


def test_team_match_ends_near_stream_end(team, orc):
    """Streams whose last match ends 0 .. 70 bytes before the end: the chain's `ip + 64 > n` exits"""
    rng = np.random.default_rng(11)
    body = chains_and_gaps(20000, seed=11)
    for tail in list(range(0, 12)) + [12, 13, 20, 40, 63, 64, 65, 70]:
        src = np.concatenate([body, body[-3000:-3000 + 500], rng.integers(0, 256, tail, dtype=np.uint8)])
        check(team, orc, src, 5, walkers=(3,))


def test_team_several_streams_per_cta(team, orc):
    """The compress path runs at most 3 team CTAs, so every team goes through several streams (stream switches
    and the final QUIT); chunks must be the oracle's"""
    team.emu_set_all_device(0)
    for n, ts, bs in ((1 << 20, 4, 0), (300000, 4, 65536), (200000, 2, 0), (260000, 8, 0)):
        src = bench_words(n).view(np.uint8)[:n].copy()
        ra, a = compress(orc, "orc_compress_ctx", 5, 1, ts, src, n + 16, "lz4", bs)
        rb, b = compress(team, "blosc_compress_ctx", 5, 1, ts, src, n + 16, "lz4", bs)
        assert ra == rb and ra > 0 and (a[:ra] == b[:ra]).all(), (n, ts, bs, ra, rb)
    c = counters(team)
    assert c[CHAINS] > 0 and c[SEQS] > 0, c

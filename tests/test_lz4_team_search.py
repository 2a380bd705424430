"""The LZ4 team encoder's search after a chained miss (dev_lz4.cuh, lz4t_search): the walker takes the first four
probes of the search from the prepared verdicts and parks a literal-free searched sequence like a chained one.  Streams
that reach each branch -- a hit at probe 0..3, a stale verdict at a probe, four misses, a hit with literals, a catch-up
longer than the verdict's 7 bytes, an LZ4T_LONG match and a 270+ match found by the search -- must give
LZ4_compress_fast's bytes and return value at every acceleration, table flavour, walker warp and capacity.  The
emulator's branch counters (emu_lz4t_search_counters of tests/emu/lz4t_search_stage.cpp, totals since that library
was loaded) show that each branch ran.
On the GPU the same streams, interleaved as the byte-planes of a typesize-4 chunk, go through encode_team_kernel."""
import ctypes as C
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from datagen import bench_words, ci, compress, ptr
from test_lz4_team import U16_MAX, chains_and_gaps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# emu_lz4t_search_counters (dev_lz4.cuh, LZ4T_S_*)
HIT0, HIT1, HIT2, HIT3, STALE, MISS4, LIT, CAPPED, LONG, HUGE = range(10)
NAMES = ("hit at probe 0", "hit at probe 1", "hit at probe 2", "hit at probe 3", "stale verdict", "four misses",
         "literals", "catch-up past 7", "LZ4T_LONG", "270+ match")
_total = np.zeros(10, np.int64)


def search_counters(emu):
    c = (C.c_longlong * 10)()
    assert emu.emu_lz4t_search_counters(c) == 10
    return np.array(c[:], np.int64)


def edited_repeats(n, seed, period, alphabet, width):
    """A block of `period` bytes over `alphabet` letters, repeated with 1..5 runs of up to `width` bytes rewritten
    per copy: every rewrite breaks the chain that follows the previous copy, and the search finds that copy or an
    older one a few bytes later, at a catch-up length set by how often the small alphabet repeats a byte"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, alphabet, period, dtype=np.uint8)
    parts, size = [rng.integers(0, 256, 300, dtype=np.uint8)], 300
    while size < n:
        b = base.copy()
        for _ in range(int(rng.integers(1, 6))):
            x, w = int(rng.integers(0, period - width)), int(rng.integers(1, width + 1))
            b[x:x + w] = rng.integers(0, alphabet, w, dtype=np.uint8)
        parts.append(b)
        size += period
    return np.concatenate(parts)[:n].copy()


def plane(n, k):
    """byte-plane k of the bench.c words (plane 1 is the hard one of cfg 2)"""
    return np.ascontiguousarray(bench_words(4 * n).view(np.uint8).reshape(-1, 4)[:, k])


STREAMS = {
    "plane1": lambda n: plane(n, 1),
    "chains": lambda n: chains_and_gaps(n, seed=n + 1),
    "alpha4": lambda n: edited_repeats(n, 1, 200, 4, 3),
    "alpha16": lambda n: edited_repeats(n, 2, 700, 16, 8),
    "bytes": lambda n: edited_repeats(n, 3, 1500, 256, 1),
}


def check(emu, orc, src, accel, walker, cap=None):
    n = len(src)
    cap = n if cap is None else cap
    a = np.zeros(cap + 64, np.uint8)
    b = np.zeros(cap + 64, np.uint8)
    ra = orc.orc_lz4_compress_fast(ptr(src), ptr(a), ci(n), ci(cap), ci(accel))
    before = search_counters(emu)
    rb = emu.emu_lz4_encode_team(ptr(src), ci(n), ptr(b), ci(cap), ci(accel), ci(walker))
    _total[:] += search_counters(emu) - before
    assert ra == rb, (n, accel, cap, walker, ra, rb)
    if ra > 0:
        assert (a[:ra] == b[:ra]).all(), (n, accel, cap, walker)
        assert (b[ra:] == 0).all()
    return ra


@pytest.fixture(scope="module")
def team(tmp_path_factory):
    """the emulated library with the search's branch counters of tests/emu/lz4t_search_stage.cpp (which includes
    backend_emu.cpp whole), built into a temporary directory"""
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("lz4t_search_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "c-blosc_b200", "csrc", "blosc_b200.c"), "-o",
                    str(d / "host.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "lz4t_search_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    path = str(d / "liblz4t_search_stage.so")
    subprocess.run(["g++", "-shared", "-o", path, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    lib = C.CDLL(path)
    lib.emu_lz4_encode_team.restype = C.c_int
    lib.emu_lz4t_search_counters.restype = C.c_int
    return lib


SIZES = [40000, U16_MAX, 100000]                       # both table flavours, and the boundary between them


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("name", sorted(STREAMS))
def test_search_streams(team, orc, name, n):
    """every stream at accelerations 1, 5 and 9 (the walker warp rotates over streams, sizes and accelerations, so
    each stream and size meets three of the four and every accelerations all four), then at accel 5 with exactly
    the room it needs, one byte less and half of it"""
    src = STREAMS[name](n)
    w0 = sorted(STREAMS).index(name) + SIZES.index(n)
    for i, accel in enumerate((1, 5, 9)):
        full = check(team, orc, src, accel, (w0 + i) % 4)
        assert full > 0
        if accel == 5:
            for k, cap in enumerate((full, full - 1, full // 2)):
                assert check(team, orc, src, accel, (w0 + k + 1) % 4, cap) == (full if cap == full else 0)


@pytest.mark.parametrize("accel", [1, 5, 6, 9])
def test_search_breaks_near_the_end(team, orc, accel):
    """A chain that breaks 64 .. 100 bytes before the end: the search's probes and the chain's `ip + 64 > n` exit
    meet the end of the stream; accel 6 puts probe 2 exactly 8 bytes past the anchor"""
    rng = np.random.default_rng(accel)
    body = edited_repeats(20000, 4, 300, 4, 2)
    for tail in (40, 52, 60, 64, 70, 80, 100):
        src = np.concatenate([body, body[-600:-600 + tail], rng.integers(0, 4, 12, dtype=np.uint8)])
        check(team, orc, src, accel, tail % 4)


def test_search_catch_up_at_the_start(team, orc):
    """Repeats of the first bytes of the stream: the catch-up runs into position 0 (snap < 8)"""
    rng = np.random.default_rng(9)
    head = rng.integers(0, 4, 40, dtype=np.uint8)
    parts = [head]
    for k in range(400):
        h = head.copy()
        h[int(rng.integers(0, 12))] ^= 1
        parts += [h, rng.integers(0, 4, int(rng.integers(1, 9)), dtype=np.uint8)]
    src = np.concatenate(parts)
    for accel in (1, 5, 9):
        check(team, orc, src, accel, accel % 4)


def test_every_search_branch_ran(team):
    """the ledger: every branch of the search was reached by the streams above"""
    missing = [NAMES[k] for k in range(10) if _total[k] == 0]
    assert not missing, (missing, _total)


# ---- GPU: the crafted streams as the four byte-planes of a typesize-4 chunk, through encode_team_kernel ----

def interleave(planes):
    """elements whose byte k comes from planes[k]: the shuffle of typesize 4 gives the planes back, one stream each"""
    return np.ascontiguousarray(np.stack(planes, axis=1)).reshape(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [40000, 100000])
def test_gpu_team_search_chunks(pkg, orc, cuda, n):
    torch = cuda
    names = sorted(STREAMS)
    planes = [STREAMS[names[k % len(names)]](n) for k in range(4)]
    planes2 = [STREAMS[names[(k + 2) % len(names)]](n) for k in range(4)]
    src = np.concatenate([interleave(planes), interleave(planes2)])          # two blocks of four streams each
    nbytes, bs = len(src), 4 * n
    ra, a = compress(orc, "orc_compress_ctx", 5, 1, 4, src, nbytes + 16, "lz4", bs)
    assert ra > 16
    for nt in (1, 2):
        dest = np.zeros(nbytes + 16 + 64, np.uint8)
        rb = pkg.compress_ctx(5, 1, 4, nbytes, src, dest, nbytes + 16, "lz4", bs, nt)
        assert rb == ra and (dest[:ra] == a[:ra]).all(), (n, nt, ra, rb)
        d_src = torch.from_numpy(src).cuda()
        d_dest = torch.zeros(nbytes + 16, dtype=torch.uint8, device="cuda")
        rd = pkg.compress_ctx(5, 1, 4, nbytes, d_src, d_dest, nbytes + 16, "lz4", bs, nt)
        torch.cuda.synchronize()
        assert rd == ra and (d_dest[:ra].cpu().numpy() == a[:ra]).all(), (n, nt, ra, rd)


@pytest.mark.gpu
def test_gpu_team_forced_bench_buffer(pkg, cuda):
    """The 256 MiB bench.c buffer with the team encoder forced on (BLOSC_B200_LZ4_TEAM=1, read once per process, so
    in a child process) at typesizes 2, 4, 8 and 16: cbytes as BASELINE.md records them, and the round trip"""
    code = textwrap.dedent("""
        import json, sys
        import torch
        sys.path.insert(0, %r); sys.path.insert(0, %r)
        import __graft_entry__ as g
        from datagen import bench_words
        pkg = g.load_package()
        nbytes = 256 << 20
        d_src = torch.from_numpy(bench_words(nbytes)).cuda()
        out = {}
        for ts in (2, 4, 8, 16):
            d_chunk = torch.zeros(nbytes + 16, dtype=torch.uint8, device="cuda")
            cb = pkg.compress_ctx(5, 1, ts, nbytes, d_src, d_chunk, nbytes + 16, "lz4")
            d_back = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
            r = pkg.decompress_ctx(d_chunk, d_back, nbytes)
            torch.cuda.synchronize()
            out[ts] = [cb, r, bool(torch.equal(d_back, d_src))]
        print(json.dumps(out))
    """) % (ROOT, os.path.join(ROOT, "tests"))
    env = dict(os.environ, BLOSC_B200_LZ4_TEAM="1")
    res = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stderr[-3000:]
    got = json.loads(res.stdout.strip().splitlines()[-1])
    baseline = {"2": 37749776, "4": 20401680, "8": 7313680, "16": 10199056}      # BASELINE.md, lz4 / shuffle rows
    for ts, cb in baseline.items():
        assert got[ts] == [cb, 256 << 20, True], (ts, got[ts])

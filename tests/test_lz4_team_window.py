"""The LZ4 team walker's chained windows (dev_lz4.cuh, team mode): the walker hops along the prepared verdicts, checks
up to 16 sequences against the live table in one warp step and commits the valid prefix.  Streams that end windows in
every way -- a stale element at the first position and later, a valid miss, a valid LZ4T_LONG (and a 270+ match), the
end of the stream, a full window, the next position past the checked tiles -- and whose windows hold two stores of
one hash, must give LZ4_compress_fast's bytes and return value at every acceleration, table flavour, walker warp and
short capacity (test_lz4_team.check).  The emulator's window counters (emu_lz4t_window_counters of
tests/emu/lz4t_window_stage.cpp, totals since that library was loaded) show that each case ran."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import test_lz4_team as tlt
from datagen import compress
from test_lz4_team import U16_MAX, chains_and_gaps, colliding
from test_lz4_team_search import edited_repeats, interleave, plane

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# emu_lz4t_window_counters (dev_lz4.cuh, LZ4T_W_*)
WINDOWS, ELEMS, STALE0, STALEJ, FWD, CROSS, MISS0, MISSJ, LONG0, LONGJ, HUGE, END, CAP, TILE, FULL = range(15)
NAMES = ("windows", "elements", "stale at element 0", "stale at a later element", "lookup answered inside the window",
         "h(q_j - 2) == h(q_k)", "miss at element 0", "miss at a later element", "LZ4T_LONG at element 0",
         "LZ4T_LONG at a later element", "270+ match", "end of the stream", "full window", "tile horizon",
         "output too small at a window's flush")
_total = np.zeros(15, np.int64)


def window_counters(emu):
    c = (C.c_longlong * 15)()
    assert emu.emu_lz4t_window_counters(c) == 15
    return np.array(c[:], np.int64)


def check(emu, orc, src, accel, cap=None, walkers=range(4)):
    """test_lz4_team.check on this module's library; its counter baseline (test_lz4_team._seen, kept for the
    emulated library of the other team tests) is left as it was"""
    seen = tlt._seen
    before = window_counters(emu)
    try:
        ra, _ = tlt.check(emu, orc, src, accel, cap, walkers)
    finally:
        tlt._seen = seen
    d = window_counters(emu) - before
    _total[:] += d
    return ra, d


@pytest.fixture(scope="module")
def team(tmp_path_factory):
    """the emulated library with the window counters of tests/emu/lz4t_window_stage.cpp (which includes
    backend_emu.cpp whole), built into a temporary directory"""
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("lz4t_window_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "c-blosc_b200", "csrc", "blosc_b200.c"), "-o",
                    str(d / "host.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "lz4t_window_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    path = str(d / "liblz4t_window_stage.so")
    subprocess.run(["g++", "-shared", "-o", path, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    lib = C.CDLL(path)
    lib.emu_lz4_encode_team.restype = C.c_int
    lib.emu_lz4t_window_counters.restype = C.c_int
    return lib


def test_hard_plane_windows(team, orc):
    """The hard byte-plane of cfg 2 (plane 1 of the bench.c words), in both table flavours: windows must average well
    above one sequence, and the whole stream must come out as LZ4_compress_fast's"""
    for n, accel in ((40000, 5), (120000, 5), (60000, 1), (100000, 9)):
        ra, d = check(team, orc, plane(n, 1), accel, walkers=(n % 4, (n + 1) % 4))
        assert ra > 0
        assert d[ELEMS] > 4 * d[WINDOWS] > 0, d


STREAMS = {
    "plane1": lambda n: plane(n, 1),
    "plane2": lambda n: plane(n, 2),
    "chains": lambda n: chains_and_gaps(n, seed=n + 5),
    "colliding": lambda n: colliding(n, n < U16_MAX, seed=7),
    "alpha4": lambda n: edited_repeats(n, 5, 200, 4, 3),
    "alpha16": lambda n: edited_repeats(n, 6, 700, 16, 8),
}


@pytest.mark.parametrize("n", [50000, 120000])
@pytest.mark.parametrize("name", sorted(STREAMS))
def test_window_streams(team, orc, name, n):
    """every stream at accelerations 1 and 5 on every walker warp, then at accel 5 with capacities from a tenth of
    what it needs to one byte less: a chain crosses the limit at some window's flush"""
    src = STREAMS[name](n)
    full = 0
    for accel in (1, 5):
        ra, _ = check(team, orc, src, accel)
        assert ra > 0
        full = ra
    for k, cap in enumerate([full * i // 10 for i in range(1, 10)] + [full - 1, full]):
        ra, _ = check(team, orc, src, 5, cap=cap, walkers=(k % 4,))
        assert (ra > 0) == (cap >= full)


def test_windows_meet_the_end(team, orc):
    """chains that run into the last 64 bytes of the stream at every distance from its end"""
    rng = np.random.default_rng(21)
    body = plane(20000, 1)
    for tail in list(range(0, 13)) + [20, 40, 63, 64, 65, 70, 90]:
        src = np.concatenate([body, body[-5000:-5000 + 400], rng.integers(0, 4, tail, dtype=np.uint8)])
        check(team, orc, src, 5 if tail % 2 else 1, walkers=(tail % 4,))


def test_window_cycle_columns_match_the_device_enum():
    """scripts/lz4_cycles.py reads the window columns (dev_lz4.cuh, the enum after LZ4C_N) by index"""
    import importlib.util
    import re
    src = open(os.path.join(ROOT, "c-blosc_b200", "csrc", "dev_lz4.cuh")).read()
    body = re.sub(r"/\*.*?\*/", "", re.search(r"enum \{\s*(LZ4C_WINDOWS = LZ4C_N.*?)\};", src, re.S).group(1), flags=re.S)
    names = [t.strip().split(" =")[0][len("LZ4C_"):] for t in body.split(",") if t.strip()]
    assert names[-1] == "NREC"
    spec = importlib.util.spec_from_file_location("lz4_cycles", os.path.join(ROOT, "scripts", "lz4_cycles.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    for i, c in enumerate(names):
        assert getattr(mod, c) == mod.NCOL + i, c


def test_every_window_end_ran(team):
    """the ledger: every way a window ends, and every hash sharing inside a window, was reached by the streams above"""
    missing = [NAMES[k] for k in range(15) if _total[k] == 0]
    assert not missing, (missing, _total)


# ---- GPU: the streams as the four byte-planes of a typesize-4 chunk, through encode_team_kernel ----

@pytest.mark.gpu
@pytest.mark.parametrize("n", [50000, 120000])
def test_gpu_team_window_chunks(pkg, orc, cuda, n):
    torch = cuda
    names = sorted(STREAMS)
    src = np.concatenate([interleave([STREAMS[names[(k + s) % len(names)]](n) for k in range(4)]) for s in (0, 4)])
    nbytes, bs = len(src), 4 * n
    ra, a = compress(orc, "orc_compress_ctx", 5, 1, 4, src, nbytes + 16, "lz4", bs)
    assert ra > 16
    d_src = torch.from_numpy(src).cuda()
    for cap in (nbytes + 16, ra, ra - 1):
        d_dest = torch.zeros(nbytes + 16, dtype=torch.uint8, device="cuda")
        rd = pkg.compress_ctx(5, 1, 4, nbytes, d_src, d_dest, cap, "lz4", bs)
        torch.cuda.synchronize()
        want, wa = (ra, a) if cap >= ra else compress(orc, "orc_compress_ctx", 5, 1, 4, src, cap, "lz4", bs)
        assert rd == want, (n, cap, rd, want)
        if rd > 0:
            assert (d_dest[:rd].cpu().numpy() == wa[:rd]).all(), (n, cap)

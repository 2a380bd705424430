"""blosc_b200_getslice_step / blosc_b200_frame_getslice_step: a[start:stop:step] of an N-d C-order array, planned and
gathered from the box and its steps.

Every result is checked against numpy (or torch) slicing of the source array with the same steps, with sentinel bytes
after the output left untouched.  CPU: the product's host code and kernels inside the SIMT emulator
(tests/emu/getslice_step_stage.cpp, which counts launches, shows the decode launch's listed blocks and which box
kernels ran), and the box arithmetic against brute force over every flat index (tests/emu/box_step_shim.c).  GPU: the
CUDA library through the Python API with torch tensors."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from datagen import bench_words, ci, compress, gen, ptr, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ll = C.c_longlong
vp = C.c_void_p
CODECS = (("blosclz", None), ("lz4", None), ("lz4hc", None), ("zstd", "BLOSC_B200_ZSTD"),
          ("zlib", "BLOSC_B200_ZLIB"), ("snappy", "BLOSC_B200_SNAPPY"))
TYPESIZES = (1, 2, 3, 4, 8, 16)
NITEMS = 5040                                                   # 2^4 * 3^2 * 5 * 7
NEVER_SPLIT, FORWARD_COMPAT_SPLIT = 2, 4
SHAPES = {1: (5040,), 2: (72, 70), 3: (14, 18, 20), 4: (7, 8, 9, 10), 8: (2, 3, 2, 2, 5, 3, 7, 2)}


def _bind(lib):
    lib.blosc_b200_getslice.restype = ll
    lib.blosc_b200_getslice.argtypes = [vp, ci, vp, vp, vp, vp]
    lib.blosc_b200_getslice_step.restype = ll
    lib.blosc_b200_getslice_step.argtypes = [vp, ci, vp, vp, vp, vp, vp]
    lib.blosc_b200_frame_getslice.restype = ll
    lib.blosc_b200_frame_getslice.argtypes = [vp, sz, ci, vp, vp, vp, vp]
    lib.blosc_b200_frame_getslice_step.restype = ll
    lib.blosc_b200_frame_getslice_step.argtypes = [vp, sz, ci, vp, vp, vp, vp, vp]
    lib.blosc_b200_frame_compress.restype = ll
    lib.blosc_b200_frame_compress.argtypes = [ci, ci, sz, sz, vp, vp, sz, C.c_char_p, sz, sz, ci]
    lib.blosc_b200_frame_bound.restype = sz
    lib.blosc_b200_frame_bound.argtypes = [sz, sz, sz]
    lib.blosc_b200_frame_chunk.restype = ll
    lib.blosc_b200_frame_chunk.argtypes = [vp, sz, sz, C.POINTER(sz)]
    lib.blosc_getitem.restype = ci
    lib.blosc_compress_ctx.restype = ci
    return lib


@pytest.fixture(scope="session")
def slib(tmp_path_factory):
    """the emulated library with the counters of tests/emu/getslice_step_stage.cpp and the box arithmetic exported by
    tests/emu/box_step_shim.c, built into a temporary directory"""
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("getslice_step_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(emu_dir, "box_step_shim.c"), "-o", str(d / "host.o")],
                   check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "getslice_step_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    path = str(d / "libgetslice_step_stage.so")
    subprocess.run(["g++", "-shared", "-o", path, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    lib = _bind(C.CDLL(path))
    lib.emu_last_decode_blocks.restype = ci
    lib.emu_all_launches.restype = ll
    lib.emu_last_box_stepped.restype = ci
    lib.emu_last_box_run.restype = ll
    lib.emu_set_device_ptrs.argtypes = [vp, vp]
    lib.blosc_set_splitmode.argtypes = [ci]
    lib.emu_box_size.restype = sz
    lib.emu_box_build.argtypes = [ci, vp, vp, vp, vp, vp]
    for f in ("emu_box_ndim", "emu_box_stepped"):
        getattr(lib, f).argtypes = [vp]
    for f in ("emu_box_run", "emu_box_count"):
        getattr(lib, f).argtypes = [vp]
        getattr(lib, f).restype = ll
    for f in ("emu_box_next", "emu_box_rank", "emu_box_unrank"):
        getattr(lib, f).argtypes = [vp, ll]
        getattr(lib, f).restype = ll
    lib.blosc_set_splitmode(NEVER_SPLIT)                          # small forced blocks: many of them per chunk
    return lib


# ---------------------------------------------------------------------------------------------------------------
# expected results, from the geometry alone
# ---------------------------------------------------------------------------------------------------------------
def _sl(start, stop, step):
    return tuple(slice(s, e, t) for s, e, t in zip(start, stop, step))


def _want(src, ts, shape, start, stop, step):
    return np.ascontiguousarray(src.reshape(*shape, ts)[_sl(start, stop, step)]).reshape(-1)


def _selected(shape, start, stop, step):
    """the flat indices of the selected items, ascending"""
    return np.arange(int(np.prod(shape)), dtype=np.int64).reshape(shape)[_sl(start, stop, step)].reshape(-1)


def _touched(shape, start, stop, step, ts, bs):
    """blocks that hold a byte of a selected item"""
    f = _selected(shape, start, stop, step)
    return np.unique(np.concatenate([(f * ts) // bs, (f * ts + ts - 1) // bs])).size


def _arr(v):
    return np.ascontiguousarray(v, dtype=np.int64)


def _getslice(lib, src_p, shape, start, stop, step, dest):
    sh, st, sp = _arr(shape), _arr(start), _arr(stop)
    t = None if step is None else _arr(step)
    return lib.blosc_b200_getslice_step(src_p, len(shape), sh.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                        None if t is None else t.ctypes.data, dest.ctypes.data)


def _frame_getslice(lib, frame_p, fb, shape, start, stop, step, dest_p):
    sh, st, sp, t = _arr(shape), _arr(start), _arr(stop), _arr(step)
    return lib.blosc_b200_frame_getslice_step(frame_p, fb, len(shape), sh.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                              t.ctypes.data, dest_p)


def _boxes(shape, rng, k):
    """k seeded boxes, none empty, with steps from {1, 2, 3, 7, > extent}.  Some dimensions are whole with step 1 (they
    merge into a step-1 dimension before them, and must not merge into a stepped one), some whole but stepped."""
    out = []
    for _ in range(k):
        start, stop, step = [], [], []
        for s in shape:
            kind = rng.integers(0, 4)
            if kind == 0:
                a, b, t = 0, s, 1
            elif kind == 1:
                a, b, t = 0, s, int(rng.choice([2, 3, 7, s + 1]))
            else:
                a = int(rng.integers(0, s))
                b = int(rng.integers(a + 1, s + 1))
                t = int(rng.choice([1, 2, 3, 7, b - a + int(rng.integers(0, 3))]))
            start.append(a)
            stop.append(b)
            step.append(max(t, 1))
        out.append((start, stop, step))
    return out


def _check(lib, chunk, src, ts, shape, start, stop, step):
    want = _want(src, ts, shape, start, stop, step)
    out = np.full(want.size + 16, 0xAA, np.uint8)
    r = _getslice(lib, ptr(chunk), shape, start, stop, step, out)
    assert r == want.size, (shape, start, stop, step, r, want.size)
    assert (out[:r] == want).all() and (out[r:] == 0xAA).all(), (shape, start, stop, step)
    return r


def _compress(lib, comp, clevel, shuf, ts, src, bs, monkeypatch=None, switch=None):
    if switch:
        monkeypatch.setenv(switch, "1")
    r, c = compress(lib, "blosc_compress_ctx", clevel, shuf, ts, src, len(src) + 16, comp, bs)
    assert r > 0, (comp, ts, shuf, r)
    return c[:r].copy()


# ---------------------------------------------------------------------------------------------------------------
# CPU: the box arithmetic
# ---------------------------------------------------------------------------------------------------------------
def _box(lib, shape, start, stop, step):
    b = np.zeros(lib.emu_box_size(), np.uint8)
    sh, st, sp, t = _arr(shape), _arr(start), _arr(stop), _arr(step)
    assert lib.emu_box_build(len(shape), sh.ctypes.data, st.ctypes.data, sp.ctypes.data, t.ctypes.data, b.ctypes.data) == 0
    return b


@pytest.mark.parametrize("shape", [(23,), (6, 7), (4, 5, 6), (3, 4, 2, 5), (1, 6, 1, 4)])
def test_box_arithmetic_brute_force(slib, shape):
    """next / rank / unrank of stepped boxes against the selected flat indices, at every flat index"""
    n = int(np.prod(shape))
    rng = np.random.default_rng(len(shape) * 100 + n)
    boxes = _boxes(shape, rng, 40) + [([0] * len(shape), list(shape), [2] * len(shape)),
                                      ([s - 1 for s in shape], list(shape), [5] * len(shape))]
    for start, stop, step in boxes:
        b = _box(slib, shape, start, stop, step)
        sel = _selected(shape, start, stop, step)
        assert slib.emu_box_count(b.ctypes.data) == sel.size
        for x in range(n + 1):
            i = int(np.searchsorted(sel, x))
            assert slib.emu_box_next(b.ctypes.data, x) == (sel[i] if i < sel.size else n), (start, stop, step, x)
            assert slib.emu_box_rank(b.ctypes.data, x) == i, (start, stop, step, x)
        for p in range(sel.size):
            assert slib.emu_box_unrank(b.ctypes.data, p) == sel[p], (start, stop, step, p)


def test_box_normalisation(slib):
    """steps that select one coordinate become 1, whole step-1 dimensions merge only into step-1 ones, and the run is
    one item under an innermost step"""
    cases = (  # shape, start, stop, step -> ndim, stepped, run
        ((6, 7), (0, 0), (6, 7), (1, 1), 1, 0, 42),
        ((6, 7), (0, 0), (6, 7), (2, 1), 2, 1, 7),              # whole step-1 dimension after a stepped one: no merge
        ((6, 7), (0, 0), (6, 7), (1, 2), 2, 1, 1),              # whole but stepped: no merge, runs of one item
        ((6, 7), (2, 0), (3, 7), (5, 1), 1, 0, 7),              # one coordinate: step 1, then the merge
        ((6, 7), (1, 3), (6, 4), (2, 9), 2, 1, 1),
        ((4, 5, 6), (0, 0, 0), (4, 5, 6), (1, 1, 3), 2, 1, 1),  # the first two merge, the stepped last stays
        ((4, 5, 6), (0, 0, 0), (4, 5, 6), (2, 1, 1), 2, 1, 30),
        ((4, 5, 6), (1, 0, 0), (4, 5, 6), (9, 2, 1), 3, 1, 6),  # step 9 selects one: 1; whole 6 after step 2 stays
        ((1, 6, 1, 4), (0, 0, 0, 0), (1, 6, 1, 4), (3, 1, 8, 1), 1, 0, 24),
    )
    for shape, start, stop, step, ndim, stepped, run in cases:
        b = _box(slib, shape, start, stop, step)
        got = (slib.emu_box_ndim(b.ctypes.data), slib.emu_box_stepped(b.ctypes.data), slib.emu_box_run(b.ctypes.data))
        assert got == (ndim, stepped, run), (shape, start, stop, step, got)


def test_box_step_int64_max(slib):
    """a step of INT64_MAX selects the start alone, with no overflow"""
    big = (1 << 63) - 1
    b = _box(slib, (1 << 40, 3), (5, 0), (1 << 40, 3), (big, big))
    assert slib.emu_box_count(b.ctypes.data) == 1 and slib.emu_box_stepped(b.ctypes.data) == 0
    assert slib.emu_box_unrank(b.ctypes.data, 0) == 15


# ---------------------------------------------------------------------------------------------------------------
# CPU: the emulator
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("comp,switch", CODECS)
@pytest.mark.parametrize("shuf", [0, 1, 2])
def test_getslice_step_matrix_emu(slib, monkeypatch, comp, switch, shuf):
    """every codec, filter, typesize and ndim: seeded stepped boxes against numpy"""
    for ts, split in [(ts, NEVER_SPLIT) for ts in TYPESIZES] + [(16, FORWARD_COMPAT_SPLIT)]:
        src = gen("mixed" if ts % 2 else "i32", NITEMS * ts, seed=ts)
        slib.blosc_set_splitmode(split)
        try:
            chunk = _compress(slib, comp, 5, shuf, ts, src, 1024, monkeypatch, switch)
        finally:
            slib.blosc_set_splitmode(NEVER_SPLIT)
        for ndim, shape in SHAPES.items():
            for start, stop, step in _boxes(shape, np.random.default_rng(100 * ts + ndim + shuf), 3):
                _check(slib, chunk, src, ts, shape, start, stop, step)


def test_getslice_step_ones_unchanged_emu(slib):
    """all-ones steps and step == NULL give getslice's bytes and launches, on the step-1 kernels; so does a box whose
    steps normalise to 1"""
    ts, shape = 4, (14, 18, 20)
    src = gen("i32", NITEMS * ts, seed=11)
    chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
    boxes = [(a, b, [1, 1, 1]) for a, b, _ in _boxes(shape, np.random.default_rng(4), 6)]
    boxes += [([2, 0, 5], [3, 18, 20], [7, 1, 1]), ([0, 4, 0], [14, 5, 20], [1, 30, 1]), ([3, 3, 3], [4, 4, 4], [2, 2, 2])]
    for start, stop, step in boxes:
        want = _want(src, ts, shape, start, stop, step)
        outs, launches = [], []
        for call in ("getslice", "null", "step"):
            out = np.full(want.size + 16, 0xAA, np.uint8)
            before = slib.emu_all_launches()
            if call == "getslice":
                sh, st = _arr(shape), _arr(start)
                sp = _arr([b if t == 1 else a + 1 for a, b, t in zip(start, stop, step)])   # steps > 1 select one
                r = slib.blosc_b200_getslice(ptr(chunk), 3, sh.ctypes.data, st.ctypes.data, sp.ctypes.data, ptr(out))
            else:
                r = _getslice(slib, ptr(chunk), shape, start, stop, None if call == "null" else step, out)
            launches.append(slib.emu_all_launches() - before)
            assert r == want.size and slib.emu_last_box_stepped() == 0, (call, start, stop, step)
            outs.append(out)
        assert (outs[0][:want.size] == want).all() and (outs[0][want.size:] == 0xAA).all()
        assert all((o == outs[0]).all() for o in outs) and launches[0] == launches[1] == launches[2] == 5, launches
    _check(slib, chunk, src, ts, shape, [0, 0, 0], list(shape), [1, 1, 2])
    assert slib.emu_last_box_stepped() == 1 and slib.emu_last_box_run() == 1


def test_getslice_step_special_emu(slib):
    """whole-but-stepped dimensions, steps past the extent, dimensions that must not merge, the short last block,
    empty boxes (nothing launched), on a compressed and a memcpyed chunk, typesizes 4 and 3"""
    for ts in (4, 3):
        src = gen("i32" if ts == 4 else "mixed", NITEMS * ts, seed=ts)
        for clevel in (5, 0):
            chunk = _compress(slib, "lz4", clevel, 1, ts, src, 1024)
            shape = (72, 70)
            for start, stop, step in (([0, 0], [72, 70], [2, 2]), ([0, 0], [72, 70], [3, 1]), ([0, 0], [72, 70], [1, 7]),
                                      ([1, 2], [72, 70], [71, 68]), ([5, 69], [72, 70], [5, 1]), ([0, 3], [72, 70], [1, 3]),
                                      ([70, 0], [72, 70], [1, 69]), ([0, 0], [72, 70], [72, 70]), ([0, 5], [72, 6], [2, 9])):
                _check(slib, chunk, src, ts, shape, start, stop, step)
            for start, stop, step in (([0, 0, 0, 0], [7, 8, 9, 10], [2, 1, 1, 1]), ([1, 0, 0, 0], [7, 8, 9, 10], [1, 1, 3, 1]),
                                      ([0, 0, 0, 1], [7, 8, 9, 10], [1, 2, 1, 4]), ([6, 7, 8, 0], [7, 8, 9, 10], [1, 1, 1, 3])):
                _check(slib, chunk, src, ts, (7, 8, 9, 10), start, stop, step)
            _check(slib, chunk, src, ts, (NITEMS,), [NITEMS - 1], [NITEMS], [3])
            out = np.full(64, 0xAA, np.uint8)
            before = slib.emu_all_launches()
            assert _getslice(slib, ptr(chunk), shape, [3, 5], [3, 9], [2, 2], out) == 0
            assert slib.emu_all_launches() == before and (out == 0xAA).all()


@pytest.mark.parametrize("clevel", [5, 0])
@pytest.mark.parametrize("src_dev,dest_dev", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_getslice_step_placements_emu(slib, clevel, src_dev, dest_dev):
    """src and dest in host and device memory (a memcpyed chunk in device memory is read in place, with no plan)"""
    ts, shape = 4, (14, 18, 20)
    src = gen("i32", NITEMS * ts, seed=7)
    chunk = _compress(slib, "lz4", clevel, 1, ts, src, 1024)
    rng = np.random.default_rng(clevel + 10 * src_dev + 20 * dest_dev)
    for start, stop, step in _boxes(shape, rng, 5) + [([0, 0, 0], list(shape), [3, 2, 7])]:
        want = _want(src, ts, shape, start, stop, step)
        out = np.full(want.size + 16, 0xAA, np.uint8)
        slib.emu_set_device_ptrs(chunk.ctypes.data if src_dev else None, out.ctypes.data if dest_dev else None)
        try:
            before = slib.emu_all_launches()
            r = _getslice(slib, ptr(chunk), shape, start, stop, step, out)
            grown = slib.emu_all_launches() - before
        finally:
            slib.emu_set_device_ptrs(None, None)
        assert r == want.size and (out[:r] == want).all() and (out[r:] == 0xAA).all()
        if clevel == 0 and src_dev:
            assert grown == 1                                     # the gather alone, in place


def test_getslice_step_decodes_touched_blocks_emu(slib):
    """the decode launch lists exactly the blocks that hold a byte of a selected item; a[::k] with k * typesize of two
    blocks or more skips blocks"""
    for ts, shape in ((4, (72, 70)), (3, (7, 8, 9, 10)), (16, (14, 18, 20)), (4, (NITEMS,))):
        src = gen("mixed" if ts == 3 else "i32", NITEMS * ts, seed=ts)
        chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
        bs = int(chunk[8:12].view(np.int32)[0])
        nblocks = -(-NITEMS * ts // bs)
        assert not chunk[2] & 0x2
        boxes = _boxes(shape, np.random.default_rng(ts + len(shape)), 6)
        if len(shape) == 1:
            boxes += [([0], [NITEMS], [k]) for k in (2 * bs // ts + 1, 3 * bs // ts, 1000)]
        for start, stop, step in boxes:
            _check(slib, chunk, src, ts, shape, start, stop, step)
            want = _touched(shape, start, stop, step, ts, bs)
            assert slib.emu_last_decode_blocks() == want, (start, stop, step)
            if len(shape) == 1 and step[0] * ts >= 2 * bs:          # a whole block between two items
                assert want < nblocks


def test_getslice_step_launches_emu(slib):
    """a stepped read of 10 items and one of 10^4 one-item runs make the same 5 launches"""
    src = bench_words(80000)
    chunk = _compress(slib, "lz4", 5, 1, 4, src, 4096)
    assert not chunk[2] & 0x2
    counts = []
    for shape, start, stop, step in (((1000, 20), [5, 0], [6, 20], [1, 2]),      # 10 items
                                     ((20000,), [0], [20000], [2]),              # 10^4 one-item runs
                                     ((10000, 2), [0, 1], [10000, 2], [1, 1])):  # 10^4 runs, unstepped
        before = slib.emu_all_launches()
        _check(slib, chunk, src, 4, shape, start, stop, step)
        counts.append(slib.emu_all_launches() - before)
        assert slib.emu_last_box_run() == 1 and slib.emu_last_box_stepped() == (step != [1, 1])
    assert counts == [5, 5, 5], counts                            # touch, slot scan, decode, unfilter, gather


def test_getslice_step_damaged_block_emu(slib):
    """a damaged block that no selected item touches is not read; one that one touches gives blosc_d's code, dest
    untouched"""
    ts, shape = 4, (72, 70)
    src = gen("i32", NITEMS * ts, seed=3)
    chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
    bs = int(chunk[8:12].view(np.int32)[0])
    h = chunk.copy()
    h[16 + 4 * 5:16 + 4 * 6].view(np.int32)[0] = 0x7fff0000      # block 5's bstarts entry
    item5 = 5 * bs // ts                                           # the first item of block 5
    per = bs // ts                                                 # items a block
    for src_dev in (0, 1):
        slib.emu_set_device_ptrs(h.ctypes.data if src_dev else None, None)
        try:
            code = slib.blosc_getitem(ptr(h), ci(item5), ci(1), ptr(np.zeros(64, np.uint8)))
            assert code < 0
            flat = (NITEMS,)
            _check(slib, h, src, ts, flat, [item5 - 1], [NITEMS], [per + 1])          # jumps over block 5
            assert 5 * bs > (item5 - 1) * ts and (item5 - 1 + per + 1) * ts >= 6 * bs
            out = np.full(8192, 0xAA, np.uint8)
            assert _getslice(slib, ptr(h), flat, [item5 - 3], [NITEMS], [per], out) == code and (out == 0xAA).all()
            r5, c5 = divmod(item5, 70)
            assert _getslice(slib, ptr(h), shape, [0, c5], [72, c5 + 1], [r5 or 1, 1], out) == code
            assert (out == 0xAA).all()
        finally:
            slib.emu_set_device_ptrs(None, None)


def test_getslice_step_rejects_emu(slib, capfd):
    ts = 4
    src = gen("i32", NITEMS * ts, seed=2)
    chunk = _compress(slib, "lz4", 5, 1, ts, src, 1024)
    out = np.full(64, 0xAA, np.uint8)
    capfd.readouterr()
    for shape, start, stop, step, msg in (
            ((72, 70), (0, 0), (2, 3), (1, 0), "step[1] = 0"), ((72, 70), (0, 0), (2, 3), (-1, 1), "step[0] = -1"),
            ((72, 70), (0, 0), (0, 0), (0, 1), "step[0] = 0"),
            ((), (), (), (), "ndim"), ((1,) * 8 + (5040,), (0,) * 9, (1,) * 9, (1,) * 9, "ndim"),
            ((-72, -70), (0, 0), (1, 1), (1, 1), "negative"), ((72, 71), (0, 0), (1, 1), (1, 1), "items"),
            ((1 << 40, 1 << 40), (0, 0), (1, 1), (1, 1), "overflows"), ((72, 70), (3, 0), (2, 1), (1, 1), "inside"),
            ((72, 70), (0, 0), (1, 71), (1, 1), "inside"), ((72, 70), (-1, 0), (1, 1), (2, 2), "inside")):
        before = slib.emu_all_launches()
        sh, st, sp, t = (_arr(v) if len(v) else np.zeros(1, np.int64) for v in (shape, start, stop, step))
        r = slib.blosc_b200_getslice_step(ptr(chunk), len(shape), sh.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                          t.ctypes.data, ptr(out))
        assert r == -1 and (out == 0xAA).all() and slib.emu_all_launches() == before, (shape, step, r)
        err = capfd.readouterr().err
        assert err.count("blosc_b200") == 1 and msg in err, (shape, step, err)
    for patch, code in ((lambda h: h.__setitem__(0, 3), -9), (lambda h: h.__setitem__(1, 9), -9),
                        (lambda h: h.__setitem__(2, (h[2] & 0x1f) | (6 << 5)), -5),
                        (lambda h: h[8:12].view(np.int32).__setitem__(0, 0), -1)):
        h = chunk.copy()
        patch(h)
        assert _getslice(slib, ptr(h), (72, 70), (0, 0), (5, 7), (2, 3), out) == code and (out == 0xAA).all()


def _frame(lib, src, ts, chunksize, clevel=5):
    fb = lib.blosc_b200_frame_bound(len(src), ts, chunksize)
    frame = np.zeros(fb, np.uint8)
    r = lib.blosc_b200_frame_compress(clevel, 1, ts, len(src), ptr(src), ptr(frame), fb, b"lz4", 1024, chunksize, 1)
    assert r > 0
    return frame[:r].copy()


def _check_frame(lib, frame, src, ts, shape, start, stop, step):
    want = _want(src, ts, shape, start, stop, step)
    out = np.full(want.size + 16, 0xAA, np.uint8)
    r = _frame_getslice(lib, frame.ctypes.data, len(frame), shape, start, stop, step, out.ctypes.data)
    assert r == want.size and (out[:r] == want).all() and (out[r:] == 0xAA).all(), (shape, start, stop, step, r)


@pytest.mark.parametrize("dev", [0, 1])
def test_frame_getslice_step_emu(slib, dev):
    """stepped boxes across chunk boundaries, a chunksize that is no multiple of the row, a short last chunk"""
    ts, shape = 4, (50, 37)
    src = gen("i32", 50 * 37 * ts, seed=5)
    frame = _frame(slib, src, ts, 1000)                           # 250 items a chunk, 8 chunks, the last of 100
    slib.emu_set_all_device(dev)
    try:
        boxes = _boxes(shape, np.random.default_rng(dev + 7), 8) + [([0, 0], [50, 37], [3, 4]), ([6, 36], [50, 37], [7, 1]),
                                                                   ([1, 2], [50, 30], [1, 9]), ([0, 9], [50, 10], [13, 1])]
        for start, stop, step in boxes:
            _check_frame(slib, frame, src, ts, shape, start, stop, step)
        for start, stop, step in _boxes((10, 5, 37), np.random.default_rng(19), 4):
            _check_frame(slib, frame, src, ts, (10, 5, 37), start, stop, step)
    finally:
        slib.emu_set_all_device(0)


def test_frame_getslice_step_skips_chunks_emu(slib, capfd):
    """chunks that hold no selected item are not read: a damaged one leaves the read intact; a damaged touched one
    decides the result, with a host dest untouched"""
    ts, shape = 4, (50, 37)
    src = gen("i32", 50 * 37 * ts, seed=6)
    frame = _frame(slib, src, ts, 1000)                           # chunk c holds items [250 c, 250 c + 250)
    off = [slib.blosc_b200_frame_chunk(frame.ctypes.data, len(frame), i, None) for i in range(8)]
    for patch, code in ((lambda f: f.__setitem__(off[2] + 3, 2), -1), (lambda f: f.__setitem__(off[2], 3), -9)):
        f = frame.copy()
        patch(f)
        for dev in (0, 1):
            slib.emu_set_all_device(dev)
            try:
                # rows 0, 20, 40: items [0, 37), [740, 777), [1480, 1517) in chunks 0, 2, 5
                out = np.full(3 * 37 * ts + 16, 0xAA, np.uint8)
                capfd.readouterr()
                r = _frame_getslice(slib, f.ctypes.data, len(f), shape, (0, 0), (50, 37), (20, 1), out.ctypes.data)
                assert r == code and (dev or (out == 0xAA).all()), (code, r)
                if code == -1:
                    assert "blosc_b200" in capfd.readouterr().err
                _check_frame(slib, f, src, ts, shape, [0, 0], [50, 37], [27, 1])          # rows 0, 27: chunks 0, 3, 4
                _check_frame(slib, f, src, ts, (1850,), [0], [1850], [750])               # items 0, 750, 1500
            finally:
                slib.emu_set_all_device(0)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the CUDA library
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def glib(pkg):
    return _bind(pkg.lib)


def _gpu_check(pkg, torch, chunk_h, chunk_d, src, ts, shape, start, stop, step):
    want = _want(src, ts, shape, start, stop, step)
    for s_buf in (chunk_h, chunk_d):
        for dest_dev in (False, True):
            out = torch.full((want.size + 16,), 0xAA, dtype=torch.uint8, device="cuda") if dest_dev else \
                np.full(want.size + 16, 0xAA, np.uint8)
            r = pkg.getslice(s_buf, shape, start, stop, out, step=step)
            got = out.cpu().numpy() if dest_dev else out
            assert r == want.size and (got[:r] == want).all() and (got[r:] == 0xAA).all(), (shape, start, stop, step, r)


@pytest.mark.gpu
@pytest.mark.parametrize("comp,switch", (("blosclz", None), ("lz4", None), ("zstd", "BLOSC_B200_ZSTD")))
@pytest.mark.parametrize("shuf", [0, 1, 2])
def test_getslice_step_matrix_gpu(pkg, glib, cuda, monkeypatch, comp, switch, shuf):
    """seeded stepped boxes against torch slicing of the CUDA tensor, typesizes 1, 4, 3 and 16 (the warp gather)"""
    torch = cuda
    n = 1 << 18
    shapes = {1: (n,), 2: (512, 512), 3: (64, 64, 64), 8: (4, 4, 4, 4, 4, 4, 8, 8)}
    for i, ts in enumerate((1, 4, 3, 16)):
        src = (gen("mixed", n * ts, seed=ts) if i % 2 else bench_words(n * ts))
        d_src = torch.from_numpy(src).cuda()
        for bs in (0, 16384):
            chunk = _compress(glib, comp, 5, shuf, ts, src, bs, monkeypatch, switch)
            d_chunk = torch.from_numpy(chunk).cuda()
            for ndim, shape in shapes.items():
                for start, stop, step in _boxes(shape, np.random.default_rng(ts + ndim + bs), 2):
                    _gpu_check(pkg, torch, chunk, d_chunk, src, ts, shape, start, stop, step)
                    want = d_src.view(*shape, ts)[_sl(start, stop, step)].contiguous().view(-1)
                    out = torch.full((want.numel(),), 0xAA, dtype=torch.uint8, device="cuda")
                    assert pkg.getslice(d_chunk, shape, start, stop, out, step=step) == want.numel()
                    assert torch.equal(out, want)
            _gpu_check(pkg, torch, chunk, d_chunk, src, ts, (512, 512), [0, 0], [512, 512], [2, 2])
            _gpu_check(pkg, torch, chunk, d_chunk, src, ts, (512, 512), [1, 7], [512, 8], [3, 1])


@pytest.fixture(scope="module")
def big(pkg, cuda):
    """a 256 MiB LZ4 + shuffle chunk of bench.c words, typesize 4, on the device, with its source"""
    torch = cuda
    src = torch.from_numpy(bench_words(256 << 20)).cuda()
    d_chunk = torch.zeros((256 << 20) + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(5, 1, 4, 256 << 20, src, d_chunk, (256 << 20) + 16, "lz4")
    assert cb > 0
    return src, d_chunk[:cb].clone()


@pytest.mark.gpu
def test_getslice_step_big_chunk_gpu(pkg, cuda, big):
    """8192 x 8192 float32 at [::2, ::2], [::16, 3::16], [::1024] and the column [::4, 17], against torch"""
    torch = cuda
    src, d_chunk = big
    a = src.view(torch.float32).view(8192, 8192)
    for start, stop, step in (((0, 0), (8192, 8192), (2, 2)), ((0, 3), (8192, 8192), (16, 16)),
                              ((0, 0), (8192, 8192), (1024, 1)), ((0, 17), (8192, 18), (4, 1))):
        want = a[_sl(start, stop, step)].contiguous().view(torch.uint8).view(-1)
        out = torch.full((want.numel() + 16,), 0xAA, dtype=torch.uint8, device="cuda")
        before = pkg.launch_count()
        assert pkg.getslice(d_chunk, (8192, 8192), start, stop, out, step=step) == want.numel()
        assert pkg.launch_count() - before == 5, (start, stop, step)
        assert torch.equal(out[:want.numel()], want) and bool((out[want.numel():] == 0xAA).all()), (start, stop, step)


@pytest.mark.gpu
def test_getslice_step_skips_blocks_gpu(pkg, cuda, big):
    """a 1-d [::2**20] of the 256 MiB chunk decodes only the blocks it touches, in one decode launch: it reads right
    with every other block damaged"""
    torch = cuda
    src, d_chunk = big
    h = d_chunk.cpu().numpy().copy()
    bs = int(h[8:12].view(np.int32)[0])
    nblocks = -(-(256 << 20) // bs)
    touched = {(i << 20) * 4 // bs for i in range(64)}
    assert len(touched) == 64 < nblocks
    for b in set(range(nblocks)) - touched:                       # every untouched block's bstarts entry
        h[16 + 4 * b:16 + 4 * (b + 1)].view(np.int32)[0] = 0x7fff0000
    d_bad = torch.from_numpy(h).cuda()
    untouched = min(set(range(nblocks)) - touched)
    assert pkg.getitem(d_bad, untouched * bs // 4, 1, torch.zeros(64, dtype=torch.uint8, device="cuda")) < 0
    want = src.view(torch.int32)[::1 << 20].contiguous().view(torch.uint8)
    out = torch.zeros(want.numel(), dtype=torch.uint8, device="cuda")
    pkg.set_profiling(True)
    try:
        pkg.prof_reset()
        assert pkg.getslice(d_bad, (1 << 26,), (0,), (1 << 26,), out, step=(1 << 20,)) == want.numel() == 256
        torch.cuda.synchronize()
        prof = pkg.prof_get()
    finally:
        pkg.set_profiling(False)
    assert torch.equal(out, want)
    assert prof["decode"][1] == 1 and prof["gather"][1] == 1, prof


@pytest.mark.gpu
@pytest.mark.parametrize("frame_dev", [False, True])
def test_frame_getslice_step_gpu(pkg, glib, cuda, frame_dev):
    torch = cuda
    ts, shape = 4, (3000, 1001)
    src = bench_words(3000 * 1001 * ts)
    frame = _frame(glib, src, ts, 1 << 20)                        # 262144 items a chunk: 12 chunks, the last one short
    f_buf = torch.from_numpy(frame).cuda() if frame_dev else frame
    for start, stop, step in _boxes(shape, np.random.default_rng(3), 4) + [([0, 0], list(shape), [2, 2]),
                                                                         ([0, 500], [3000, 501], [7, 1]),
                                                                         ([261, 0], [3000, 1001], [1300, 1]),
                                                                         ([1, 3], [3000, 1001], [3, 1000])]:
        want = _want(src, ts, shape, start, stop, step)
        for dest_dev in (False, True):
            out = torch.full((want.size + 16,), 0xAA, dtype=torch.uint8, device="cuda") if dest_dev else \
                np.full(want.size + 16, 0xAA, np.uint8)
            assert pkg.frame_getslice(f_buf, len(frame), shape, start, stop, out, step=step) == want.size
            got = out.cpu().numpy() if dest_dev else out
            assert (got[:want.size] == want).all() and (got[want.size:] == 0xAA).all(), (start, stop, step)


@pytest.mark.gpu
def test_getslice_step_two_threads_gpu(pkg, cuda):
    """two host threads reading stepped boxes of the same chunk and frame at once"""
    torch = cuda
    ts, shape = 4, (1024, 1536)
    src = bench_words(1024 * 1536 * ts)
    d_chunk = torch.from_numpy(_compress(pkg.lib, "lz4", 5, 1, ts, src, 0)).cuda()
    frame = _frame(pkg.lib, src, ts, 1 << 20)
    d_frame = torch.from_numpy(frame).cuda()
    errors = []

    def reader(seed):
        try:
            for rep, (start, stop, step) in enumerate(_boxes(shape, np.random.default_rng(seed), 6)):
                want = _want(src, ts, shape, start, stop, step)
                out = torch.full((want.size + 8,), 0xAA, dtype=torch.uint8, device="cuda")
                r = pkg.getslice(d_chunk, shape, start, stop, out, step=step) if rep % 2 else \
                    pkg.frame_getslice(d_frame, len(frame), shape, start, stop, out, step=step)
                got = out.cpu().numpy()
                if r != want.size or not (got[:r] == want).all() or not (got[r:] == 0xAA).all():
                    errors.append((seed, rep, r, want.size))
        except Exception as e:                                      # noqa: BLE001 -- reported below
            errors.append((seed, repr(e)))

    threads = [threading.Thread(target=reader, args=(s,)) for s in (1, 2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


@pytest.mark.gpu
def test_getslice_step_python_args_gpu(pkg, cuda):
    """step=None calls the step-less symbol; a step of the wrong length raises; a bad step returns -1"""
    torch = cuda
    src = bench_words(4096)
    d_chunk = torch.from_numpy(_compress(pkg.lib, "lz4", 5, 1, 4, src, 0)).cuda()
    out = torch.full((4096,), 0xAA, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        pkg.getslice(d_chunk, (32, 32), (0, 0), (32, 32), out, step=(2,))
    assert pkg.getslice(d_chunk, (32, 32), (0, 0), (32, 32), out, step=(0, 1)) == -1
    assert bool((out == 0xAA).all())
    assert pkg.getslice(d_chunk, (32, 32), (0, 0), (32, 32), out, step=None) == 4096
    assert (out.cpu().numpy() == src).all()

"""blosc_b200_getoindex / blosc_b200_frame_getoindex: orthogonal index selections of an N-d C-order array (numpy's
a[np.ix_(...)] with slices kept as slices), index lists per dimension planned and gathered on the GPU.

Every result is checked against numpy (or torch) indexing of the source array, with sentinel bytes after the output
left untouched.  CPU: the product's host code and kernels inside the SIMT emulator (tests/emu/getoindex_stage.cpp,
which counts launches, read-backs and syncs, shows the decode launch's listed blocks and which frame chunks were
gathered).  GPU: the CUDA library through the Python API with torch tensors."""
import ctypes as C
import os
import subprocess

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
    lib.blosc_b200_getoindex.restype = ll
    lib.blosc_b200_getoindex.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, vp]
    lib.blosc_b200_frame_getoindex.restype = ll
    lib.blosc_b200_frame_getoindex.argtypes = [vp, sz, ci, vp, vp, vp, vp, vp, vp, vp]
    lib.blosc_b200_getslice_step.restype = ll
    lib.blosc_b200_getslice_step.argtypes = [vp, ci, vp, vp, vp, vp, vp]
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
def olib(tmp_path_factory):
    """the emulated library with the counters of tests/emu/getoindex_stage.cpp, built into a temporary directory"""
    emu_dir = os.path.join(ROOT, "tests", "emu")
    d = tmp_path_factory.mktemp("getoindex_stage")
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-I", emu_dir, "-x", "c++"]
    subprocess.run(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "c-blosc_b200", "csrc", "blosc_b200.c"), "-o",
                    str(d / "host.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "getoindex_stage.cpp"), "-o", str(d / "stage.o")], check=True)
    subprocess.run(cxx + ["-c", os.path.join(emu_dir, "simt_emu.cpp"), "-o", str(d / "simt.o")], check=True)
    path = str(d / "libgetoindex_stage.so")
    subprocess.run(["g++", "-shared", "-o", path, str(d / "host.o"), str(d / "stage.o"), str(d / "simt.o"), "-lpthread"],
                   check=True)
    lib = _bind(C.CDLL(path))
    lib.emu_last_decode_blocks.restype = ci
    lib.emu_all_launches.restype = ll
    lib.emu_last_box_stepped.restype = ci
    lib.emu_set_device_ptrs.argtypes = [vp, vp]
    lib.blosc_set_splitmode.argtypes = [ci]
    lib.emu_oindex_ngathers.restype = ci
    lib.emu_oindex_window.restype = ll
    lib.emu_oindex_window.argtypes = [ci]
    lib.emu_oindex_last_run.restype = ci
    lib.emu_d2h_copies.restype = ll
    lib.emu_syncs.restype = ll
    lib.blosc_set_splitmode(NEVER_SPLIT)                          # small forced blocks: many of them per chunk
    return lib


# ---------------------------------------------------------------------------------------------------------------
# selections and their expected results
# ---------------------------------------------------------------------------------------------------------------
def _coords(shape, sel):
    """the coordinates each dimension selects, in order"""
    return [np.arange(n)[s] if isinstance(s, slice) else np.asarray(s, dtype=np.int64) for s, n in zip(sel, shape)]


def _want(src, ts, shape, sel):
    return np.ascontiguousarray(src.reshape(*shape, ts)[np.ix_(*_coords(shape, sel))]).reshape(-1)


def _flat(shape, sel):
    """the flat indices of the selected items, in output order"""
    return np.arange(int(np.prod(shape)), dtype=np.int64).reshape(shape)[np.ix_(*_coords(shape, sel))].reshape(-1)


def _touched(shape, sel, ts, bs):
    """blocks that hold a byte of a selected item"""
    f = _flat(shape, sel)
    return np.unique(np.concatenate([(f * ts) // bs, (f * ts + ts - 1) // bs])).size


LIST_KINDS = ("sorted", "reversed", "random", "repeats", "one", "perm")


def _list(n, rng, kind):
    if kind == "one":
        return np.array([rng.integers(0, n)], np.int64)
    if kind == "perm":
        return rng.permutation(n).astype(np.int64)
    k = int(rng.integers(1, max(2, n) + 1))
    v = rng.integers(0, n, k).astype(np.int64)
    if kind == "sorted":
        return np.unique(v)
    if kind == "reversed":
        return np.unique(v)[::-1].copy()
    if kind == "repeats":
        return np.repeat(v[: max(1, k // 2)], 2)
    return v


def _slice(n, rng):
    kind = rng.integers(0, 3)
    if kind == 0:
        return slice(0, n, 1)
    a = int(rng.integers(0, n))
    b = int(rng.integers(a + 1, n + 1))
    return slice(a, b, 1 if kind == 1 else int(rng.choice([2, 3, 7])))


def _sels(shape, rng, k):
    """k seeded selections: every dimension a list of some kind or a slice (whole, partial or stepped), at least one a
    list"""
    out = []
    for _ in range(k):
        lists = rng.random(len(shape)) < 0.5
        lists[rng.integers(0, len(shape))] = True
        out.append([_list(n, rng, LIST_KINDS[rng.integers(0, len(LIST_KINDS))]) if is_list else _slice(n, rng)
                    for n, is_list in zip(shape, lists)])
    return out


def _args(shape, sel):
    """the C call's arguments: shape, start, stop, step, the index pointer array and nindex, with the arrays to keep
    alive"""
    n = len(shape)
    sh = np.ascontiguousarray(shape, dtype=np.int64)
    st, sp, t, ni = (np.zeros(max(n, 1), np.int64) for _ in range(4))
    ptrs = (C.c_void_p * max(n, 1))()
    keep = []
    for k, s in enumerate(sel):
        if isinstance(s, slice):
            st[k], sp[k], t[k] = s.start, s.stop, s.step
        else:
            h = np.ascontiguousarray(s, dtype=np.int64)
            keep.append(h)
            ptrs[k], ni[k] = h.ctypes.data, h.size
    return sh, st, sp, t, ptrs, ni, keep


def _getoindex(lib, src_p, shape, sel, dest_p):
    sh, st, sp, t, ptrs, ni, keep = _args(shape, sel)
    return lib.blosc_b200_getoindex(src_p, len(shape), sh.ctypes.data, st.ctypes.data, sp.ctypes.data, t.ctypes.data,
                                    C.cast(ptrs, vp), ni.ctypes.data, dest_p)


def _frame_getoindex(lib, frame_p, fb, shape, sel, dest_p):
    sh, st, sp, t, ptrs, ni, keep = _args(shape, sel)
    return lib.blosc_b200_frame_getoindex(frame_p, fb, len(shape), sh.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                          t.ctypes.data, C.cast(ptrs, vp), ni.ctypes.data, dest_p)


def _check(lib, chunk, src, ts, shape, sel):
    want = _want(src, ts, shape, sel)
    out = np.full(want.size + 16, 0xAA, np.uint8)
    r = _getoindex(lib, ptr(chunk), shape, sel, ptr(out))
    assert r == want.size, (shape, sel, r, want.size)
    assert (out[:r] == want).all() and (out[r:] == 0xAA).all(), (shape, sel)
    return r


def _compress(lib, comp, clevel, shuf, ts, src, bs, monkeypatch=None, switch=None):
    if switch:
        monkeypatch.setenv(switch, "1")
    r, c = compress(lib, "blosc_compress_ctx", clevel, shuf, ts, src, len(src) + 16, comp, bs)
    assert r > 0, (comp, ts, shuf, r)
    return c[:r].copy()


# ---------------------------------------------------------------------------------------------------------------
# CPU: the emulator
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("comp,switch", CODECS)
@pytest.mark.parametrize("shuf", [0, 1, 2])
def test_getoindex_matrix_emu(olib, monkeypatch, comp, switch, shuf):
    """every codec, filter, typesize and ndim: seeded selections of lists and slices against numpy"""
    for ts, split in [(ts, NEVER_SPLIT) for ts in TYPESIZES] + [(16, FORWARD_COMPAT_SPLIT)]:
        src = gen("mixed" if ts % 2 else "i32", NITEMS * ts, seed=ts)
        olib.blosc_set_splitmode(split)
        try:
            chunk = _compress(olib, comp, 5, shuf, ts, src, 1024, monkeypatch, switch)
        finally:
            olib.blosc_set_splitmode(NEVER_SPLIT)
        for ndim, shape in SHAPES.items():
            for sel in _sels(shape, np.random.default_rng(100 * ts + ndim + shuf), 3):
                _check(olib, chunk, src, ts, shape, sel)


def test_getoindex_list_kinds_emu(olib):
    """every kind of list on the innermost and on outer dimensions, with whole, partial and stepped slices, on a
    compressed and a memcpyed chunk, typesizes 4 and 3; the memcpyed chunk of typesize 3 also with a blocksize of 1000,
    no multiple of it, so that items straddle blocks"""
    rng = np.random.default_rng(5)
    for ts, clevel, bs in ((4, 5, 0), (4, 0, 0), (3, 5, 0), (3, 0, 0), (3, 0, 1000)):
        src = gen("i32" if ts == 4 else "mixed", NITEMS * ts, seed=ts)
        chunk = _compress(olib, "lz4", clevel, 1, ts, src, 1024)
        if bs:
            chunk[8:12].view(np.int32)[0] = bs
        for dev in (0, 1):
            olib.emu_set_device_ptrs(chunk.ctypes.data if dev else None, None)
            try:
                for kind in LIST_KINDS:
                    for shape, sel in (((72, 70), [_list(72, rng, kind), slice(0, 70, 1)]),   # rows: runs of a row
                                       ((72, 70), [slice(0, 72, 1), _list(70, rng, kind)]),   # columns: one-item runs
                                       ((72, 70), [_list(72, rng, kind), _list(70, rng, kind)]),
                                       ((72, 70), [slice(3, 60, 5), _list(70, rng, kind)]),
                                       ((14, 18, 20), [_list(14, rng, kind), slice(2, 9, 1), slice(0, 20, 1)]),
                                       ((14, 18, 20), [slice(0, 14, 1), slice(0, 18, 1), _list(20, rng, kind)]),
                                       ((14, 18, 20), [slice(1, 14, 3), _list(18, rng, kind), slice(0, 20, 2)]),
                                       ((NITEMS,), [_list(NITEMS, rng, kind)])):
                        _check(olib, chunk, src, ts, shape, sel)
            finally:
                olib.emu_set_device_ptrs(None, None)


@pytest.mark.parametrize("clevel", [5, 0])
@pytest.mark.parametrize("place", ["hhh", "dhh", "hdh", "hhd", "ddh", "dhd", "ddd"])
def test_getoindex_placements_emu(olib, clevel, place):
    """src, dest and the lists (place: their memory, h / d, in that order) in host and device memory; a memcpyed
    chunk in device memory is read in place after the list check alone"""
    ts, shape = 4, (14, 18, 20)
    src = gen("i32", NITEMS * ts, seed=7)
    chunk = _compress(olib, "lz4", clevel, 1, ts, src, 1024)
    rng = np.random.default_rng(clevel + 3 * len(place) + sum(ord(c) for c in place))
    sels = [[s if isinstance(s, slice) or k == min(k for k, x in enumerate(sel) if not isinstance(x, slice))
             else slice(0, n, 1) for k, (s, n) in enumerate(zip(sel, shape))] for sel in _sels(shape, rng, 4)]
    for sel in sels + [[np.array([13, 0, 5], np.int64), slice(0, 18, 1), slice(0, 20, 1)]]:   # one list each
        want = _want(src, ts, shape, sel)
        out = np.full(want.size + 16, 0xAA, np.uint8)
        sh, st, sp, t, ptrs, ni, keep = _args(shape, sel)
        devs = ([chunk.ctypes.data] if place[0] == "d" else []) + ([out.ctypes.data] if place[1] == "d" else []) + \
            ([keep[0].ctypes.data] if place[2] == "d" else [])
        if place == "ddd":
            olib.emu_set_all_device(1)
        else:
            olib.emu_set_device_ptrs(*(devs + [None, None])[:2])
        try:
            before = olib.emu_all_launches()
            r = olib.blosc_b200_getoindex(ptr(chunk), 3, sh.ctypes.data, st.ctypes.data, sp.ctypes.data, t.ctypes.data,
                                          C.cast(ptrs, vp), ni.ctypes.data, ptr(out))
            grown = olib.emu_all_launches() - before
        finally:
            olib.emu_set_device_ptrs(None, None)
            olib.emu_set_all_device(0)
        assert r == want.size and (out[:r] == want).all() and (out[r:] == 0xAA).all(), (place, sel)
        # a compressed chunk: touch, slot scan, decode, unfilter, gather; a memcpyed one: no decode; in place: the
        # check and the gather
        assert grown == (5 if clevel else 2 if place[0] == "d" else 3), (place, grown)


def test_getoindex_decodes_touched_blocks_emu(olib):
    """the decode launch lists exactly the blocks that hold a byte of a selected item"""
    for ts, shape in ((4, (72, 70)), (3, (7, 8, 9, 10)), (16, (14, 18, 20)), (4, (NITEMS,))):
        src = gen("mixed" if ts == 3 else "i32", NITEMS * ts, seed=ts)
        chunk = _compress(olib, "lz4", 5, 1, ts, src, 1024)
        bs = int(chunk[8:12].view(np.int32)[0])
        assert not chunk[2] & 0x2
        rng = np.random.default_rng(ts + len(shape))
        sels = _sels(shape, rng, 6)
        sels.append([np.array([shape[0] - 1, 0], np.int64)] + [slice(0, n, 1) for n in shape[1:]])
        for sel in sels:
            _check(olib, chunk, src, ts, shape, sel)
            assert olib.emu_last_decode_blocks() == _touched(shape, sel, ts, bs), sel


def test_getoindex_launches_emu(olib):
    """lists of 1 and of 10^4 entries (and a 10^4 x 2 selection of one-item runs) make the same five launches, the
    same read-backs and the same syncs"""
    src = bench_words(80000)
    chunk = _compress(olib, "lz4", 5, 1, 4, src, 4096)
    assert not chunk[2] & 0x2
    rng = np.random.default_rng(1)
    counts = []
    for shape, sel in (((1000, 20), [np.array([5], np.int64), slice(0, 20, 1)]),
                       ((20000,), [rng.integers(0, 20000, 10000).astype(np.int64)]),
                       ((1000, 20), [rng.integers(0, 1000, 10000).astype(np.int64), slice(0, 20, 1)]),
                       ((10000, 2), [slice(0, 10000, 1), np.array([1, 0], np.int64)])):
        before = (olib.emu_all_launches(), olib.emu_d2h_copies(), olib.emu_syncs())
        _check(olib, chunk, src, 4, shape, sel)
        counts.append((olib.emu_all_launches() - before[0], olib.emu_d2h_copies() - before[1],
                       olib.emu_syncs() - before[2]))
    assert counts[0][0] == 5 and len(set(counts)) == 1, counts   # touch, slot scan, decode, unfilter, gather


def test_getoindex_slices_only_emu(olib):
    """index == NULL and all-NULL lists give getslice_step's bytes through getslice_step's kernels"""
    ts, shape = 4, (14, 18, 20)
    src = gen("i32", NITEMS * ts, seed=11)
    chunk = _compress(olib, "lz4", 5, 1, ts, src, 1024)
    for start, stop, step in (((0, 0, 0), (14, 18, 20), (1, 1, 1)), ((2, 3, 1), (13, 17, 20), (3, 1, 2)),
                              ((1, 0, 5), (2, 18, 20), (1, 1, 1))):
        sel = [slice(a, b, c) for a, b, c in zip(start, stop, step)]
        want = _want(src, ts, shape, sel)
        sh, st, sp, t = (np.ascontiguousarray(v, dtype=np.int64) for v in (shape, start, stop, step))
        nulls = (C.c_void_p * 3)()
        outs, launches = [], []
        for call in ("step", "null", "nulls"):
            out = np.full(want.size + 16, 0xAA, np.uint8)
            olib.emu_oindex_reset()
            before = olib.emu_all_launches()
            if call == "step":
                r = olib.blosc_b200_getslice_step(ptr(chunk), 3, sh.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                                  t.ctypes.data, ptr(out))
            else:
                r = olib.blosc_b200_getoindex(ptr(chunk), 3, sh.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                              t.ctypes.data, None if call == "null" else C.cast(nulls, vp), None,
                                              ptr(out))
            launches.append(olib.emu_all_launches() - before)
            assert r == want.size and olib.emu_oindex_ngathers() == 0, call
            assert olib.emu_last_box_stepped() == (max(step) > 1 and start[0] + 1 != stop[0]), call
            outs.append(out)
        assert (outs[0][:want.size] == want).all() and all((o == outs[0]).all() for o in outs)
        assert launches == [5, 5, 5], launches


def test_getoindex_rejects_emu(olib, capfd):
    ts = 4
    src = gen("i32", NITEMS * ts, seed=2)
    chunk = _compress(olib, "lz4", 5, 1, ts, src, 1024)
    out = np.full(64, 0xAA, np.uint8)
    capfd.readouterr()
    good = np.array([1, 2], np.int64)
    # the list entries, checked on the GPU by the planning launch: the first bad (k, position) is named
    for sel, msg in (([np.array([1, 72, 3], np.int64), slice(0, 2, 1)], "index[0][1] = 72"),
                     ([np.array([1, 2, -1], np.int64), slice(0, 2, 1)], "index[0][2] = -1"),
                     ([good, np.array([0, 70, -5, 99], np.int64)], "index[1][1] = 70"),
                     ([np.array([9, 80, 1, -3], np.int64), np.array([-1], np.int64)], "index[0][1] = 80"),
                     ([slice(0, 3, 1), np.array([0, 1, 2, 3, 4, 5, 1 << 40], np.int64)], "index[1][6] = 1099511627776")):
        before = olib.emu_all_launches()
        r = _getoindex(olib, ptr(chunk), (72, 70), sel, ptr(out))
        err = capfd.readouterr().err
        assert r == -1 and (out == 0xAA).all() and olib.emu_all_launches() - before == 2, (sel, r)   # touch + scan
        assert err.count("blosc_b200") == 1 and msg in err, err
    # before anything is launched: getslice_step's geometry checks on the slice dimensions, nindex < 0, overflow
    for shape, sel, msg in (
            ((72, 70), [good, slice(0, 3, 0)], "step[1] = 0"), ((72, 70), [good, slice(5, 3, 1)], "inside"),
            ((72, 70), [good, slice(0, 71, 1)], "inside"), ((72, 71), [good, slice(0, 3, 1)], "items"),
            ((-72, -70), [good, slice(0, 1, 1)], "negative"), ((1 << 40, 1 << 40), [good, slice(0, 1, 1)], "overflows"),
            ((1,) * 8 + (5040,), [good] + [slice(0, 1, 1)] * 8, "ndim")):
        before = olib.emu_all_launches()
        r = _getoindex(olib, ptr(chunk), shape, sel, ptr(out))
        err = capfd.readouterr().err
        assert r == -1 and (out == 0xAA).all() and olib.emu_all_launches() == before, (shape, sel, r)
        assert err.count("blosc_b200") == 1 and msg in err, (shape, err)
    sh, st, sp, t, ptrs, ni, keep = _args((72, 70), [good, slice(0, 3, 1)])
    ni[0] = -1
    r = olib.blosc_b200_getoindex(ptr(chunk), 2, sh.ctypes.data, st.ctypes.data, sp.ctypes.data, t.ctypes.data,
                                  C.cast(ptrs, vp), ni.ctypes.data, ptr(out))
    assert r == -1 and "nindex[0] = -1" in capfd.readouterr().err and (out == 0xAA).all()
    # an output of 2^62 items of 4 bytes: the list lengths are checked, never read
    sh, st, sp, t, ptrs, ni, keep = _args((72, 70), [good, good])
    ni[0], ni[1] = 1 << 31, 1 << 31
    before = olib.emu_all_launches()
    r = olib.blosc_b200_getoindex(ptr(chunk), 2, sh.ctypes.data, st.ctypes.data, sp.ctypes.data, t.ctypes.data,
                                  C.cast(ptrs, vp), ni.ctypes.data, ptr(out))
    err = capfd.readouterr().err
    assert r == -1 and "overflow" in err and olib.emu_all_launches() == before and (out == 0xAA).all(), err
    # the header codes of getslice
    for patch, code in ((lambda h: h.__setitem__(0, 3), -9), (lambda h: h.__setitem__(2, (h[2] & 0x1f) | (6 << 5)), -5)):
        h = chunk.copy()
        patch(h)
        assert _getoindex(olib, ptr(h), (72, 70), [good, slice(0, 7, 3)], ptr(out)) == code and (out == 0xAA).all()


def test_getoindex_empty_emu(olib):
    """an empty list, or an empty slice next to a list, returns 0 with nothing launched and no list read"""
    ts = 4
    src = gen("i32", NITEMS * ts, seed=2)
    chunk = _compress(olib, "lz4", 5, 1, ts, src, 1024)
    out = np.full(64, 0xAA, np.uint8)
    for sel in ([np.zeros(0, np.int64), slice(0, 70, 1)], [np.array([1, 99], np.int64), slice(5, 5, 1)],
                [np.array([-1], np.int64), np.zeros(0, np.int64)]):
        before = (olib.emu_all_launches(), olib.emu_d2h_copies())
        assert _getoindex(olib, ptr(chunk), (72, 70), sel, ptr(out)) == 0
        assert (olib.emu_all_launches(), olib.emu_d2h_copies()) == before and (out == 0xAA).all()


def test_getoindex_damaged_block_emu(olib):
    """a damaged block that no selected item touches is not read; one that one touches gives blosc_d's code, dest
    untouched"""
    ts, shape = 4, (72, 70)
    src = gen("i32", NITEMS * ts, seed=3)
    chunk = _compress(olib, "lz4", 5, 1, ts, src, 1024)
    bs = int(chunk[8:12].view(np.int32)[0])
    h = chunk.copy()
    h[16 + 4 * 5:16 + 4 * 6].view(np.int32)[0] = 0x7fff0000      # block 5's bstarts entry
    rows = sorted({(f * ts) // bs for f in range(NITEMS)} - {5})
    bad_row = (5 * bs // ts) // 70                               # a row with an item in block 5
    clean = [r for r in range(72) if all(((r * 70 + c) * ts) // bs != 5 and ((r * 70 + c) * ts + 3) // bs != 5
                                         for c in range(70))]
    assert rows and bad_row not in clean
    for src_dev in (0, 1):
        olib.emu_set_device_ptrs(h.ctypes.data if src_dev else None, None)
        try:
            code = olib.blosc_getitem(ptr(h), ci(5 * bs // ts), ci(1), ptr(np.zeros(64, np.uint8)))
            assert code < 0
            _check(olib, h, src, ts, shape, [np.array(clean[::-3], np.int64), slice(0, 70, 1)])
            out = np.full(8192, 0xAA, np.uint8)
            sel = [np.array([clean[0], bad_row], np.int64), slice(0, 70, 2)]
            assert _getoindex(olib, ptr(h), shape, sel, ptr(out)) == code and (out == 0xAA).all()
        finally:
            olib.emu_set_device_ptrs(None, None)


def _frame(lib, src, ts, chunksize, clevel=5):
    fb = lib.blosc_b200_frame_bound(len(src), ts, chunksize)
    frame = np.zeros(fb, np.uint8)
    r = lib.blosc_b200_frame_compress(clevel, 1, ts, len(src), ptr(src), ptr(frame), fb, b"lz4", 1024, chunksize, 1)
    assert r > 0
    return frame[:r].copy()


def _check_frame(lib, frame, src, ts, shape, sel):
    want = _want(src, ts, shape, sel)
    out = np.full(want.size + 16, 0xAA, np.uint8)
    r = _frame_getoindex(lib, frame.ctypes.data, len(frame), shape, sel, out.ctypes.data)
    assert r == want.size and (out[:r] == want).all() and (out[r:] == 0xAA).all(), (shape, sel, r)


@pytest.mark.parametrize("dev", [0, 1])
@pytest.mark.parametrize("clevel", [5, 0])
def test_frame_getoindex_emu(olib, dev, clevel):
    """selections across chunk boundaries, a chunksize that is no multiple of the row, a short last chunk"""
    ts, shape = 4, (50, 37)
    src = gen("i32", 50 * 37 * ts, seed=5)
    frame = _frame(olib, src, ts, 1000, clevel)                   # 250 items a chunk, 8 chunks, the last of 100
    olib.emu_set_all_device(dev)
    try:
        rng = np.random.default_rng(dev + 7 + clevel)
        sels = _sels(shape, rng, 8) + [[np.array([49, 0, 6, 6, 27], np.int64), slice(0, 37, 1)],
                                       [slice(0, 50, 1), np.array([36, 0, 18], np.int64)],
                                       [slice(3, 50, 7), np.array([5], np.int64)],
                                       [rng.permutation(50), rng.permutation(37)]]
        for sel in sels:
            _check_frame(olib, frame, src, ts, shape, sel)
        for sel in _sels((10, 5, 37), np.random.default_rng(19), 4):
            _check_frame(olib, frame, src, ts, (10, 5, 37), sel)
        _check_frame(olib, frame, src, ts, (1850,), [rng.integers(0, 1850, 300)])
    finally:
        olib.emu_set_all_device(0)


def test_frame_getoindex_skips_chunks_emu(olib, capfd):
    """chunks that hold no selected item are neither read nor decoded: a damaged one leaves the read intact; a damaged
    touched one decides the result, the first in ascending order, with a host dest untouched"""
    ts, shape = 4, (50, 37)
    src = gen("i32", 50 * 37 * ts, seed=6)
    frame = _frame(olib, src, ts, 1000)                           # chunk c holds items [250 c, 250 c + 250)
    off = [olib.blosc_b200_frame_chunk(frame.ctypes.data, len(frame), i, None) for i in range(8)]
    # rows 40, 0, 20: items [1480, 1517), [0, 37), [740, 777) in chunks 5 and 6, 0, 2 and 3
    olib.emu_oindex_reset()
    _check_frame(olib, frame, src, ts, shape, [np.array([40, 0, 20], np.int64), slice(0, 37, 1)])
    assert [olib.emu_oindex_window(i) for i in range(olib.emu_oindex_ngathers())] == [0, 500, 750, 1250, 1500]
    for patch, code in ((lambda f: f.__setitem__(off[2] + 3, 2), -1), (lambda f: f.__setitem__(off[2], 3), -9)):
        f = frame.copy()
        patch(f)
        g = f.copy()
        patch2 = lambda x: x.__setitem__(off[5], 3)               # noqa: E731 -- a later damaged chunk
        patch2(g)
        for dev in (0, 1):
            olib.emu_set_all_device(dev)
            try:
                for buf in (f, g):                                # the first damaged chunk decides: chunk 2's code
                    out = np.full(3 * 37 * ts + 16, 0xAA, np.uint8)
                    capfd.readouterr()
                    r = _frame_getoindex(olib, buf.ctypes.data, len(buf), shape,
                                         [np.array([40, 0, 20], np.int64), slice(0, 37, 1)], out.ctypes.data)
                    assert r == code and (dev or (out == 0xAA).all()), (code, r)
                    if code == -1:
                        assert "blosc_b200" in capfd.readouterr().err
                _check_frame(olib, f, src, ts, shape, [np.array([27, 0], np.int64), slice(0, 37, 1)])  # chunks 0, 3, 4
                _check_frame(olib, f, src, ts, (1850,), [np.array([1500, 0, 750], np.int64)])         # chunks 6, 0, 3
            finally:
                olib.emu_set_all_device(0)
    # a bad entry: one message, nothing gathered
    olib.emu_oindex_reset()
    out = np.full(64, 0xAA, np.uint8)
    capfd.readouterr()
    r = _frame_getoindex(olib, frame.ctypes.data, len(frame), shape, [np.array([1, 50, 51], np.int64), slice(0, 3, 1)],
                         out.ctypes.data)
    err = capfd.readouterr().err
    assert r == -1 and "index[0][1] = 50" in err and err.count("blosc_b200") == 1 and (out == 0xAA).all()
    assert olib.emu_oindex_ngathers() == 0


# ---------------------------------------------------------------------------------------------------------------
# GPU: the CUDA library
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def glib(pkg):
    return _bind(pkg.lib)


def _torch_sel(torch, sel, kind):
    """the selection with its lists as host int64 arrays (kind "h") or int64 CUDA tensors ("d")"""
    return [s if isinstance(s, slice) or kind == "h" else torch.from_numpy(s).cuda() for s in sel]


def _gpu_check(pkg, torch, chunk_h, chunk_d, src, ts, shape, sel):
    want = _want(src, ts, shape, sel)
    for s_buf in (chunk_h, chunk_d):
        for kind in ("h", "d"):
            for dest_dev in (False, True):
                out = torch.full((want.size + 16,), 0xAA, dtype=torch.uint8, device="cuda") if dest_dev else \
                    np.full(want.size + 16, 0xAA, np.uint8)
                r = pkg.getoindex(s_buf, shape, _torch_sel(torch, sel, kind), out)
                got = out.cpu().numpy() if dest_dev else out
                assert r == want.size and (got[:r] == want).all() and (got[r:] == 0xAA).all(), (shape, sel, kind, r)


@pytest.mark.gpu
@pytest.mark.parametrize("comp,switch", (("blosclz", None), ("lz4", None), ("zstd", "BLOSC_B200_ZSTD")))
@pytest.mark.parametrize("shuf", [0, 1, 2])
def test_getoindex_matrix_gpu(pkg, glib, cuda, monkeypatch, comp, switch, shuf):
    """seeded selections against numpy, typesizes 1, 4, 3 and 16, every placement of data, dest and lists"""
    torch = cuda
    n = 1 << 18
    shapes = {1: (n,), 2: (512, 512), 3: (64, 64, 64), 8: (4, 4, 4, 4, 4, 4, 8, 8)}
    for i, ts in enumerate((1, 4, 3, 16)):
        src = (gen("mixed", n * ts, seed=ts) if i % 2 else bench_words(n * ts))
        for bs in (0, 16384):
            chunk = _compress(glib, comp, 5, shuf, ts, src, bs, monkeypatch, switch)
            d_chunk = torch.from_numpy(chunk).cuda()
            for ndim, shape in shapes.items():
                for sel in _sels(shape, np.random.default_rng(ts + ndim + bs), 2):
                    _gpu_check(pkg, torch, chunk, d_chunk, src, ts, shape, sel)


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
def test_getoindex_big_chunk_gpu(pkg, cuda, big):
    """8192 x 8192 float32: torch.randperm / torch.randint rows and columns on the device, and a bool mask, against
    torch advanced indexing, into a device and a host dest, in five launches"""
    torch = cuda
    src, d_chunk = big
    a = src.view(torch.float32).view(8192, 8192)
    g = torch.Generator(device="cuda").manual_seed(1)
    rows = torch.randperm(8192, device="cuda", generator=g)[:1024]
    cols = torch.randint(0, 8192, (256,), device="cuda", generator=g)
    mask = torch.rand(8192, device="cuda", generator=g) < 0.01
    for sel, want in (([rows, slice(None)], a[rows]), ([rows.sort().values, slice(None)], a[rows.sort().values]),
                      ([slice(None), cols], a[:, cols]), ([rows[:512], cols], a[rows[:512]][:, cols]),
                      ([mask, slice(100, 9000, 3)], a[mask][:, 100::3]), ([17, cols], a[17, cols])):
        want = want.contiguous().view(torch.uint8).view(-1)
        for dest_dev in (True, False):
            out = torch.full((want.numel() + 16,), 0xAA, dtype=torch.uint8, device="cuda" if dest_dev else "cpu")
            before = pkg.launch_count()
            assert pkg.getoindex(d_chunk, (8192, 8192), sel, out) == want.numel()
            if dest_dev:
                assert pkg.launch_count() - before == 5
            assert torch.equal(out[:want.numel()].cuda(), want) and bool((out[want.numel():] == 0xAA).all())
    flat = src.view(torch.float32)
    idx = torch.randint(0, 1 << 26, (100000,), device="cuda", generator=g)
    out = torch.empty(400000, dtype=torch.uint8, device="cuda")
    assert pkg.getoindex(d_chunk, (1 << 26,), [idx], out) == 400000
    assert torch.equal(out, flat[idx].view(torch.uint8))
    host_src = d_chunk.cpu().pin_memory()
    out.fill_(0)
    assert pkg.getoindex(host_src, (1 << 26,), [idx.cpu().numpy()], out) == 400000
    assert torch.equal(out, flat[idx].view(torch.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize("frame_dev", [False, True])
def test_frame_getoindex_gpu(pkg, glib, cuda, frame_dev):
    """a 12-chunk frame in device and host memory: device and host lists across chunk boundaries"""
    torch = cuda
    ts, shape = 4, (3000, 1001)
    src = bench_words(3000 * 1001 * ts)
    frame = _frame(glib, src, ts, 1 << 20)                        # 262144 items a chunk: 12 chunks, the last one short
    f_buf = torch.from_numpy(frame).cuda() if frame_dev else frame
    rng = np.random.default_rng(3)
    sels = _sels(shape, rng, 4) + [[rng.permutation(3000)[:700], slice(0, 1001, 1)],
                                   [slice(0, 3000, 1), rng.integers(0, 1001, 64)],
                                   [rng.integers(0, 3000, 300), rng.integers(0, 1001, 200)],
                                   [slice(5, 3000, 261), np.array([1000, 0, 500])]]
    for sel in sels:
        want = _want(src, ts, shape, sel)
        for kind in ("h", "d"):
            for dest_dev in (False, True):
                out = torch.full((want.size + 16,), 0xAA, dtype=torch.uint8, device="cuda") if dest_dev else \
                    np.full(want.size + 16, 0xAA, np.uint8)
                assert pkg.frame_getoindex(f_buf, len(frame), shape, _torch_sel(torch, sel, kind), out) == want.size
                got = out.cpu().numpy() if dest_dev else out
                assert (got[:want.size] == want).all() and (got[want.size:] == 0xAA).all(), (sel, kind)


@pytest.mark.gpu
def test_getoindex_python_args_gpu(pkg, cuda):
    """ints, bool masks, None slice fields; int32 CUDA lists raise TypeError, negative slice fields ValueError; a bad
    entry returns -1 with dest untouched"""
    torch = cuda
    src = bench_words(4096 * 4)
    d_chunk = torch.from_numpy(_compress(pkg.lib, "lz4", 5, 1, 4, src, 0)).cuda()
    a = torch.from_numpy(src).cuda().view(torch.int32).view(64, 64)
    out = torch.full((4096 * 4,), 0xAA, dtype=torch.uint8, device="cuda")
    with pytest.raises(TypeError):
        pkg.getoindex(d_chunk, (64, 64), [torch.tensor([1, 2], dtype=torch.int32, device="cuda"), slice(None)], out)
    with pytest.raises(ValueError):
        pkg.getoindex(d_chunk, (64, 64), [[1, 2], slice(-3, None)], out)
    with pytest.raises(ValueError):
        pkg.getoindex(d_chunk, (64, 64), [[1, 2]], out)
    mask = torch.arange(64, device="cuda") % 5 == 1
    for sel, want in (([mask, 3], a[mask, 3]), ([[5, 1, 5], slice(None, None, 9)], a[[5, 1, 5]][:, ::9]),
                      ([np.array([True] * 64), [63]], a[:, [63]]), ([slice(2, None), torch.tensor([7], device="cuda")],
                                                                   a[2:, [7]]), ([4, slice(None)], a[4])):
        want = want.contiguous().view(torch.uint8).view(-1)
        assert pkg.getoindex(d_chunk, (64, 64), sel, out) == want.numel()
        assert torch.equal(out[:want.numel()], want)
    out.fill_(0xAA)
    assert pkg.getoindex(d_chunk, (64, 64), [torch.tensor([3, 64], device="cuda"), slice(None)], out) == -1
    assert bool((out == 0xAA).all())
    assert pkg.getoindex(d_chunk, (64, 64), [[], slice(None)], out) == 0


@pytest.mark.gpu
def test_getoindex_other_device_gpu(pkg, cuda):
    """a list on another device than the call's returns -1 before anything is read"""
    torch = cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    src = bench_words(4096 * 4)
    d_chunk = torch.from_numpy(_compress(pkg.lib, "lz4", 5, 1, 4, src, 0)).cuda(0)
    out = torch.full((4096 * 4,), 0xAA, dtype=torch.uint8, device="cuda:0")
    idx = torch.tensor([1, 2], device="cuda:1")
    assert pkg.getoindex(d_chunk, (64, 64), [idx, slice(None)], out) == -1
    assert bool((out == 0xAA).all())

"""c-blosc_b200 -- Python host-side mirror of the c-blosc C API over libblosc_b200.so.

The product is the C-ABI shared library (``include/blosc_b200.h``,
``c-blosc_b200/csrc``); this module is a thin ctypes binding that keeps the reference's
names, argument order and return codes (reference ``blosc/blosc.h:221-312``) so tests read
like the reference's own.  Buffers may be ``bytes``/``bytearray``/numpy arrays (host
pointers) or torch CUDA tensors (device pointers); the library tells them apart itself.

The directory name contains a hyphen (it is the name the build contract asks for), so it
is loaded with importlib under the module name ``cblosc_b200`` -- see
``__graft_entry__.load_package()``.

There is deliberately no fallback: if the CUDA library is missing this import raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libblosc_b200.so")

BLOSC_NOSHUFFLE, BLOSC_SHUFFLE, BLOSC_BITSHUFFLE = 0, 1, 2
BLOSC_MAX_OVERHEAD = 16
FILT_SHUFFLE, FILT_UNSHUFFLE, FILT_BITSHUFFLE, FILT_BITUNSHUFFLE = 0, 1, 2, 3
KERNEL_KINDS = ("filter", "encode", "scan", "compact", "decode", "unfilter", "index", "parse", "zenc", "denc", "senc",
                "gather", "plan")
HAS_FAST_PARSE = True      # BLOSC_B200_PARSE=fast: segment-parallel LZ4 parse (csrc/dev_lz4fast.cuh)


def _load(path: str) -> C.CDLL:
    if not os.path.exists(path):
        raise ImportError(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  c-blosc_b200 has no CPU fallback.")
    lib = C.CDLL(path)
    vp, sz, ci = C.c_void_p, C.c_size_t, C.c_int
    lib.blosc_compress_ctx.restype = ci
    lib.blosc_compress_ctx.argtypes = [ci, ci, sz, sz, vp, vp, sz, C.c_char_p, sz, ci]
    lib.blosc_decompress_ctx.restype = ci
    lib.blosc_decompress_ctx.argtypes = [vp, vp, sz, ci]
    lib.blosc_getitem.restype = ci
    lib.blosc_getitem.argtypes = [vp, ci, ci, vp]
    lib.blosc_compress.restype = ci
    lib.blosc_compress.argtypes = [ci, ci, sz, sz, vp, vp, sz]
    lib.blosc_decompress.restype = ci
    lib.blosc_decompress.argtypes = [vp, vp, sz]
    lib.blosc_b200_filter.restype = ci
    lib.blosc_b200_filter.argtypes = [ci, sz, sz, vp, vp]
    lib.blosc_b200_set_profiling.argtypes = [ci]
    lib.blosc_b200_prof_get.argtypes = [ci, C.POINTER(C.c_double), C.POINTER(C.c_longlong)]
    lib.blosc_b200_launch_count.restype = C.c_longlong
    lib.blosc_set_compressor.argtypes = [C.c_char_p]
    lib.blosc_set_splitmode.argtypes = [ci]
    lib.blosc_set_blocksize.argtypes = [sz]
    lib.blosc_cbuffer_sizes.argtypes = [vp, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
    ll = C.c_longlong
    lib.blosc_b200_frame_bound.restype = sz
    lib.blosc_b200_frame_bound.argtypes = [sz, sz, sz]
    lib.blosc_b200_frame_compress.restype = ll
    lib.blosc_b200_frame_compress.argtypes = [ci, ci, sz, sz, vp, vp, sz, C.c_char_p, sz, sz, ci]
    lib.blosc_b200_frame_decompress.restype = ll
    lib.blosc_b200_frame_decompress.argtypes = [vp, sz, vp, sz, ci]
    lib.blosc_b200_frame_getitem.restype = ll
    lib.blosc_b200_frame_getitem.argtypes = [vp, sz, sz, sz, vp]
    lib.blosc_b200_getitems.restype = ll
    lib.blosc_b200_getitems.argtypes = [vp, ci, vp, vp, vp]
    lib.blosc_b200_frame_getitems.restype = ll
    lib.blosc_b200_frame_getitems.argtypes = [vp, sz, sz, vp, vp, vp]
    lib.blosc_b200_getslice.restype = ll
    lib.blosc_b200_getslice.argtypes = [vp, ci, vp, vp, vp, vp]
    lib.blosc_b200_frame_getslice.restype = ll
    lib.blosc_b200_frame_getslice.argtypes = [vp, sz, ci, vp, vp, vp, vp]
    lib.blosc_b200_getslice_step.restype = ll
    lib.blosc_b200_getslice_step.argtypes = [vp, ci, vp, vp, vp, vp, vp]
    lib.blosc_b200_frame_getslice_step.restype = ll
    lib.blosc_b200_frame_getslice_step.argtypes = [vp, sz, ci, vp, vp, vp, vp, vp]
    lib.blosc_b200_getslices.restype = ll
    lib.blosc_b200_getslices.argtypes = [vp, ci, vp, vp, ll, vp, vp]
    lib.blosc_b200_frame_getslices.restype = ll
    lib.blosc_b200_frame_getslices.argtypes = [vp, sz, ci, vp, vp, ll, vp, vp]
    lib.blosc_b200_getoindex.restype = ll
    lib.blosc_b200_getoindex.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, vp]
    lib.blosc_b200_frame_getoindex.restype = ll
    lib.blosc_b200_frame_getoindex.argtypes = [vp, sz, ci, vp, vp, vp, vp, vp, vp, vp]
    lib.blosc_b200_grid_getslice.restype = ll
    lib.blosc_b200_grid_getslice.argtypes = [ci, vp, vp, sz, vp, vp, vp, vp, vp, vp]
    lib.blosc_b200_grid_bound.restype = sz
    lib.blosc_b200_grid_bound.argtypes = [ci, vp, vp, sz]
    lib.blosc_b200_grid_compress.restype = ll
    lib.blosc_b200_grid_compress.argtypes = [ci, ci, sz, C.c_char_p, sz, ci, ci, vp, vp, sz, vp, vp, ci, vp, sz, vp]
    lib.blosc_b200_frame_info.restype = ci
    lib.blosc_b200_frame_info.argtypes = [vp, sz, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
    lib.blosc_b200_frame_chunk.restype = ll
    lib.blosc_b200_frame_chunk.argtypes = [vp, sz, sz, C.POINTER(sz)]
    return lib


lib = _load(os.environ.get("BLOSC_B200_LIB", LIB_PATH))


def _ptr(buf):
    """Raw address of a host buffer (bytes-like / numpy) or a torch tensor (host or CUDA)."""
    if buf is None:
        return None
    if isinstance(buf, int):
        return buf
    if hasattr(buf, "data_ptr"):            # torch.Tensor
        return buf.data_ptr()
    if hasattr(buf, "ctypes"):              # numpy
        return buf.ctypes.data
    if isinstance(buf, bytes):              # points into the bytes object; caller keeps it alive
        return C.cast(C.c_char_p(buf), C.c_void_p).value
    if isinstance(buf, bytearray):
        return C.addressof((C.c_char * len(buf)).from_buffer(buf))
    raise TypeError(f"unsupported buffer type {type(buf)}")


def compress_ctx(clevel, doshuffle, typesize, nbytes, src, dest, destsize, compressor, blocksize=0, numinternalthreads=1):
    """blosc_compress_ctx (reference blosc.h:245-248)."""
    return lib.blosc_compress_ctx(clevel, doshuffle, typesize, nbytes, _ptr(src), _ptr(dest), destsize,
                                  compressor.encode() if isinstance(compressor, str) else compressor,
                                  blocksize, numinternalthreads)


def decompress_ctx(src, dest, destsize, numinternalthreads=1):
    """blosc_decompress_ctx (reference blosc.h:301-302)."""
    return lib.blosc_decompress_ctx(_ptr(src), _ptr(dest), destsize, numinternalthreads)


def getitem(src, start, nitems, dest):
    """blosc_getitem (reference blosc.h:312)."""
    return lib.blosc_getitem(_ptr(src), start, nitems, _ptr(dest))


def _is_cuda(a):
    return getattr(a, "is_cuda", False)


def _range_list(a, dtype, cuda_dtypes):
    """One range list as (array or tensor to keep alive, its address, its length).  A CUDA tensor stays on its device
    (made contiguous there) and must already have one of `cuda_dtypes`: a cast on the device could silently truncate.
    Sequences and numpy arrays become C-contiguous host arrays of `dtype`."""
    if _is_cuda(a):
        if str(a.dtype) not in cuda_dtypes:
            raise TypeError(f"CUDA range lists must be {' or '.join(cuda_dtypes)}, not {a.dtype}")
        t = a.contiguous().reshape(-1)
        return t, t.data_ptr(), t.numel()
    import numpy as np
    h = np.ascontiguousarray(a, dtype=dtype).reshape(-1)
    return h, h.ctypes.data, h.size


def _ranges(starts, nitems, dtype, cuda_dtypes):
    """starts / nitems (sequences, numpy arrays or CUDA tensors) as two lists checked to have one length"""
    st, n = _range_list(starts, dtype, cuda_dtypes), _range_list(nitems, dtype, cuda_dtypes)
    if st[2] != n[2]:
        raise ValueError(f"{st[2]} starts but {n[2]} counts")
    return st, n


def getitems(src, starts, nitems, dest):
    """Many item ranges of one chunk in one call (blosc_b200_getitems): range r is items
    [starts[r], starts[r] + nitems[r]); they land back to back in `dest`, in request order.  Returns the bytes
    written, or blosc_getitem's code for the first bad range (dest is then untouched).  starts / nitems may be
    int32 CUDA tensors, on the device of the call: the read is then planned on the GPU."""
    st, n = _ranges(starts, nitems, "int32", ("torch.int32",))
    return int(lib.blosc_b200_getitems(_ptr(src), st[2], st[1], n[1], _ptr(dest)))


def _box(shape, start, stop):
    """shape / start / stop (sequences of ints) as three int64 host arrays of one length"""
    import numpy as np
    g = [np.ascontiguousarray(v, dtype=np.int64).reshape(-1) for v in (shape, start, stop)]
    if not g[0].size == g[1].size == g[2].size:
        raise ValueError(f"shape, start and stop have {g[0].size}, {g[1].size} and {g[2].size} entries")
    return g


def _step(sh, step):
    """step as an int64 host array of the shape's length"""
    import numpy as np
    t = np.ascontiguousarray(step, dtype=np.int64).reshape(-1)
    if t.size != sh.size:
        raise ValueError(f"shape and step have {sh.size} and {t.size} entries")
    return t


def getslice(src, shape, start, stop, dest, step=None):
    """A box of the C-order array of `shape` that the chunk holds (blosc_b200_getslice): items [start[k], stop[k]) of
    each dimension, written to `dest` as one contiguous C-order array.  With `step` (one positive int per dimension),
    every step[k]-th of them (blosc_b200_getslice_step): numpy's a[start:stop:step], made contiguous.  Returns the bytes
    written, or a negative code (dest is then untouched)."""
    sh, st, sp = _box(shape, start, stop)
    if step is None:
        return int(lib.blosc_b200_getslice(_ptr(src), sh.size, sh.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                           _ptr(dest)))
    t = _step(sh, step)
    return int(lib.blosc_b200_getslice_step(_ptr(src), sh.size, sh.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                            t.ctypes.data, _ptr(dest)))


def _boxes(shape, extent, starts):
    """shape / extent as two int64 host arrays of one length, and the corners as (array or tensor to keep alive, its
    address, their number); `starts` has shape (K, ndim)"""
    import numpy as np
    sh, ex = (np.ascontiguousarray(v, dtype=np.int64).reshape(-1) for v in (shape, extent))
    if sh.size != ex.size:
        raise ValueError(f"shape and extent have {sh.size} and {ex.size} entries")
    dims = tuple(starts.shape) if hasattr(starts, "shape") else np.shape(starts)
    if dims == (0,):                                    # an empty sequence: no boxes
        dims = (0, sh.size)
    if len(dims) != 2 or dims[1] != sh.size:
        raise ValueError(f"starts must have shape (K, {sh.size}), not {dims}")
    st = _range_list(starts, "int64", ("torch.int64",))
    return sh, ex, (st[0], st[1], dims[0])


def getslices(src, shape, extent, starts, dest):
    """K boxes of one extent of the C-order array of `shape` that the chunk holds (blosc_b200_getslices): box i covers
    items [starts[i][k], starts[i][k] + extent[k]) of each dimension and lands at dest + i * B, B its bytes, so `dest`
    is the stack of the K slices.  starts: (K, ndim), an int64 CUDA tensor (on the device of the call), a numpy array
    or a sequence.  Returns the bytes written, or a negative code (dest is then untouched)."""
    sh, ex, st = _boxes(shape, extent, starts)
    return int(lib.blosc_b200_getslices(_ptr(src), sh.size, sh.ctypes.data, ex.ctypes.data, st[2], st[1], _ptr(dest)))


def _fill(fill, itemsize):
    """a grid's fill value as itemsize bytes in a numpy array (bytes, or a numpy scalar of that size), or None"""
    import numpy as np
    if fill is None:
        return None
    f = np.frombuffer(bytes(fill), np.uint8) if isinstance(fill, (bytes, bytearray)) else \
        np.ascontiguousarray(fill).reshape(-1).view(np.uint8)
    if f.size != itemsize:
        raise ValueError(f"fill has {f.size} bytes, not the itemsize {itemsize}")
    return f


def _grid_shapes(shape, chunkshape):
    import numpy as np
    sh = np.ascontiguousarray(shape, dtype=np.int64).reshape(-1)
    cs = np.ascontiguousarray(chunkshape, dtype=np.int64).reshape(-1)
    if cs.size != sh.size:
        raise ValueError(f"shape and chunkshape have {sh.size} and {cs.size} entries")
    return sh, cs


def _nbytes(buf):
    if hasattr(buf, "untyped_storage"):     # torch.Tensor
        return buf.numel() * buf.element_size()
    return buf.nbytes if hasattr(buf, "nbytes") else len(buf)


def grid_bound(shape, chunkshape, itemsize) -> int:
    """Bytes that always hold grid_compress's chunks (blosc_b200_grid_bound); 0 on overflow"""
    sh, cs = _grid_shapes(shape, chunkshape)
    return int(lib.blosc_b200_grid_bound(sh.size, sh.ctypes.data, cs.ctypes.data, itemsize))


def grid_compress(src, shape, chunkshape, itemsize, clevel, doshuffle, compressor, dest, destsize=None, typesize=None,
                  blocksize=0, fill=None, skip_fill=False, numinternalthreads=1):
    """The C-order array `src` of `shape` (itemsize-byte items; a numpy array or a torch tensor, host or CUDA) written
    as the regular grid of Blosc-1 chunks that grid_getslice reads (zarr v2, HDF5 blosc; blosc_b200_grid_compress): each
    chunk is compress_ctx of its sub-array at full chunk shape, edge padding `fill` (as in grid_getslice; None: zeros),
    header typesize `typesize` (default itemsize).  The chunks go back to back into `dest` (host or CUDA; destsize
    default: all of it) in grid C order.  skip_fill: a chunk that holds only `fill` is not written.  Returns (nbytes,
    offsets): the bytes written, or 0 when they do not fit, or a negative code, and the nchunks + 1 int64 offsets of the
    chunks in dest (grid_chunks cuts them out)."""
    import numpy as np
    sh, cs = _grid_shapes(shape, chunkshape)
    nchunks = 1
    if (cs >= 1).all() and (sh >= 0).all():               # else the library rejects the geometry
        for s, c in zip(sh.tolist(), cs.tolist()):
            nchunks *= -(-s // c)
    offsets = np.zeros(nchunks + 1, np.int64)
    f = _fill(fill, itemsize)
    n = lib.blosc_b200_grid_compress(clevel, doshuffle, itemsize if typesize is None else typesize, _name(compressor),
                                     blocksize, numinternalthreads, sh.size, sh.ctypes.data, cs.ctypes.data, itemsize,
                                     _ptr(src), None if f is None else f.ctypes.data, int(bool(skip_fill)), _ptr(dest),
                                     _nbytes(dest) if destsize is None else destsize, offsets.ctypes.data)
    return int(n), offsets


def grid_chunks(dest, offsets):
    """The chunks grid_compress wrote into `dest`, in grid C order, as views of it (None for a chunk skip_fill left
    out), ready to pass as grid_getslice's `chunks`"""
    d = dest.reshape(-1)
    if hasattr(d, "untyped_storage"):
        import torch
        d = d.view(torch.uint8)
    elif hasattr(d, "view"):
        import numpy as np
        d = d.view(np.uint8)
    o = [int(x) for x in offsets]
    return [d[a:b] if b > a else None for a, b in zip(o[:-1], o[1:])]


def grid_getslice(chunks, shape, chunkshape, itemsize, start, stop, dest, step=None, fill=None):
    """A box, with steps, of the C-order array of `shape` stored as a regular grid of chunks (zarr v2, HDF5 blosc,
    PyTables; blosc_b200_grid_getslice): `chunks` lists the ceil(shape[k] / chunkshape[k]) chunks per dimension in C
    order of the grid, each a Blosc-1 chunk of its sub-array at full chunk shape (bytes, bytearray, a numpy array or a
    torch tensor on the host or on CUDA), or None for a missing chunk, whose items are `fill` (itemsize bytes, or a
    numpy scalar of that size; None: zeros).  Items are `itemsize` bytes whatever the chunks' header typesize.  Writes
    numpy's a[start:stop:step] to `dest` as one contiguous C-order array, as getslice does.  Returns the bytes written,
    or a negative code (a host dest is then untouched)."""
    import numpy as np
    sh, st, sp = _box(shape, start, stop)
    cs = np.ascontiguousarray(chunkshape, dtype=np.int64).reshape(-1)
    if cs.size != sh.size:
        raise ValueError(f"shape and chunkshape have {sh.size} and {cs.size} entries")
    if (cs >= 1).all() and (sh >= 0).all():                # else the library rejects the geometry
        nchunks = 1
        for s, c in zip(sh.tolist(), cs.tolist()):
            nchunks *= -(-s // c)
        if len(chunks) != nchunks:
            raise ValueError(f"{len(chunks)} chunks, but the grid has {nchunks}")
    table = (C.c_void_p * max(len(chunks), 1))(*[_ptr(c) for c in chunks])
    f = _fill(fill, itemsize)
    t = None if step is None else _step(sh, step)
    return int(lib.blosc_b200_grid_getslice(sh.size, sh.ctypes.data, cs.ctypes.data, itemsize, table,
                                            None if f is None else f.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                            None if t is None else t.ctypes.data, _ptr(dest)))


def _name(compressor):
    return compressor.encode() if isinstance(compressor, str) else compressor


def frame_bound(nbytes, typesize=1, chunksize=0) -> int:
    """Worst-case size of a frame (blosc_b200_frame_bound)."""
    return int(lib.blosc_b200_frame_bound(nbytes, typesize, chunksize))


def frame_compress(clevel, doshuffle, typesize, nbytes, src, dest, destsize, compressor, blocksize=0, chunksize=0,
                   numinternalthreads=1):
    """Buffers of any size as a sequence of independent Blosc-1 chunks, several in flight."""
    return int(lib.blosc_b200_frame_compress(clevel, doshuffle, typesize, nbytes, _ptr(src), _ptr(dest), destsize,
                                             _name(compressor), blocksize, chunksize, numinternalthreads))


def frame_decompress(frame, framesize, dest, destsize, numinternalthreads=1):
    return int(lib.blosc_b200_frame_decompress(_ptr(frame), framesize, _ptr(dest), destsize, numinternalthreads))


def frame_getitem(frame, framesize, start, nitems, dest):
    return int(lib.blosc_b200_frame_getitem(_ptr(frame), framesize, start, nitems, _ptr(dest)))


def frame_getitems(frame, framesize, starts, nitems, dest):
    """getitems over a frame (blosc_b200_frame_getitems); ranges may cross chunk boundaries.  starts / nitems may be
    int64 or uint64 CUDA tensors: on the device of the call, the read is then planned on the GPU (on another device,
    they are copied to the host for the plan)."""
    st, n = _ranges(starts, nitems, "uint64", ("torch.int64", "torch.uint64"))
    return int(lib.blosc_b200_frame_getitems(_ptr(frame), framesize, st[2], st[1], n[1], _ptr(dest)))


def frame_getslice(frame, framesize, shape, start, stop, dest, step=None):
    """getslice over the array a frame holds (blosc_b200_frame_getslice, or blosc_b200_frame_getslice_step with
    `step`); the box may cross chunk boundaries."""
    sh, st, sp = _box(shape, start, stop)
    if step is None:
        return int(lib.blosc_b200_frame_getslice(_ptr(frame), framesize, sh.size, sh.ctypes.data, st.ctypes.data,
                                                 sp.ctypes.data, _ptr(dest)))
    t = _step(sh, step)
    return int(lib.blosc_b200_frame_getslice_step(_ptr(frame), framesize, sh.size, sh.ctypes.data, st.ctypes.data,
                                                  sp.ctypes.data, t.ctypes.data, _ptr(dest)))


def frame_getslices(frame, framesize, shape, extent, starts, dest):
    """getslices over the array a frame holds (blosc_b200_frame_getslices); boxes may cross chunk boundaries."""
    sh, ex, st = _boxes(shape, extent, starts)
    return int(lib.blosc_b200_frame_getslices(_ptr(frame), framesize, sh.size, sh.ctypes.data, ex.ctypes.data, st[2],
                                              st[1], _ptr(dest)))


def _selection(shape, selection):
    """An orthogonal selection as the C call takes it: shape, start, stop and step as int64 host arrays (the slices,
    list dimensions whole), the lists to keep alive, the index pointer array (None when no dimension is a list) and
    the list lengths."""
    import numpy as np
    sh = np.ascontiguousarray(shape, dtype=np.int64).reshape(-1)
    if len(selection) != sh.size:
        raise ValueError(f"shape and selection have {sh.size} and {len(selection)} entries")
    n = sh.size
    st, sp, t, nidx = (np.zeros(n, np.int64) for _ in range(4))
    ptrs, keep = (C.c_void_p * max(n, 1))(), []
    for k, s in enumerate(selection):
        st[k], sp[k], t[k] = 0, sh[k], 1
        if isinstance(s, slice):
            a, b, c = (0 if s.start is None else s.start), (sh[k] if s.stop is None else s.stop), \
                (1 if s.step is None else s.step)
            if a < 0 or b < 0 or c < 1:
                raise ValueError(f"dimension {k}: negative slice fields and steps below 1 are not supported ({s})")
            st[k] = min(a, sh[k])
            sp[k] = min(max(b, st[k]), sh[k])
            t[k] = c
            continue
        if isinstance(s, (int, np.integer)) and not isinstance(s, (bool, np.bool_)):
            if s < 0:
                raise ValueError(f"dimension {k}: negative index {s} is not supported")
            st[k], sp[k] = s, s + 1
            continue
        if _is_cuda(s):
            if s.dim() != 1:
                raise ValueError(f"dimension {k}: an index list must be 1-d")
            if str(s.dtype) == "torch.bool":
                if s.numel() != sh[k]:
                    raise ValueError(f"dimension {k}: a mask of {s.numel()} entries for an extent of {sh[k]}")
                s = s.nonzero().reshape(-1)                 # syncs with the device
            elif str(s.dtype) != "torch.int64":
                raise TypeError(f"CUDA index lists must be torch.int64 or torch.bool, not {s.dtype}")
            s = s.contiguous()
            keep.append(s)
            ptrs[k], nidx[k] = s.data_ptr(), s.numel()
        else:
            h = np.asarray(s.numpy() if hasattr(s, "numpy") else s)
            if h.ndim != 1:
                raise ValueError(f"dimension {k}: an index list must be 1-d")
            if h.dtype == np.bool_:
                if h.size != sh[k]:
                    raise ValueError(f"dimension {k}: a mask of {h.size} entries for an extent of {sh[k]}")
                h = np.flatnonzero(h)
            elif h.size and h.dtype.kind not in "iu":
                raise TypeError(f"dimension {k}: index lists must be integers, not {h.dtype}")
            h = np.ascontiguousarray(h, dtype=np.int64)
            keep.append(h)
            ptrs[k], nidx[k] = h.ctypes.data, h.size
        if not nidx[k]:                                     # an empty list, which is never read: any non-NULL address
            ptrs[k] = sh.ctypes.data
    return sh, st, sp, t, keep, (ptrs if keep else None), nidx


def getoindex(src, shape, selection, dest):
    """An orthogonal index selection of the C-order array of `shape` that the chunk holds (blosc_b200_getoindex):
    numpy's a[np.ix_(...)] with slices kept as slices, made contiguous in C order (zarr's oindex).  `selection` has one
    entry per dimension: a slice (positive fields; None takes numpy's default), an int (one coordinate, as numpy's
    a[..., i, ...], which drops the dimension: the bytes are the same), a 1-d integer sequence or numpy array (uploaded
    once), an int64 CUDA tensor on the device of the call (read in place; other CUDA dtypes raise TypeError), or a 1-d
    bool mask of the dimension's length, turned into its indices with nonzero (on a CUDA mask that syncs with the
    device).  Entries may be unsorted and repeat.  A selection with no list is getslice with its steps.  Returns the
    bytes written, or a negative code (dest is then untouched)."""
    sh, st, sp, t, keep, ptrs, nidx = _selection(shape, selection)
    if ptrs is None:
        return getslice(src, sh, st, sp, dest, step=t)
    return int(lib.blosc_b200_getoindex(_ptr(src), sh.size, sh.ctypes.data, st.ctypes.data, sp.ctypes.data,
                                        t.ctypes.data, C.cast(ptrs, C.c_void_p), nidx.ctypes.data, _ptr(dest)))


def frame_getoindex(frame, framesize, shape, selection, dest):
    """getoindex over the array a frame holds (blosc_b200_frame_getoindex); the selection may cross chunk
    boundaries, and chunks that hold no selected item are not read."""
    sh, st, sp, t, keep, ptrs, nidx = _selection(shape, selection)
    if ptrs is None:
        return frame_getslice(frame, framesize, sh, st, sp, dest, step=t)
    return int(lib.blosc_b200_frame_getoindex(_ptr(frame), framesize, sh.size, sh.ctypes.data, st.ctypes.data,
                                              sp.ctypes.data, t.ctypes.data, C.cast(ptrs, C.c_void_p),
                                              nidx.ctypes.data, _ptr(dest)))


def frame_info(frame, framesize):
    """(nbytes, cbytes, chunksize, nchunks) or None if `frame` is not a valid frame."""
    v = [C.c_size_t(0) for _ in range(4)]
    if lib.blosc_b200_frame_info(_ptr(frame), framesize, *[C.byref(x) for x in v]) != 0:
        return None
    return tuple(int(x.value) for x in v)


def frame_chunk(frame, framesize, i):
    """(offset, cbytes) of chunk i inside the frame, or None."""
    n = C.c_size_t(0)
    off = lib.blosc_b200_frame_chunk(_ptr(frame), framesize, i, C.byref(n))
    return None if off < 0 else (int(off), int(n.value))


def filter_block(mode, typesize, blocksize, src, dest):
    """One filter over one block (GPU counterpart of blosc_internal_{,un}{,bit}shuffle)."""
    return lib.blosc_b200_filter(mode, typesize, blocksize, _ptr(src), _ptr(dest))


def set_profiling(on: bool):
    lib.blosc_b200_set_profiling(1 if on else 0)


def prof_reset():
    lib.blosc_b200_prof_reset()


def prof_get():
    """{kind: (total_ms, launches)} measured with CUDA events on the launching stream."""
    out = {}
    for i, k in enumerate(KERNEL_KINDS):
        ms, n = C.c_double(0), C.c_longlong(0)
        lib.blosc_b200_prof_get(i, C.byref(ms), C.byref(n))
        out[k] = (ms.value, n.value)
    return out


def launch_count() -> int:
    return int(lib.blosc_b200_launch_count())

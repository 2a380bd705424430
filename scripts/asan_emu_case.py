#!/usr/bin/env python
"""Workload for the AddressSanitizer build of the emulated library (make -C tests/emu asan):
  LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python scripts/asan_emu_case.py
exact / fast / lz4hc / BloscLZ paths, exact-size buffers, damaged chunks."""
import os, sys, ctypes as C, numpy as np
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
from datagen import gen, compress, decompress
emu=C.CDLL(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'emu', '_build', 'libblosc_b200_emu_asan.so'))
emu.blosc_compress_ctx.restype=C.c_int; emu.blosc_decompress_ctx.restype=C.c_int; emu.blosc_getitem.restype=C.c_int
rng=np.random.default_rng(1)
cases=0
for parse in ("exact","fast"):
    os.environ['BLOSC_B200_PARSE']=parse
    for kind in ("bench","text","mixed","zeros","rand","f32"):
        for n in (13, 1000, 70001, 300001):
            src=gen(kind,n)
            for comp,ts,shuf,cl in (("lz4",4,1,5),("lz4",1,0,9),("lz4hc",8,1,5),("blosclz",4,1,5),("blosclz",8,2,5),("lz4",16,2,1),("blosclz",2,1,9)):
                dest=np.full(n+16,0xAA,np.uint8)        # exact-size buffers: ASan sees any overrun
                r=emu.blosc_compress_ctx(C.c_int(cl),C.c_int(shuf),C.c_size_t(ts),C.c_size_t(n),src.ctypes.data_as(C.c_void_p),dest.ctypes.data_as(C.c_void_p),C.c_size_t(n+16),comp.encode(),C.c_size_t(0),C.c_int(1))
                assert r>0
                chunk=dest[:r].copy(); out=np.zeros(n,np.uint8)
                assert emu.blosc_decompress_ctx(chunk.ctypes.data_as(C.c_void_p),out.ctypes.data_as(C.c_void_p),C.c_size_t(n),C.c_int(1))==n and (out==src).all()
                # damaged copies
                for t in range(3):
                    c=chunk.copy(); pos=rng.integers(16,r,3); c[pos]=rng.integers(0,256,3,dtype=np.uint8)
                    emu.blosc_decompress_ctx(c.ctypes.data_as(C.c_void_p),out.ctypes.data_as(C.c_void_p),C.c_size_t(n),C.c_int(1))
                cases+=1
os.environ.pop('BLOSC_B200_PARSE', None)
os.environ['BLOSC_B200_ZSTD']='1'          # the zstd encoder: several zstd blocks per frame (forced blocksize), raw streams
for kind in ("bench","text","lowent","mixed","zeros","rand"):
    for n in (13, 1000, 70001, 300001):
        src=gen(kind,n)
        for ts,shuf,cl,bs in ((4,1,5,0),(1,0,9,0),(8,2,1,0),(3,1,5,200000)):
            dest=np.full(n+16,0xAA,np.uint8)
            r=emu.blosc_compress_ctx(C.c_int(cl),C.c_int(shuf),C.c_size_t(ts),C.c_size_t(n),src.ctypes.data_as(C.c_void_p),dest.ctypes.data_as(C.c_void_p),C.c_size_t(n+16),b"zstd",C.c_size_t(bs),C.c_int(1))
            assert r>0
            chunk=dest[:r].copy(); out=np.zeros(n,np.uint8)
            assert emu.blosc_decompress_ctx(chunk.ctypes.data_as(C.c_void_p),out.ctypes.data_as(C.c_void_p),C.c_size_t(n),C.c_int(1))==n and (out==src).all()
            cases+=1
print("asan workload ok, cases", cases)

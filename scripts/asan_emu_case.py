#!/usr/bin/env python
"""Workload for the AddressSanitizer build of the emulated library (make -C tests/emu asan):
  LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python scripts/asan_emu_case.py
exact / fast / lz4hc / BloscLZ paths, exact-size buffers, damaged chunks, crafted and damaged zstd frames and zlib streams,
crafted, random and damaged LZ4 and BloscLZ streams."""
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
os.environ.pop('BLOSC_B200_ZSTD', None)
# the zstd entropy stage on chosen sequence records (emu_zstd_frame): the records-driven scenarios of
# tests/test_zstd_encode_edges.py, each frame decoded by zstd_frame.py and by this library's decoder
import test_zstd_encode_edges as edges
emu.emu_zstd_frame.restype=C.c_int; emu.emu_zstd_frame.argtypes=[C.c_void_p,C.c_int,C.c_void_p,C.c_void_p,C.c_void_p]
emu.emu_zstd_decode.restype=C.c_int; emu.emu_zstd_decode.argtypes=[C.c_void_p,C.c_int,C.c_void_p,C.c_int]
for sc in edges.SCENARIOS:
    for name,p in sc().items():
        edges.encode_and_check(emu,None,p)
        cases+=1
# the zstd decoder on crafted frames (tests/test_zstd_decode_edges.py): accepted, rejected, STRICT and damaged frames,
# each in an input buffer of exactly its size, so that a read past the input shows; then the same frames as chunks
import test_zstd_decode_edges as zedges
frames=[(f,len(c)) for f,c,_ in zedges.ACCEPT.values()]+[(f,cap) for f,cap,_ in zedges.REJECT.values()]
frames+=[(fc[0],len(fc[1])+16) for fc,_ in zedges.strict_frames().values()]+list(zedges._damage_corpus())
for f,cap in frames:
    src=np.frombuffer(f,np.uint8).copy(); out=np.zeros(max(cap,1),np.uint8)
    emu.emu_zstd_decode(src.ctypes.data_as(C.c_void_p),C.c_int(len(f)),out.ctypes.data_as(C.c_void_p),C.c_int(cap))
    cases+=1
for name,ch,n,_ in zedges.chunk_corpus(damaged=True):
    c=np.frombuffer(ch,np.uint8).copy(); out=np.zeros(n,np.uint8)
    emu.blosc_decompress_ctx(c.ctypes.data_as(C.c_void_p),out.ctypes.data_as(C.c_void_p),C.c_size_t(n),C.c_int(1))
    emu.blosc_getitem(c.ctypes.data_as(C.c_void_p),C.c_int(0),C.c_int(n),out.ctypes.data_as(C.c_void_p))
    cases+=1
# the inflate decoder on crafted streams (tests/test_zlib_decode_edges.py): accepted, rejected, Adler-32 sizes and
# damaged streams, each in an input buffer of exactly its size; then the same streams as chunks
import test_zlib_decode_edges as iedges
emu.emu_zlib_decode.restype=C.c_int; emu.emu_zlib_decode.argtypes=[C.c_void_p,C.c_int,C.c_void_p,C.c_int]
streams=[(st,len(iedges.zlib_verdict(st,1<<20))) for st in iedges.ACCEPT.values()]+[(st,cap) for st,cap,_ in iedges.REJECT.values()]
streams+=[(st,len(d)) for _,st,d in iedges.adler_streams()]+list(iedges._damage_corpus())
for st,cap in streams:
    src=np.frombuffer(st,np.uint8).copy(); out=np.zeros(max(cap,1),np.uint8)
    emu.emu_zlib_decode(src.ctypes.data_as(C.c_void_p),C.c_int(len(st)),out.ctypes.data_as(C.c_void_p),C.c_int(cap))
    cases+=1
for name,ch,n in iedges.chunk_corpus():
    c=np.frombuffer(ch,np.uint8).copy(); out=np.zeros(n,np.uint8)
    emu.blosc_decompress_ctx(c.ctypes.data_as(C.c_void_p),out.ctypes.data_as(C.c_void_p),C.c_size_t(n),C.c_int(1))
    cases+=1
# the LZ4 and BloscLZ decoders on crafted streams (tests/test_lz_decode_edges.py): accepted, rejected, random and damaged
# streams, each in an input buffer of exactly its size (the decoders' 12-byte window loads claim to stay below ip+109,
# ip+42 and ip+12 at their tiers' entry conditions); both LZ4 decoders; the ring-reuse lists; then the chunks
import random
import test_lz_decode_edges as ledges
for f in ("emu_lz4_decode","emu_lz4_decode_pair","emu_blz_decode"):
    getattr(emu,f).restype=C.c_int; getattr(emu,f).argtypes=[C.c_void_p,C.c_int,C.c_void_p,C.c_int]
lz=[(b,cap) for b,c,caps,_,_ in ledges.ACCEPT.values() for cap in (caps or [len(c)])]+[(b,cap) for b,cap,_ in ledges.REJECT.values()]
rng=random.Random(5)
for t in range(100):
    b,c=ledges.random_block(rng); lz+=[(b,len(c)),(ledges._damaged(b,rng,2),len(c))]
for b,cap in lz:
    src=np.frombuffer(b,np.uint8).copy(); out=np.zeros(max(cap,1),np.uint8)
    for f in (emu.emu_lz4_decode,emu.emu_lz4_decode_pair):
        f(src.ctypes.data_as(C.c_void_p),C.c_int(len(b)),out.ctypes.data_as(C.c_void_p),C.c_int(cap))
        cases+=1
blz=[(s,cap) for s,_,cap,_,_ in ledges.BACCEPT.values()]+[(s,cap) for s,cap,_ in ledges.BREJECT.values()]
for t in range(100):
    s,c=ledges.random_blz(rng); blz+=[(s,len(c)),(ledges._damaged(s,rng,2),len(c))]
for s,cap in blz:
    src=np.frombuffer(s,np.uint8).copy(); out=np.zeros(max(cap,1),np.uint8)
    emu.emu_blz_decode(src.ctypes.data_as(C.c_void_p),C.c_int(len(s)),out.ctypes.data_as(C.c_void_p),C.c_int(cap))
    cases+=1
emu.emu_lz4_decode_list.restype=None
for pair in (0,1):
    for name,a,(b,want) in ledges.ring_pairs():
        ledges.decode_list(emu,[a[0],b],[len(a[1]),len(want)],pair)
        cases+=1
for name,ch,n in ledges.chunk_corpus():
    c=np.frombuffer(ch,np.uint8).copy(); out=np.zeros(n,np.uint8)
    emu.blosc_decompress_ctx(c.ctypes.data_as(C.c_void_p),out.ctypes.data_as(C.c_void_p),C.c_size_t(n),C.c_int(1))
    emu.blosc_getitem(c.ctypes.data_as(C.c_void_p),C.c_int(0),C.c_int(n//ch[3]),out.ctypes.data_as(C.c_void_p))
    cases+=1
print("asan workload ok, cases", cases)

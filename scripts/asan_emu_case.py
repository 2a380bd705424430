#!/usr/bin/env python
"""Workload for the AddressSanitizer build of the emulated library (make -C tests/emu asan):
  LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python scripts/asan_emu_case.py
exact / fast / lz4hc / BloscLZ paths, exact-size buffers, damaged chunks, crafted and damaged zstd frames and zlib streams,
crafted, random and damaged LZ4 and BloscLZ streams, the snappy encoder (serial and pool maxout rules), crafted,
random and damaged snappy streams, item ranges, boxes, batches of boxes and index selections of whole and damaged
chunks and frames, and boxes of chunk grids with present, missing and damaged chunks, in host and in device memory."""
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
os.environ['BLOSC_B200_SNAPPY']='1'        # the snappy encoder and decoder: both maxout rules, raw and compressed splits
import snappy_read, snappy_write
srng=np.random.default_rng(7)
for kind in ("bench","text","lowent","mixed","zeros","rand"):
    for n in (13, 1000, 70001, 300001):
        src=gen(kind,n)
        for ts,shuf,cl,bs,nt in ((4,1,5,0,1),(1,0,9,0,4),(8,2,1,0,1),(3,1,5,200000,4)):
            dest=np.full(n+16,0xAA,np.uint8)
            r=emu.blosc_compress_ctx(C.c_int(cl),C.c_int(shuf),C.c_size_t(ts),C.c_size_t(n),src.ctypes.data_as(C.c_void_p),dest.ctypes.data_as(C.c_void_p),C.c_size_t(n+16),b"snappy",C.c_size_t(bs),C.c_int(nt))
            assert r>0
            chunk=dest[:r].copy(); out=np.zeros(n,np.uint8)
            assert emu.blosc_decompress_ctx(chunk.ctypes.data_as(C.c_void_p),out.ctypes.data_as(C.c_void_p),C.c_size_t(n),C.c_int(1))==n and (out==src).all()
            for t in range(3):
                c=chunk.copy(); pos=srng.integers(16,r,3); c[pos]=srng.integers(0,256,3,dtype=np.uint8)
                emu.blosc_decompress_ctx(c.ctypes.data_as(C.c_void_p),out.ctypes.data_as(C.c_void_p),C.c_size_t(n),C.c_int(1))
            cases+=1
for t in range(300):                        # crafted streams, then random damage and truncation, exact-size buffers
    lit=srng.integers(0,256,int(srng.integers(1,3000)),dtype=np.uint8).tobytes()
    els=[("lit",lit)]+[("c2",int(srng.integers(1,65)),int(srng.integers(1,len(lit)+1))) for _ in range(int(srng.integers(0,60)))]
    n=len(snappy_write.expand(els)); st=bytearray(snappy_write.stream(n,els))
    if t%3==1: st[int(srng.integers(0,len(st)))]=int(srng.integers(0,256))
    if t%3==2: st=st[:int(srng.integers(0,len(st)+1))]
    # one unsplit block holding the stream (a stream of n bytes would be taken for a raw split)
    if len(st)==n: st=st+b"\0"
    hdr=bytes([2,1,0x10|(2<<5),1])+n.to_bytes(4,"little")+n.to_bytes(4,"little")+(24+len(st)).to_bytes(4,"little")+(20).to_bytes(4,"little")+len(st).to_bytes(4,"little")
    c=np.frombuffer(hdr+bytes(st),np.uint8).copy(); out=np.zeros(n,np.uint8)
    r=emu.blosc_decompress_ctx(c.ctypes.data_as(C.c_void_p),out.ctypes.data_as(C.c_void_p),C.c_size_t(n),C.c_int(1))
    got,why=snappy_read.read(bytes(st),n)
    assert (r==n)==(why is None) and (why is not None or out.tobytes()==got)
    cases+=1
os.environ.pop('BLOSC_B200_SNAPPY', None)
# item ranges, boxes and batches of boxes of a chunk and of a frame: the host plan, the GPU plans and the box plan, each with the chunk or
# frame in host memory (the touched blocks staged, the block list read back) and then in device memory
# (emu_set_all_device: lists and dest too); compressed, memcpyed and damaged chunks
vp,sz,ll=C.c_void_p,C.c_size_t,C.c_longlong
P=lambda a: a.ctypes.data_as(vp)
for f,res,args in (("blosc_b200_getitems",ll,[vp,C.c_int,vp,vp,vp]),("blosc_b200_getslice",ll,[vp,C.c_int,vp,vp,vp,vp]),
                   ("blosc_b200_frame_bound",sz,[sz,sz,sz]),("blosc_b200_frame_compress",ll,[C.c_int,C.c_int,sz,sz,vp,vp,sz,C.c_char_p,sz,sz,C.c_int]),
                   ("blosc_b200_frame_getitems",ll,[vp,sz,sz,vp,vp,vp]),("blosc_b200_frame_getslice",ll,[vp,sz,C.c_int,vp,vp,vp,vp]),
                   ("blosc_b200_getslices",ll,[vp,C.c_int,vp,vp,ll,vp,vp]),("blosc_b200_frame_getslices",ll,[vp,sz,C.c_int,vp,vp,ll,vp,vp]),
                   ("blosc_b200_getslice_step",ll,[vp,C.c_int,vp,vp,vp,vp,vp]),("blosc_b200_frame_getslice_step",ll,[vp,sz,C.c_int,vp,vp,vp,vp,vp]),
                   ("blosc_b200_frame_getoindex",ll,[vp,sz,C.c_int,vp,vp,vp,vp,vp,vp,vp]),
                   ("blosc_b200_grid_getslice",ll,[C.c_int,vp,vp,sz,vp,vp,vp,vp,vp,vp])):
    getattr(emu,f).restype=res; getattr(emu,f).argtypes=args
emu.emu_set_all_device.argtypes=[C.c_int]
irng=np.random.default_rng(11)
ts,shape=4,(300,250)
n=ts*shape[0]*shape[1]
src=gen("bench",n); arr=src.view(np.uint32).reshape(shape)
box=([17,30],[123,200]); want_box=arr[17:123,30:200].tobytes()
bstep=np.array([7,3],np.int64); want_step=arr[17:123:7,30:200:3].tobytes()
ranges=[(int(s),int(k)) for s,k in zip(irng.integers(0,n//ts-600,40),irng.integers(0,600,40))]+[(5,0),(100,3),(101,900)]
st=np.array([r[0] for r in ranges],np.int32); nt=np.array([r[1] for r in ranges],np.int32)
want_items=b"".join(src[s*ts:(s+k)*ts].tobytes() for s,k in ranges)
sh=np.array(shape,np.int64); b0=np.array(box[0],np.int64); b1=np.array(box[1],np.int64)
fst=st.astype(np.uint64); fnt=nt.astype(np.uint64)
ext=np.array([9,31],np.int64)                 # a batch of boxes, overlapping and on the array's edges, and a bad corner
corners=np.array([[0,0],[291,219],[100,7],[100,7],[150,200]]+[[int(a),int(b)] for a,b in zip(irng.integers(0,292,40),irng.integers(0,220,40))],np.int64)
want_boxes=b"".join(arr[a:a+9,b:b+31].tobytes() for a,b in corners)
bad=corners.copy(); bad[30,1]=220
rows=np.array([5,290,17,17,120,0,299],np.int64); cols=np.arange(30,200,3)      # an index selection: unsorted rows, a column slice
want_osel=arr[np.ix_(rows,cols)].tobytes()
badrows=rows.copy(); badrows[3]=300
ozero=np.zeros(2,np.int64); ostop=np.array([0,200],np.int64); ostep=np.array([0,3],np.int64); ostart=np.array([0,30],np.int64)
def frame_oindex(f,fb,r,out):
    ptrs=(vp*2)(r.ctypes.data,None); ni=np.array([r.size,0],np.int64)
    return emu.blosc_b200_frame_getoindex(P(f),fb,2,P(sh),P(ostart),P(ostop),P(ostep),C.cast(ptrs,vp),P(ni),P(out))
for comp,shuf,cl in (("lz4",1,5),("blosclz",2,5),("lz4",1,0)):
    dest=np.zeros(n+16,np.uint8)
    r=emu.blosc_compress_ctx(C.c_int(cl),C.c_int(shuf),C.c_size_t(ts),C.c_size_t(n),P(src),P(dest),C.c_size_t(n+16),comp.encode(),C.c_size_t(4096),C.c_int(1))
    assert r>0
    chunk=dest[:r].copy()
    fb=emu.blosc_b200_frame_bound(n,ts,64000); fr=np.zeros(fb,np.uint8)
    fb=emu.blosc_b200_frame_compress(cl,shuf,ts,n,P(src),P(fr),fb,comp.encode(),4096,64000,1)
    assert fb>0
    frame=fr[:fb].copy()
    for dev in (0,1):
        emu.emu_set_all_device(dev)
        try:
            for c in [chunk]+[chunk.copy() for _ in range(3)]:
                if c is not chunk: pos=irng.integers(16,r,4); c[pos]=irng.integers(0,256,4,dtype=np.uint8)
                out=np.zeros(len(want_items),np.uint8)
                g=emu.blosc_b200_getitems(P(c),len(ranges),P(st),P(nt),P(out))
                assert c is not chunk or (g==len(want_items) and out.tobytes()==want_items)
                out=np.zeros(len(want_box),np.uint8)
                g=emu.blosc_b200_getslice(P(c),2,P(sh),P(b0),P(b1),P(out))
                assert c is not chunk or (g==len(want_box) and out.tobytes()==want_box)
                out=np.zeros(len(want_step),np.uint8)
                g=emu.blosc_b200_getslice_step(P(c),2,P(sh),P(b0),P(b1),P(bstep),P(out))
                assert c is not chunk or (g==len(want_step) and out.tobytes()==want_step)
                out=np.zeros(len(want_boxes),np.uint8)
                g=emu.blosc_b200_getslices(P(c),2,P(sh),P(ext),len(corners),P(corners),P(out))
                assert c is not chunk or (g==len(want_boxes) and out.tobytes()==want_boxes)
                assert emu.blosc_b200_getslices(P(c),2,P(sh),P(ext),len(bad),P(bad),P(out))<0
                cases+=5
            for f in [frame]+[frame.copy() for _ in range(2)]:
                if f is not frame: pos=irng.integers(100,fb,6); f[pos]=irng.integers(0,256,6,dtype=np.uint8)
                out=np.zeros(len(want_items),np.uint8)
                g=emu.blosc_b200_frame_getitems(P(f),fb,len(ranges),P(fst),P(fnt),P(out))
                assert f is not frame or (g==len(want_items) and out.tobytes()==want_items)
                out=np.zeros(len(want_box),np.uint8)
                g=emu.blosc_b200_frame_getslice(P(f),fb,2,P(sh),P(b0),P(b1),P(out))
                assert f is not frame or (g==len(want_box) and out.tobytes()==want_box)
                out=np.zeros(len(want_step),np.uint8)
                g=emu.blosc_b200_frame_getslice_step(P(f),fb,2,P(sh),P(b0),P(b1),P(bstep),P(out))
                assert f is not frame or (g==len(want_step) and out.tobytes()==want_step)
                out=np.zeros(len(want_boxes),np.uint8)
                g=emu.blosc_b200_frame_getslices(P(f),fb,2,P(sh),P(ext),len(corners),P(corners),P(out))
                assert f is not frame or (g==len(want_boxes) and out.tobytes()==want_boxes)
                assert emu.blosc_b200_frame_getslices(P(f),fb,2,P(sh),P(ext),len(bad),P(bad),P(out))<0
                out=np.zeros(len(want_osel),np.uint8)
                g=frame_oindex(f,fb,rows,out)
                assert f is not frame or (g==len(want_osel) and out.tobytes()==want_osel)
                assert frame_oindex(f,fb,badrows,out)<0
                cases+=7
        finally:
            emu.emu_set_all_device(0)
# boxes of the array stored as a grid of 64 x 96 chunks (edge chunks padded to full shape): every chunk present, some
# missing (read as the fill pattern), and some damaged, with and without steps, chunks in host and in device memory
cs=np.array([64,96],np.int64); grid=(5,3)
fill=np.array([0xDEADBEEF],np.uint32)
gstart=np.array([17,30],np.int64); gstop=np.array([290,240],np.int64); gstep=np.array([2,3],np.int64)
gchunks=[]
for gi in range(grid[0]):
    for gj in range(grid[1]):
        buf=np.zeros((64,96),np.uint32); part=arr[gi*64:(gi+1)*64,gj*96:(gj+1)*96]; buf[:part.shape[0],:part.shape[1]]=part
        d=buf.view(np.uint8).reshape(-1); dest=np.zeros(d.size+16,np.uint8)
        r=emu.blosc_compress_ctx(C.c_int(5),C.c_int(1),C.c_size_t(ts),C.c_size_t(d.size),P(d),P(dest),C.c_size_t(d.size+16),b"lz4",C.c_size_t(4096),C.c_int(1))
        assert r>0
        gchunks.append(dest[:r].copy())
missing={1,7,14}
filled=arr.copy()
for i in missing:
    gi,gj=divmod(i,grid[1]); filled[gi*64:(gi+1)*64,gj*96:(gj+1)*96]=fill[0]
def grid_read(chunks,step,out):
    table=(vp*len(chunks))(*[None if c is None else c.ctypes.data for c in chunks])
    return emu.blosc_b200_grid_getslice(2,P(sh),P(cs),ts,table,P(fill),P(gstart),P(gstop),None if step is None else P(step),P(out))
for dev in (0,1):
    emu.emu_set_all_device(dev)
    try:
        for step in (None,gstep):
            sl=tuple(slice(a,b,s) for a,b,s in zip(gstart,gstop,[1,1] if step is None else step))
            for kind in ("present","missing","damaged"):
                chunks=list(gchunks)
                if kind=="missing": chunks=[None if i in missing else c for i,c in enumerate(chunks)]
                if kind=="damaged":
                    for i in (4,8):
                        c=chunks[i].copy(); pos=irng.integers(16,len(c),6); c[pos]=irng.integers(0,256,6,dtype=np.uint8); chunks[i]=c
                want=np.ascontiguousarray((filled if kind=="missing" else arr)[sl]).tobytes()
                out=np.zeros(len(want),np.uint8)
                g=grid_read(chunks,step,out)
                assert kind=="damaged" or (g==len(want) and out.tobytes()==want)
                cases+=1
    finally:
        emu.emu_set_all_device(0)
print("asan workload ok, cases", cases)

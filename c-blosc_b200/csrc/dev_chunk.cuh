/*
 * dev_chunk.cuh -- chunk-level kernels: the GPU replacement of c-blosc's block
 * scheduler (reference blosc/blosc.c:803-918 serial_blosc/parallel_blosc/do_job and
 * :1706-1887 t_blosc) and of the per-block pipeline blosc_c / blosc_d (:591-800).
 *
 *   encode_kernel   one warp per LZ stream (= one split of one Blosc block): codec into a
 *                   worst-case slot (capacity neblock, as t_blosc's tmp2, :1810-1811)
 *   scan_kernel     exclusive scan of the per-block compressed sizes -> bstarts, total
 *                   cbytes and the "does it fit in destsize" verdict (:1843-1856)
 *   compact_kernel  writes the 16-byte header, bstarts[] and the int32-prefixed split
 *                   payloads at their final offsets (:1148-1247, :715, :1860)
 *   decode_kernel   one warp per LZ stream: bounds-checked walk of the size prefixes
 *                   (:761-770), raw-split copy or codec (:773-783)
 *   gather_kernel, plan_check_kernel, plan_scan_kernel
 *                   many item ranges of one chunk (blosc_b200_getitems): the copy out of
 *                   the decoded blocks, and its plan when the range lists are device memory
 *   fplan_check_kernel, fplan_scatter_kernel (+ plan_scan_kernel)
 *                   the same over a frame (blosc_b200_frame_getitems): the ranges cut into
 *                   one piece list per chunk, each read by the chunk plan
 *   box_touch_kernel, box_gather_kernel (+ plan_scan_kernel<PLAN_SLOT>)
 *                   a box of an N-d array, with a step per dimension or without
 *                   (blosc_b200_getslice_step): the touched blocks and the copy out of them,
 *                   both from the box alone (B2Box, b2_args.h)
 *   box_check_kernel, boxes_touch_kernel, boxes_gather_kernel (+ plan_scan_kernel<PLAN_SLOT>)
 *                   a batch of boxes of one extent (blosc_b200_getslices): the corners' check,
 *                   the blocks touched by any box and the copy out, from the origin box and one
 *                   flat offset per box
 *   placed_gather_kernel, placed_fill_kernel
 *                   one chunk's part of a box of an array stored as a grid of chunks
 *                   (blosc_b200_grid_getslice), written straight into its place in the output,
 *                   or the fill value over the part of a missing chunk
 *   grid_pack_kernel
 *                   one chunk's sub-array packed out of an N-d array into the chunk's input
 *                   (blosc_b200_grid_compress), compared with the fill value on request
 */
#pragma once
#include "b2_args.h"
#include "dev_blosclz.cuh"
#include "dev_common.cuh"
#include "dev_inflate.cuh"
#include "dev_lz4.cuh"
#include "dev_lz4fast.cuh"
#include "dev_lz4dpair.cuh"
#include "dev_zstd.cuh"
#include "dev_zstdenc.cuh"
#include "dev_deflate.cuh"
#include "dev_snappy.cuh"



/* Dynamic scheduling (the GPU counterpart of t_blosc's shared block counter, blosc.c:1769-1776):
 * every warp pulls the next job number from a global counter until none is left.  Jobs are
 * numbered longest-first as far as that is knowable without looking at the data: the unsplit
 * leftover block first, then split-major (split s of every block before split s+1), so that
 * the byte-planes that turn out to be hard start in the first wave and the cheap ones fill in
 * behind them.  Returns the stream index, or -1 when the queue is empty.  Every warp of a launch
 * draws exactly one ticket past the end, so a launch consumes nstreams + (warps launched) tickets. */
DEV int next_stream(int* queue, unsigned base, const StreamMap& m) {
  int job = 0;
  if (lane_id() == 0) job = (int)((unsigned)atomicAdd(queue, 1) - base);
  job = __shfl_sync(FULLMASK, job, 0);
  if (job >= m.nstreams) return -1;
  const int nfs = m.nfull * m.nsplits;
  if (m.leftover) {
    if (job == 0) return nfs;
    job--;
  }
  const int s = job / m.nfull, b = job - s * m.nfull;
  return b * m.nsplits + s;
}

/* stream index -> (block, offset inside the uncompressed buffer, length).  With a block list (DecodeArgs.blocks,
 * getitems) first_block is 0, so the offset computed for the j-th selected block is already j * blocksize of the
 * compact output (the caller's out_shift is 0); only the block number comes from the list. */
DEV void stream_locate(const StreamMap& m, int idx, int* block, long long* off, int* len, int* split,
                       const int* blocks = nullptr) {
  const int nfs = m.nfull * m.nsplits;
  if (idx < nfs) {
    const int b = idx / m.nsplits, s = idx - b * m.nsplits;
    const int neblock = m.blocksize / m.nsplits;
    *block = m.first_block + b;
    *off = (long long)(m.first_block + b) * m.blocksize + (long long)s * neblock;
    *len = neblock;
    *split = s;
  } else {
    *block = m.first_block + m.nfull;
    *off = (long long)(m.first_block + m.nfull) * m.blocksize;
    *len = m.leftover;
    *split = 0;
  }
  if (blocks) *block = blocks[*block];
}

/* The end of every encode and decode launch, for one warp that finished `mine` streams: the warp that completes the
 * count of finished streams runs `last` and puts the count back to zero for the next launch on this workspace (the
 * ticket counter is never reset: warps that got no stream may still be polling it). */
template <class Last>
DEV void streams_done(int* done, const int nstreams, const int mine, Last last) {
  if (mine == 0) return;
  __threadfence();
  int is_last = 0;
  if (lane_id() == 0) is_last = atomicAdd(done, mine) + mine == nstreams;
  is_last = __shfl_sync(FULLMASK, is_last, 0);
  if (!is_last) return;
  __threadfence();
  last();
  __syncwarp();
  if (lane_id() == 0) *done = 0;
}


/* L2 loads for words written by other SMs during this launch */
DEV int ld_cg_i32(const int* p) {
#ifdef SIMT_EMU
  return *p;
#else
  return __ldcg(p);
#endif
}

/* The bytes that blocks [b0, b1) take in the chunk: every split's size prefix and its compressed (or raw) bytes */
DEV long long scan_sum(const ScanArgs& a, const int* csizes, const int b0, const int b1) {
  long long sum = 0;
  for (int b = b0; b < b1; b++) {
    if (b < a.nfull) for (int s = 0; s < a.nsplits; s++) sum += 4 + (long long)ld_cg_i32(&csizes[(long long)b * a.nsplits + s]);
    else sum += 4 + (long long)ld_cg_i32(&csizes[(long long)a.nfull * a.nsplits]);
  }
  return sum;
}

/* Inclusive prefix sum over the warp */
DEV long long warp_prefix(const long long v) {
  long long incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const long long t = __shfl_up_sync(FULLMASK, incl, d);
    if (lane_id() >= d) incl += t;
  }
  return incl;
}

/* Blocks [b0, b1), the first of which starts at `pos`: writes their bstarts and returns 1 if serial_blosc would give
 * up on one of their splits */
DEV int scan_place(const ScanArgs& a, const int b0, const int b1, long long pos) {
  int bad = 0;
  for (int b = b0; b < b1; b++) {
    a.bstarts[b] = (int)(pos > 0x7fffffffll ? 0x7fffffffll : pos);
    const int ns = b < a.nfull ? a.nsplits : 1;
    const int neblock = b < a.nfull ? a.blocksize / a.nsplits : a.leftover;
    for (int s = 0; s < ns; s++) {
      const long long idx = b < a.nfull ? (long long)b * a.nsplits + s : (long long)a.nfull * a.nsplits;
      const int c = ld_cg_i32(&a.csizes[idx]);
      if (a.serial) {
        /* serial_blosc hands each codec call maxout = min(neblock, room left in dest) (blosc.c:646-651):
         * a clamped call only succeeds if the stream would have fitted that smaller budget, and a
         * raw split needs the full neblock (blosc.c:705-711) */
        const long long room = a.destsize - (pos + 4);
        if (room < neblock && !(room > 0 && c < neblock && ld_cg_i32(&a.needs[idx]) <= room)) bad = 1;
      }
      pos += 4 + (long long)c;
    }
  }
  return bad;
}

/* The block scan of t_blosc's ordered copy-out (blosc.c:1843-1856) by ONE warp: exclusive scan of the
 * per-block compressed sizes -> bstarts, total cbytes and the "does it fit" verdict.  Run by the warp
 * that finishes the last stream of an encode launch, so compression needs no separate scan launch
 * (a 1-CTA launch queues behind the encoders of every other chunk in flight). */
DEV void warp_scan_blocks(const ScanArgs& a) {
  const int lane = lane_id();
  const int nblocks = a.nfull + (a.has_leftover ? 1 : 0);
  const int per = (nblocks + 31) / 32;
  const int b0 = lane * per < nblocks ? lane * per : nblocks, b1 = b0 + per < nblocks ? b0 + per : nblocks;
  const long long sum = scan_sum(a, a.csizes, b0, b1);
  const long long incl = warp_prefix(sum);
  const int bad = scan_place(a, b0, b1, 16 + 4ll * nblocks + (incl - sum));
  const unsigned anybad = __ballot_sync(FULLMASK, bad);
  const long long total = 16 + 4ll * nblocks + __shfl_sync(FULLMASK, incl, 31);
  if (lane == 0) {
    a.result[B2_R_CBYTES] = (int)(total > 0x7fffffffll ? 0x7fffffffll : total);
    a.result[B2_R_FITS] = (total <= a.destsize && anybad == 0u) ? 1 : 0;       /* blosc.c:1848 / :836-839 give up */
  }
}

/* The stream loop of an exact encode launch, for one warp: every stream it draws goes to
 * `codec(idx, in, len, out, &need)`, which writes at most len bytes to out and returns the compressed size.
 * Returns the number of streams this warp finished. */
template <class Codec>
DEV int encode_streams(const EncodeArgs& a, Codec codec) {
  int mine = 0;
  for (;;) {
    const int idx = next_stream(a.queue, a.queue_base, a.map);
    if (idx < 0) break;
    int block, len, split;
    long long off;
    stream_locate(a.map, idx, &block, &off, &len, &split);
    int need = 0;
    int c = codec(idx, a.in + off, len, a.slots + off, &need);
    if (c <= 0 || c >= len) c = len;           /* blosc.c:705-714: incompressible split is stored raw */
    if (lane_id() == 0) { a.csizes[idx] = c; a.needs[idx] = need; }
    mine++;
    __syncwarp();
  }
  return mine;
}

__global__ void encode_kernel(EncodeArgs a) {
#ifdef SIMT_EMU
  u8* smem = simt::g_dynsmem;
#else
  extern __shared__ __align__(16) u8 smem[];
#endif
  const int warp = (int)(threadIdx.x >> 5);
  void* tab = smem + (size_t)warp * a.table_bytes;
  const int mine = encode_streams(a, [&](int, const u8* in, int len, u8* out, int* need) {
    if (a.codec == B2_CODEC_LZ4) {
      if (a.table_bytes == LZ4_TAB17_BYTES) return lz4_encode_warp<false, true>(in, len, out, len, a.accel, tab, need);   /* host guarantees the length range */
      if (len < 65536 + LZ4_MFLIMIT - 1) return lz4_encode_warp<true>(in, len, out, len, a.accel, tab, need);   /* lz4.c:710,1389 */
      return lz4_encode_warp<false>(in, len, out, len, a.accel, tab, need);
    }
    return blz_encode_warp(a.clevel, in, len, out, len, a.split_flag, tab, a.table_bytes, need);
  });
  streams_done(a.done, a.map.nstreams, mine, [&] { if (a.fold_scan) warp_scan_blocks(a.scan); });
}


/* LZ4 in team mode (dev_lz4.cuh): one CTA of four warps per stream -- a walker that owns the parse,
 * the table and the output, and three preparers that work ahead of it.  Shared memory: the stream's
 * hash table, then the Lz4Team block.  The walker warp alone draws tickets, counts finished streams
 * and runs the block scan, exactly as a warp of encode_kernel does. */
#define TEAM_WARPS 4
#define TEAM_CTAS_PER_SM 8
#define TEAM_SMEM_BYTES (LZ4_TABLE_BYTES + ((LZ4T_SMEM_BYTES + 15) & ~15))
#define TEAM_SM_SLOTS 1024
#ifndef SIMT_EMU
__device__ unsigned g_team_sm_seq[TEAM_SM_SLOTS];    /* team CTAs started on each SM so far (wraps; only mod 4 is used) */
#endif
__global__ void __launch_bounds__(TEAM_WARPS * 32, TEAM_CTAS_PER_SM) encode_team_kernel(EncodeArgs a) {
#ifdef SIMT_EMU
  u8* smem = simt::g_dynsmem;
#else
  extern __shared__ __align__(16) u8 smem[];
#endif
  void* tab = smem;
  Lz4Team* tm = (Lz4Team*)(smem + LZ4_TABLE_BYTES);
  const int warp = (int)(threadIdx.x >> 5);
  /* The walker is the busy warp of a team, so the walkers of co-resident teams should run on different SM
   * sub-partitions.  CTAs do not land on the SMs in blockIdx order, so each CTA takes the next slot of its SM from a
   * per-SM counter and makes the warp that runs on that sub-partition (%warpid mod 4) the walker. */
  int walker = (int)((blockIdx.x / (unsigned)(a.num_sms > 0 ? a.num_sms : 1)) & 3u);
#ifndef SIMT_EMU
  if (lane_id() == 0) { unsigned w; asm volatile("mov.u32 %0, %%warpid;" : "=r"(w)); tm->sub[warp] = (int)(w & 3u); }
  if (threadIdx.x == 0) {
    unsigned sm; asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
    tm->slot = (int)(atomicAdd(&g_team_sm_seq[sm % TEAM_SM_SLOTS], 1u) & 3u);
  }
#endif
  if (threadIdx.x == 0) { tm->cmd = 0; tm->gen = 0; }
#ifdef B2_LZ4_CYCLES
  if (threadIdx.x < LZ4C_NREC) tm->cyc[threadIdx.x] = 0;
#endif
  __syncthreads();
#ifndef SIMT_EMU
  for (int k = 3; k >= 0; k--) if (tm->sub[k] == tm->slot) walker = k;
#endif
  if (warp != walker) { lz4_team_preparer(tm, tab, (warp - walker - 1) & 3); return; }
  const int mine = encode_streams(a, [&](int idx, const u8* in, int len, u8* out, int* need) {
    LZ4C_T(c_total);
    const int c = len < 65536 + LZ4_MFLIMIT - 1 ? lz4_encode_warp<true, false, true>(in, len, out, len, a.accel, tab, need, tm)   /* lz4.c:710,1389 */
                                                 : lz4_encode_warp<false, false, true>(in, len, out, len, a.accel, tab, need, tm);
#ifdef B2_LZ4_CYCLES
    {
      const unsigned long long total = (unsigned long long)(clock64() - c_total);
      unsigned smid, wid;
      asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
      asm volatile("mov.u32 %0, %%warpid;" : "=r"(wid));
      __syncwarp();
      const int k = lane_id();
      if (idx < LZ4C_MAXSTREAMS && k < LZ4C_NREC)
        g_lz4_cycles[idx][k] = k == LZ4C_TOTAL ? total : k == LZ4C_SMID ? smid : k == LZ4C_SUBP ? (wid & 3u) : tm->cyc[k];
      __syncwarp();
      if (k < LZ4C_NREC) tm->cyc[k] = 0;
    }
#endif
    return c;
  });
  if (lane_id() == 0) *(volatile int*)&tm->cmd = LZ4T_QUIT;
  __syncwarp();
  __threadfence_block();
  bar_arrive(LZ4T_BAR_GO(0), 64); bar_arrive(LZ4T_BAR_GO(1), 64); bar_arrive(LZ4T_BAR_GO(2), 64);
  streams_done(a.done, a.map.nstreams, mine, [&] { if (a.fold_scan) warp_scan_blocks(a.scan); });
}


/* ---- segment-parallel LZ4 (dev_lz4fast.cuh): index_kernel, parse_kernel ---- */
#define INDEX_WARPS 4
/* one warp per stream, FAST_TAB_BYTES of shared memory each */
__global__ void __launch_bounds__(INDEX_WARPS * 32) index_kernel(FastArgs a) {
#ifdef SIMT_EMU
  u8* smem = simt::g_dynsmem;
#else
  extern __shared__ __align__(16) u8 smem[];
#endif
  const int warp = (int)(threadIdx.x >> 5);
  u32* tab = (u32*)(smem + (size_t)warp * FAST_TAB_BYTES);
  for (int idx = (int)blockIdx.x * INDEX_WARPS + warp; idx < a.map.nstreams; idx += (int)gridDim.x * INDEX_WARPS) {
    int block, len, split;
    long long off;
    stream_locate(a.map, idx, &block, &off, &len, &split);
    lz4f_index_warp(a.in + off, len, a.prev + off, tab, (u32)a.hash_mask);
    __syncwarp();
  }
}

/* One CTA per window of a stream (at most B2_FAST_WIN_MAX bytes): the window's bytes are staged in shared memory, then every THREAD parses one segment of FAST_SEG bytes.
 * Candidate compares -- the random accesses of LZ matching -- hit shared memory; only the chain links (prev[]) and
 * candidates in front of the window come from L2. */
/* ZSTD: the same windows and segments, parsed into zstd sequence records (dev_zstdenc.cuh) instead of LZ4 bytes, with
 * offsets <= MAXD (DZ_MAXD: the DEFLATE encoder, dev_deflate.cuh) */
template <bool ZSTD, int MAXD = 65535>
DEV void fast_parse_body(const FastArgs& a, u8* smem) {
  u32* sdata = (u32*)smem;
  int* sjob = (int*)(smem + a.win_bytes + 48);
  const int tid = (int)threadIdx.x, lane = lane_id();
  const int nfs = a.map.nfull * a.map.nsplits;
  const int njobs = nfs * a.groups_full + a.groups_left;
  const int spw = a.win_bytes / FAST_SEG;         /* segments per window (the CTA has a.threads <= spw threads) */
  for (;;) {
    if (tid == 0) { sjob[0] = (int)((unsigned)atomicAdd(a.queue, 1) - a.queue_base); sjob[1] = 0; }
    __syncthreads();
    const int job = sjob[0];
    if (job >= njobs) break;
    int idx, g, K;
    if (job < a.groups_left) { idx = nfs; g = job; K = a.segs_left; }
    else {
      /* split-major, as next_stream: the byte-planes that turn out to be hard start first */
      const int j = job - a.groups_left;
      const int per_split = a.map.nfull * a.groups_full;
      const int s = j / per_split, r = j - s * per_split;
      const int b = r / a.groups_full;
      g = r - b * a.groups_full;
      idx = b * a.map.nsplits + s; K = a.segs_full;
    }
    int block, len, split;
    long long off;
    stream_locate(a.map, idx, &block, &off, &len, &split);
    FastSeg* segs = ZSTD ? nullptr : a.segs + (long long)idx * a.segs_full;
    FastView v = fast_view(a.in + off, len);
    const int wa = g * a.win_bytes, wb = wa + a.win_bytes < len ? wa + a.win_bytes : len;
    /* stage the 16-byte granules that overlap the window (they lie inside the buffer's allocation: device
     * allocations start and end on coarser boundaries than that) */
    int i_lo = (wa + v.sal) >> 2;
    i_lo -= (int)(((uintptr_t)(v.w + i_lo) & 15u) >> 2);
    const int i_hi = i_lo + ((((wb + v.sal + 3) >> 2) - i_lo + 3) & ~3);
#ifdef SIMT_EMU
    for (int i = i_lo + tid; i < i_hi; i += (int)blockDim.x) sdata[i - i_lo] = (i >= 0 && i < v.nwords) ? v.w[i] : 0u;
#else
    {
      const uint4* g4 = (const uint4*)(v.w + i_lo);
      uint4* s4 = (uint4*)sdata;
      const int n4 = (i_hi - i_lo) >> 2;
#pragma unroll 4
      for (int i = tid; i < n4; i += (int)blockDim.x) s4[i] = __ldg(g4 + i);
    }
#endif
    __syncthreads();
    v.sm = sdata; v.sm_lo = i_lo; v.sm_hi = i_hi;
    v.lo_pos = wa; v.bias = v.sal - 4 * i_lo;      /* position p is byte p + sal - 4 i_lo of the staged words */
    /* the threads draw the window's segments from a counter: a thread whose segment was cheap takes another one
     * instead of waiting at the barrier for the slowest (the CTA may have fewer threads than the window has segments) */
    for (;;) {
      const int t = atomicAdd(&sjob[1], 1);
      const int k = g * spw + t;
      if (t >= spw || k >= K) break;
      const int sa = k * FAST_SEG, sb = sa + FAST_SEG < len ? sa + FAST_SEG : len;
      if (ZSTD) {
        const long long gk = (long long)idx * a.segs_full + k;
        a.nrec[gk] = (u32)zse_parse_lane<MAXD>(v, len, a.prev + off, sa, sb, a.recs + gk * ZE_SEG_RECS, a.depth, a.lazy);
      } else {
        lz4f_parse_lane(v, len, a.prev + off, sa, sb, a.slots + off + sa, &segs[k], a.depth, a.accel, a.lazy);
      }
    }
    __syncthreads();                               /* shared memory may be reused */
  }
}

__global__ void __launch_bounds__(B2_FAST_WIN_MAX / FAST_SEG, 3) parse_kernel(FastArgs a) {
#ifdef SIMT_EMU
  u8* smem = simt::g_dynsmem;
  if (a.codec == B2_CODEC_ZSTD) { fast_parse_body<true>(a, smem); return; }     /* the emulator launches the zstd parse under this name */
  if (a.codec == B2_CODEC_ZLIB) { fast_parse_body<true, DZ_MAXD>(a, smem); return; }   /* and the DEFLATE parse */
  if (a.codec == B2_CODEC_SNAPPY) { fast_parse_body<true>(a, smem); return; }          /* and the snappy encoder's (zparse) */
#else
  extern __shared__ __align__(16) u8 smem[];
#endif
  fast_parse_body<false>(a, smem);
}

/* the zstd and snappy encoders' parse (the backend launches it instead of parse_kernel) */
__global__ void __launch_bounds__(B2_FAST_WIN_MAX / FAST_SEG, 3) zparse_kernel(FastArgs a) {
#ifdef SIMT_EMU
  u8* smem = simt::g_dynsmem;
#else
  extern __shared__ __align__(16) u8 smem[];
#endif
  fast_parse_body<true>(a, smem);
}

/* the DEFLATE encoder's parse, offsets <= 32768 (the backend launches it instead of parse_kernel) */
__global__ void __launch_bounds__(B2_FAST_WIN_MAX / FAST_SEG, 3) dparse_kernel(FastArgs a) {
#ifdef SIMT_EMU
  u8* smem = simt::g_dynsmem;
#else
  extern __shared__ __align__(16) u8 smem[];
#endif
  fast_parse_body<true, DZ_MAXD>(a, smem);
}

/* The stream loop of a segment-parallel back half, for one warp: the warps take the streams in a grid stride, and
 * `codec(idx, off, len)` writes stream idx (bytes [off, off + len) of the input) into at most len bytes of its slot and
 * returns the compressed size.  Returns the number of streams this warp finished. */
template <class Codec>
DEV int fast_streams(const FastArgs& a, Codec codec) {
  const int warp = (int)(threadIdx.x >> 5), nwarps = (int)(blockDim.x >> 5);
  int mine = 0;
  for (int idx = (int)blockIdx.x * nwarps + warp; idx < a.map.nstreams; idx += (int)gridDim.x * nwarps) {
    int block, len, split;
    long long off;
    stream_locate(a.map, idx, &block, &off, &len, &split);
    int c = codec(idx, off, len);
    if (c <= 0 || c >= len) c = len;           /* blosc.c:705-714: incompressible split is stored raw */
    if (lane_id() == 0) { a.csizes[idx] = c; a.needs[idx] = c; }
    mine++;
    __syncwarp();
  }
  return mine;
}

/* One warp per stream: scan of its segment records (pending literals, continued matches, output offsets, compressed
 * size); the warp that finishes the last stream runs the block scan, exactly as in encode_kernel. */
#define FSCAN_WARPS 4
DEV void zenc_body(const FastArgs& a, ZeSm* S);
DEV void denc_body(const FastArgs& a, DzSm* S);
DEV void senc_body(const FastArgs& a);
__global__ void __launch_bounds__(FSCAN_WARPS * 32) fscan_kernel(FastArgs a) {
#ifdef SIMT_EMU
  if (a.codec == B2_CODEC_ZSTD) {                  /* the emulator launches the zstd entropy stage under this name */
    __shared__ ZeSm ztab[FSCAN_WARPS];
    zenc_body(a, &ztab[threadIdx.x >> 5]);
    return;
  }
  if (a.codec == B2_CODEC_ZLIB) {                  /* and the DEFLATE one */
    __shared__ DzSm dtab[FSCAN_WARPS];
    denc_body(a, &dtab[threadIdx.x >> 5]);
    return;
  }
  if (a.codec == B2_CODEC_SNAPPY) { senc_body(a); return; }          /* and the snappy stream writer */
#endif
  const int nfs = a.map.nfull * a.map.nsplits;
  const int mine = fast_streams(a, [&](int idx, long long, int len) {
    int ptail = 0;
    const int c = lz4f_stream_scan(a.segs + (long long)idx * a.segs_full, idx < nfs ? a.segs_full : a.segs_left, len, &ptail);
    if (lane_id() == 0) a.ptail[idx] = ptail;
    return c;
  });
  streams_done(a.done, a.map.nstreams, mine, [&] { if (a.fold_scan) warp_scan_blocks(a.scan); });
}


/* ---- segment-parallel zstd (dev_zstdenc.cuh): index_kernel, zparse_kernel, then one warp per frame ---- */
DEV void zenc_body(const FastArgs& a, ZeSm* S) {
  const int mine = fast_streams(a, [&](int idx, long long off, int len) {
    const long long gseg = (long long)idx * a.segs_full;
    int c = 0;
    if (lane_id() == 0)
      c = zse_frame_serial(*S, a.in + off, len, a.recs + gseg * ZE_SEG_RECS, a.nrec + gseg, (u8*)(a.prev + off), a.slots + off);
    return __shfl_sync(FULLMASK, c, 0);
  });
  streams_done(a.done, a.map.nstreams, mine, [&] { if (a.fold_scan) warp_scan_blocks(a.scan); });
}

/* One warp per stream: its frame, lane 0 codes it; the tables live in the warp's ZE_SMEM_BYTES of shared memory */
__global__ void __launch_bounds__(ZE_WARPS * 32) zenc_kernel(FastArgs a) {
#ifdef SIMT_EMU
  u8* smem = simt::g_dynsmem;
#else
  extern __shared__ __align__(16) u8 smem[];
#endif
  zenc_body(a, (ZeSm*)(smem + (size_t)(threadIdx.x >> 5) * ZE_SMEM_BYTES));
}

/* ---- segment-parallel DEFLATE (dev_deflate.cuh): index_kernel, dparse_kernel, then one warp per zlib stream ---- */
DEV void denc_body(const FastArgs& a, DzSm* S) {
  const int mine = fast_streams(a, [&](int idx, long long off, int len) {
    const long long gseg = (long long)idx * a.segs_full;
    return dz_stream(*S, a.in + off, len, a.recs + gseg * ZE_SEG_RECS, a.nrec + gseg, (u8*)(a.prev + off), a.slots + off, a.flevel);
  });
  streams_done(a.done, a.map.nstreams, mine, [&] { if (a.fold_scan) warp_scan_blocks(a.scan); });
}

/* One warp per stream: its zlib stream; the tables and the bit window live in the warp's DZ_SMEM_BYTES */
__global__ void __launch_bounds__(DZ_WARPS * 32) denc_kernel(FastArgs a) {
#ifdef SIMT_EMU
  u8* smem = simt::g_dynsmem;
#else
  extern __shared__ __align__(16) u8 smem[];
#endif
  denc_body(a, (DzSm*)(smem + (size_t)(threadIdx.x >> 5) * DZ_SMEM_BYTES));
}


/* ---- snappy (dev_snappy.cuh): index_kernel, zparse_kernel, then one warp per snappy stream ---- */
/* snappy_max_compressed_length (snappy.cc MaxCompressedLength): the output room blosc_c asks for (blosc.c:640-645) */
DEV long long sn_bound(int n) { return 32 + (long long)n + n / 6; }

/* The block scan of warp_scan_blocks with blosc_c's snappy maxout rule in front, by ONE warp.  blosc_c hands snappy
 * maxout = snappy_max_compressed_length(neblock), clamped to the room left (blosc.c:640-651), and snappy_compress
 * refuses any smaller buffer: a split whose room is below that bound is stored raw if neblock still fits (:705-714),
 * and otherwise the call gives up.  The room is measured from the stream's own sizes:
 *   - pool (t_blosc, !serial): per block, from 0 with maxbytes = ebsize (blosc.c:1745,1810);
 *   - serial: from the chunk's start with maxbytes = destsize.  The first split short of its bound is found on the
 *     compressed sizes; from there on every full split is short of it too (the room only shrinks), so they become
 *     raw, and the leftover split is judged at its new position.
 * Raw splits get csizes = their length, so compaction copies them from the input (`csizes` is a.csizes, writable). */
#ifdef SIMT_EMU
static int* g_sn_presizes = nullptr;          /* emulator builds: where to copy the stream sizes the rule starts from */
static int g_sn_presizes_cap = 0;
#endif
DEV void warp_scan_blocks_snappy(const ScanArgs& a, int* csizes, const int ebsize) {
  const int lane = lane_id();
  const int nblocks = a.nfull + (a.has_leftover ? 1 : 0);
#ifdef SIMT_EMU
  {
    const int ns = a.nfull * a.nsplits + (a.has_leftover ? 1 : 0);
    if (lane == 0 && g_sn_presizes) for (int i = 0; i < ns && i < g_sn_presizes_cap; i++) g_sn_presizes[i] = csizes[i];
    __syncwarp();
  }
#endif
  const int per = (nblocks + 31) / 32;
  const int b0 = lane * per < nblocks ? lane * per : nblocks, b1 = b0 + per < nblocks ? b0 + per : nblocks;
  int bad = 0;
  if (!a.serial) {
    for (int b = b0; b < b1; b++) {
      const int ns = b < a.nfull ? a.nsplits : 1;
      const int neblock = b < a.nfull ? a.blocksize / a.nsplits : a.leftover;
      long long nt = 0;
      for (int s = 0; s < ns; s++) {
        const long long idx = b < a.nfull ? (long long)b * a.nsplits + s : (long long)a.nfull * a.nsplits;
        int c = ld_cg_i32(&csizes[idx]);
        nt += 4;
        const long long room = ebsize - nt;
        if (room < sn_bound(neblock)) {
          if (room >= neblock) { if (c != neblock) { c = neblock; csizes[idx] = c; } }
          else bad = 1;
        }
        nt += c;
      }
    }
  }
  long long first = 0x7fffffffffffffffll;     /* serial: the first split short of its bound */
  long long pos0 = 0, total = 0;
  for (int pass = 0; pass < 2; pass++) {
    const long long sum = scan_sum(a, csizes, b0, b1);
    const long long incl = warp_prefix(sum);
    pos0 = 16 + 4ll * nblocks + (incl - sum);
    total = 16 + 4ll * nblocks + __shfl_sync(FULLMASK, incl, 31);
    if (!a.serial || pass == 1) break;
    long long pos = pos0, mine = first;
    for (int b = b0; b < b1 && mine == first; b++) {
      const int ns = b < a.nfull ? a.nsplits : 1;
      const int neblock = b < a.nfull ? a.blocksize / a.nsplits : a.leftover;
      for (int s = 0; s < ns; s++) {
        const long long idx = b < a.nfull ? (long long)b * a.nsplits + s : (long long)a.nfull * a.nsplits;
        if (a.destsize - (pos + 4) < sn_bound(neblock)) { mine = idx; break; }
        pos += 4 + (long long)ld_cg_i32(&csizes[idx]);
      }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
      const long long t = __shfl_xor_sync(FULLMASK, mine, d);
      mine = t < mine ? t : mine;
    }
    first = mine;
    if (first == 0x7fffffffffffffffll) break;
    for (int b = b0 < a.nfull ? b0 : a.nfull; b < b1 && b < a.nfull; b++)
      for (int s = 0; s < a.nsplits; s++) {
        const long long idx = (long long)b * a.nsplits + s;
        if (idx >= first) csizes[idx] = a.blocksize / a.nsplits;
      }
  }
  long long pos = pos0, grow = 0;
  for (int b = b0; b < b1; b++) {
    a.bstarts[b] = (int)(pos > 0x7fffffffll ? 0x7fffffffll : pos);
    const int ns = b < a.nfull ? a.nsplits : 1;
    const int neblock = b < a.nfull ? a.blocksize / a.nsplits : a.leftover;
    for (int s = 0; s < ns; s++) {
      const long long idx = b < a.nfull ? (long long)b * a.nsplits + s : (long long)a.nfull * a.nsplits;
      int c = ld_cg_i32(&csizes[idx]);
      if (a.serial && idx >= first) {
        const long long room = a.destsize - (pos + 4);
        if (room < sn_bound(neblock)) {
          if (room >= neblock) { if (c != neblock) { grow += neblock - c; c = neblock; csizes[idx] = c; } }   /* only the leftover split can still change */
          else bad = 1;
        }
      }
      pos += 4 + (long long)c;
    }
  }
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) grow += __shfl_xor_sync(FULLMASK, grow, d);
  total += grow;
  const unsigned anybad = __ballot_sync(FULLMASK, bad);
  if (lane == 0) {
    a.result[B2_R_CBYTES] = (int)(total > 0x7fffffffll ? 0x7fffffffll : total);
    a.result[B2_R_FITS] = (total <= a.destsize && anybad == 0u) ? 1 : 0;       /* blosc.c:1848 / :836-839 give up */
  }
}

/* One warp per stream: its snappy stream; whoever completes the stream count runs the snappy block scan */
#define SN_WARPS 4
DEV void senc_body(const FastArgs& a) {
  const int mine = fast_streams(a, [&](int idx, long long off, int len) {
    const long long gseg = (long long)idx * a.segs_full;
    return sn_stream(a.in + off, len, a.recs + gseg * ZE_SEG_RECS, a.nrec + gseg, (u8*)(a.prev + off), a.slots + off);
  });
  /* (always folded: the host never launches scan_kernel for snappy) */
  streams_done(a.done, a.map.nstreams, mine, [&] { warp_scan_blocks_snappy(a.scan, a.csizes, a.ebsize); });
}

__global__ void __launch_bounds__(SN_WARPS * 32) senc_kernel(FastArgs a) { senc_body(a); }

#define SCAN_THREADS 1024
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(ScanArgs a) {
  __shared__ long long part[SCAN_THREADS];
  const int tid = (int)threadIdx.x;
  const int nblocks = a.nfull + (a.has_leftover ? 1 : 0);
  const int per = (nblocks + SCAN_THREADS - 1) / SCAN_THREADS;
  const int b0 = tid * per, b1 = b0 + per < nblocks ? b0 + per : nblocks;
  part[tid] = scan_sum(a, a.csizes, b0, b1);
  __syncthreads();
  /* Hillis-Steele inclusive scan over the 1024 partials */
  for (int d = 1; d < SCAN_THREADS; d <<= 1) {
    const long long v = tid >= d ? part[tid - d] : 0;
    __syncthreads();
    part[tid] += v;
    __syncthreads();
  }
  /* the status word, zero between calls, collects the threads' give-up verdicts */
  if (scan_place(a, b0, b1, 16 + 4ll * nblocks + (tid ? part[tid - 1] : 0))) atomicOr(&a.result[B2_R_STATUS], 1);
  __syncthreads();
  if (tid == SCAN_THREADS - 1) {
    const long long total = 16 + 4ll * nblocks + part[SCAN_THREADS - 1];
    a.result[B2_R_CBYTES] = (int)(total > 0x7fffffffll ? 0x7fffffffll : total);
    a.result[B2_R_FITS] = (total <= a.destsize && a.result[B2_R_STATUS] == 0) ? 1 : 0;   /* blosc.c:1848 / :836-839 give up */
    a.result[B2_R_STATUS] = 0;
  }
}

/* CTA-cooperative copy, any alignment; vectorised when src/dst are mutually aligned */
DEV void cta_copy_bytes(u8* __restrict__ dst, const u8* __restrict__ src, int n) {
  const int tid = (int)threadIdx.x, nt = (int)blockDim.x;
  if ((((uintptr_t)dst ^ (uintptr_t)src) & 15u) == 0 && n >= 64) {
    int head = (int)((16u - ((uintptr_t)dst & 15u)) & 15u);
    if (head > n) head = n;
    for (int i = tid; i < head; i += nt) dst[i] = src[i];
    const int nv = (n - head) >> 4;
    const uint4* s4 = (const uint4*)(src + head);
    uint4* d4 = (uint4*)(dst + head);
    for (int i = tid; i < nv; i += nt) d4[i] = s4[i];
    for (int i = head + (nv << 4) + tid; i < n; i += nt) dst[i] = src[i];
  } else {
    for (int i = tid; i < n; i += nt) dst[i] = src[i];
  }
}


#define COMPACT_THREADS 256
__global__ void __launch_bounds__(COMPACT_THREADS) compact_kernel(CompactArgs a) {
  if (a.result[1] == 0) return;                 /* does not fit: host falls back to a MEMCPYED chunk */
  const int tid = (int)threadIdx.x;
  if (blockIdx.x == 0 && tid == 0) {            /* blosc.c:1154-1215 + :1275 */
    st_u32_bytes(a.dest, a.hdr0);
    st_u32_bytes(a.dest + 4, (u32)a.nbytes32);
    st_u32_bytes(a.dest + 8, (u32)a.map.blocksize);
    st_u32_bytes(a.dest + 12, (u32)a.result[0]);
  }
  for (int b = (int)blockIdx.x; b < a.nblocks; b += (int)gridDim.x) {
    int pos = a.bstarts[b];
    if (tid == 0) st_u32_bytes(a.dest + 16 + 4ll * b, (u32)pos);     /* blosc.c:816,1847 */
    const int ns = b < a.map.nfull ? a.map.nsplits : 1;
    for (int s = 0; s < ns; s++) {
      const int idx = b < a.map.nfull ? b * a.map.nsplits + s : a.map.nfull * a.map.nsplits;
      int blk, len, sp;
      long long off;
      stream_locate(a.map, idx, &blk, &off, &len, &sp);
      const int c = a.csizes[idx];
      if (tid == 0) st_u32_bytes(a.dest + pos, (u32)c);               /* blosc.c:715 */
      if (a.segs && c != len)
        lz4f_stitch_cta(a.dest + pos + 4, c, a.in + off, len, a.slots + off, a.segs + (long long)idx * a.segs_full,
                        b < a.map.nfull ? a.segs_full : a.segs_left, a.ptail[idx]);
      else cta_copy_bytes(a.dest + pos + 4, (c == len ? a.in : a.slots) + off, c);
      pos += 4 + c;
    }
  }
}


/* byte-wise: the size prefixes may sit in the last bytes of a caller-owned device chunk, and the
 * word-pair form of ld_u32 would touch up to 3 bytes past cbytes */
DEV int ld_i32(const u8* p) { return (int)((u32)p[0] | ((u32)p[1] << 8) | ((u32)p[2] << 16) | ((u32)p[3] << 24)); }

/* The stream loop of a decode launch, for one warp: every stream it draws is located by walking the size prefixes of
 * its block up to its split (blosc.c:760-771, :784), then copied if stored raw (:773-776) or handed to
 * `codec(src, cs, out, len)`, which returns the decoded size (:778-782).  Failures go to a.status; the warp that
 * completes the stream count publishes it to status_out and puts the counters back to zero. */
template <class Codec>
DEV void decode_streams(const DecodeArgs& a, Codec codec) {
  int mine = 0;
  for (;;) {
    const int idx = next_stream(a.queue, a.queue_base, a.map);
    if (idx < 0) break;
    int block, len, split;
    long long off;
    stream_locate(a.map, idx, &block, &off, &len, &split, a.blocks);
    int so = ld_i32(a.chunk + 16 + 4ll * block);
    int cs = 0, err = 0;
    for (int s = 0; s <= split; s++) {
      if (so < 0 || so > a.cbytes - 4) { err = B2_ERR_BOUNDS; break; }
      cs = ld_i32(a.chunk + so);
      so += 4;
      if (cs < 0 || cs > a.cbytes - so) { err = B2_ERR_BOUNDS; break; }
      if (s < split) so += cs;
    }
    if (!err) {
      u8* out = a.out + (off - a.out_shift);
      const u8* src = a.chunk + so;
      if (cs == len) warp_copy_bytes(out, src, len);                    /* stored raw */
      else if (codec(src, cs, out, len) != len) err = B2_ERR_CODEC;
    }
    if (err && lane_id() == 0) atomicMin(a.status, err);
    mine++;
    __syncwarp();
  }
  streams_done(a.done, a.map.nstreams, mine, [&] {
    if (lane_id() == 0) { *a.status_out = ld_cg_i32(a.status); *a.status = 0; }
  });
}

#define DECODE_WARPS 4
/* dynamic shared memory: DECODE_WARPS * LZ4D_SMEM bytes (per-warp ring of recent output) */
/* One instantiation per codec: the bit-serial inflate must not cost the LZ decoders registers,
 * stack or instruction-cache footprint. */
template <int CODEC>
__global__ void __launch_bounds__(DECODE_WARPS * 32) decode_kernel(DecodeArgs a) {
#ifdef SIMT_EMU
  u8* smem = simt::g_dynsmem;
#else
  extern __shared__ __align__(16) u8 smem[];
#endif
  u8* wsmem = smem + (size_t)(threadIdx.x >> 5) * LZ4D_SMEM;
  decode_streams(a, [&](const u8* src, int cs, u8* out, int len) {
    if (CODEC == B2_CODEC_LZ4) return lz4_decode_warp(src, cs, out, len, wsmem);
    if (CODEC == B2_CODEC_ZLIB) return zlib_decode_warp(src, cs, out, len, wsmem);
    if (CODEC == B2_CODEC_ZSTD) return zstd_decode_warp(src, cs, out, len, wsmem);
    if (CODEC == B2_CODEC_SNAPPY) return snappy_decode_warp(src, cs, out, len, wsmem);
#ifdef SIMT_EMU
    if (a.codec == B2_CODEC_SNAPPY) return snappy_decode_warp(src, cs, out, len, wsmem);   /* the emulator launches it as decode_kernel<0> */
#endif
    return blz_decode_warp(src, cs, out, len);
  });
}


/* getitems: copies every requested range out of the compact scratch that one decode (and unfilter) launch made of
 * the touched blocks.  Work is cut by bytes, not by range, so a long range does not serialise the launch: warp job k
 * covers bytes [k * GATHER_SPAN, (k + 1) * GATHER_SPAN) of the concatenated ranges and binary-searches the prefix of
 * range lengths for its first range.  Each piece is copied 16 bytes per lane when source and destination share their
 * alignment mod 16, bytewise at the edges and otherwise. */
#define GATHER_WARPS 8
#define GATHER_SPAN 8192
DEV void warp_copy_vec(u8* __restrict__ dst, const u8* __restrict__ src, int n) {
  const int lane = lane_id();
  if ((((uintptr_t)dst ^ (uintptr_t)src) & 15u) == 0 && n >= 32) {
    const int head = (int)((16u - ((uintptr_t)dst & 15u)) & 15u);
    if (lane < head) dst[lane] = src[lane];
    const int nv = (n - head) >> 4;
    const uint4* s4 = (const uint4*)(src + head);
    uint4* d4 = (uint4*)(dst + head);
    for (int i = lane; i < nv; i += 32) d4[i] = s4[i];
    for (int i = head + (nv << 4) + lane; i < n; i += 32) dst[i] = src[i];
  } else {
    for (int i = lane; i < n; i += 32) dst[i] = src[i];
  }
}

/* The block-mapped copy of the N-d gathers: bytes [s, s + n) of a chunk (chunk offsets are below 2^31, blocks of bs
 * bytes) to out.  With slot NULL the chunk is read in place at src; else only its touched blocks were decoded, into
 * the compact scratch at src, block b at slot[b] * bs.  slot_copy_warp is the whole warp's copy, one warp_copy_vec per
 * piece, each piece cut at block edges; slot_copy_lane is one lane's, bytewise, reading slot[] again only when it
 * crosses a block edge. */
DEV void slot_copy_warp(u8* out, const u8* src, const int* slot, unsigned bs, unsigned s, long long n) {
  while (n > 0) {
    int m = (int)n;
    const u8* from = src + s;
    if (slot) {
      const unsigned blk = s / bs, left = (blk + 1) * bs - s;
      if ((unsigned)m > left) m = (int)left;
      from = src + (long long)slot[blk] * bs + (s - blk * bs);
    }
    warp_copy_vec(out, from, m);
    out += m; s += (unsigned)m; n -= m;
  }
}

DEV void slot_copy_lane(u8* out, const u8* src, const int* slot, unsigned bs, unsigned s, int n) {
  if (!slot) {
    for (int x = 0; x < n; x++) out[x] = src[s + x];
    return;
  }
  unsigned bend = 0;
  const u8* base = src;
  for (int x = 0; x < n; x++, s++) {
    if (s >= bend) {
      const unsigned blk = s / bs;
      bend = (blk + 1) * bs;
      base = src + (long long)slot[blk] * bs - (long long)blk * bs;
    }
    out[x] = base[s];
  }
}

__global__ void __launch_bounds__(GATHER_WARPS * 32) gather_kernel(GatherArgs a) {
  if (a.status && ld_cg_i32(a.status) < 0) return;       /* a stream failed to decode: dest stays untouched */
  const long long warps = (long long)gridDim.x * GATHER_WARPS;
  for (long long lo = ((long long)blockIdx.x * GATHER_WARPS + (threadIdx.x >> 5)) * GATHER_SPAN; lo < a.total;
       lo += warps * GATHER_SPAN) {
    const long long hi = lo + GATHER_SPAN < a.total ? lo + GATHER_SPAN : a.total;
    int l = 0, h = a.nranges - 1;                          /* the last range with pos <= lo */
    while (l < h) {
      const int m = (l + h + 1) >> 1;
      if (a.ranges[m].pos <= lo) l = m; else h = m - 1;
    }
    for (int r = l; r < a.nranges; r++) {
      const GatherRange g = a.ranges[r];
      if (g.pos >= hi) break;
      const long long end = a.ranges[r + 1].pos;
      const long long p0 = lo > g.pos ? lo : g.pos, p1 = hi < end ? hi : end;
      warp_copy_vec(a.dst + g.dst + (p0 - g.pos), a.src + g.src + (p0 - g.pos), (int)(p1 - p0));
    }
  }
}

#ifdef SIMT_EMU
/* The CPU emulator's launcher of gather_kernel (the other kernels are launched by tests/emu/backend_emu.cpp, which
 * includes this header): a few CTAs, so that every warp goes through several spans.  It counts its own launches. */
static long long g_emu_gather_launches = 0;
static unsigned emu_gather_ctas(long long total) {
  const long long ctas = (total + (long long)GATHER_WARPS * GATHER_SPAN - 1) / ((long long)GATHER_WARPS * GATHER_SPAN);
  return (unsigned)(ctas > 3 ? 3 : ctas);
}
extern "C" int b2_launch_gather(const GatherArgs* a, b2_stream_t) {
  if (a->total <= 0) return 0;
  g_emu_gather_launches++;
  GatherArgs args = *a;
  simt::launch(simt::Dim3(emu_gather_ctas(a->total)), simt::Dim3(GATHER_WARPS * 32), 0, [&] { gather_kernel(args); });
  return 0;
}
#endif


/* getitems planned on the GPU (PlanArgs), for range lists in device memory: the same gather table and block list the
 * host plan builds, with no copy of the lists to the host.  plan_check_kernel, one thread per range: blosc_getitem's
 * checks (b2_range_check), the first failing index by atomicMin, each range's byte length, and its block interval
 * marked in a difference array (+1 at the first block, -1 after the last), so a whole-chunk range costs two atomics. */
__global__ void __launch_bounds__(PLAN_THREADS) plan_check_kernel(PlanArgs a) {
  for (long long r = (long long)blockIdx.x * PLAN_THREADS + threadIdx.x; r < a.nranges;
       r += (long long)gridDim.x * PLAN_THREADS) {
    long long lo = 0, hi = 0;
    if (b2_range_check(a.starts[r], a.nitems[r], a.typesize, a.nbytes, &lo, &hi)) {
      atomicMin(&a.rec->bad, (unsigned)r);
      a.len[r] = 0;
      continue;
    }
    const long long n = hi > lo ? hi - lo : 0;
    a.len[r] = n;
    if (n > 0 && !a.in_place) {
      atomicAdd(a.cover + lo / a.blocksize, 1);
      atomicAdd(a.cover + (hi - 1) / a.blocksize + 1, -1);
    }
  }
}

/* The frame plan (FramePlanArgs) in front of the chunk plan, for frame range lists in device memory.
 * fplan_check_kernel, one thread per range: the frame's check (b2_frame_range_bad), the first failing index by
 * atomicMin, each range's byte length, and its chunk interval marked in a difference array, as plan_check_kernel marks
 * blocks.  An empty range touches no chunk. */
__global__ void __launch_bounds__(PLAN_THREADS) fplan_check_kernel(FramePlanArgs a) {
  const unsigned long long ipc = (unsigned long long)a.ipc;
  for (long long r = (long long)blockIdx.x * PLAN_THREADS + threadIdx.x; r < a.nranges;
       r += (long long)gridDim.x * PLAN_THREADS) {
    const unsigned long long s = a.starts ? a.starts[r] : 0, n = a.nitems[r];
    if (b2_frame_range_bad(s, n, a.total_items)) {
      atomicMin(&a.rec->bad, (unsigned long long)r);
      a.dst[r] = 0;
      continue;
    }
    a.dst[r] = (long long)n * a.typesize;
    if (n > 0) {
      atomicAdd((unsigned long long*)a.count + s / ipc, 1ull);
      atomicAdd((unsigned long long*)a.count + (s + n - 1) / ipc + 1, ~0ull);
    }
  }
}

/* fplan_scatter_kernel, one thread per range, once the scans have run: the range's pieces, one per chunk it touches,
 * each into a slot of its chunk's bucket taken from the chunk's cursor.  The order inside a bucket depends on timing;
 * every piece carries its own dest offset, so the bytes written do not. */
__global__ void __launch_bounds__(PLAN_THREADS) fplan_scatter_kernel(FramePlanArgs a) {
  const unsigned long long ipc = (unsigned long long)a.ipc;
  for (long long r = (long long)blockIdx.x * PLAN_THREADS + threadIdx.x; r < a.nranges;
       r += (long long)gridDim.x * PLAN_THREADS) {
    const unsigned long long end = a.starts[r] + a.nitems[r];
    long long dst = a.dst[r];
    for (unsigned long long at = a.starts[r], c = at / ipc; at < end; c++) {
      const unsigned long long stop = (c + 1) * ipc < end ? (c + 1) * ipc : end;
      const long long slot = (long long)atomicAdd((unsigned long long*)a.cursor + c, 1ull);
      a.pstart[slot] = (int)(at - c * ipc);
      a.pnitems[slot] = (int)(stop - at);
      a.pdst[slot] = dst;
      dst += (long long)(stop - at) * a.typesize;
      at = stop;
    }
  }
}

/* The scans of the plans, one device-wide exclusive scan each.  Chunk plan: PLAN_COVER turns the difference array into
 * each block's coverage (in place), PLAN_SLOT numbers the covered blocks and lists them, PLAN_POS makes each range's
 * position from its length and writes its gather entry.  Frame plan: FPLAN_DST makes each range's offset in dest from
 * its length (in place), FPLAN_COUNT turns the difference array into each chunk's pieces (in place), FPLAN_BASE makes
 * each chunk's bucket base (its cursor) and FPLAN_TOUCH lists the chunks with pieces. */
template <int MODE> struct PlanVal { typedef long long T; };
template <> struct PlanVal<PLAN_COVER> { typedef int T; };
template <> struct PlanVal<PLAN_SLOT> { typedef int T; };

template <int MODE> DEV typename PlanVal<MODE>::T plan_load(const PlanArgs& a, long long i) {
  if constexpr (MODE == PLAN_COVER) return a.cover[i];
  else if constexpr (MODE == PLAN_SLOT) return a.cover[i] > 0;
  else return a.len[i];
}

template <int MODE, typename T> DEV void plan_store(const PlanArgs& a, long long i, long long n, T excl, T x) {
  if constexpr (MODE == PLAN_COVER) {
    a.cover[i] = excl + x;
  } else if constexpr (MODE == PLAN_SLOT) {
    if (x) { a.slot[i] = excl; a.blocks[excl] = (int)i; }
    if (i == n - 1) { a.rec->nlisted = excl + x; a.rec->has_left = x && a.leftover; }
  } else {
    GatherRange g;
    g.pos = excl;
    g.dst = a.dsts ? a.dsts[i] : excl;
    g.src = 0;
    if (x > 0) {                       /* where the range starts in the gather's source */
      const long long lo = (long long)a.starts[i] * a.typesize;
      if (a.in_place) g.src = lo;
      else {
        const long long first = lo / a.blocksize;
        g.src = (long long)a.slot[first] * a.blocksize + (lo - first * a.blocksize);
      }
    }
    a.ranges[i] = g;
    if (i == n - 1) {
      GatherRange e;
      e.src = e.dst = 0; e.pos = excl + x;
      a.ranges[n] = e;
      a.rec->total = excl + x;
    }
  }
}

template <int MODE> DEV long long plan_load(const FramePlanArgs& a, long long i) {
  if constexpr (MODE == FPLAN_DST) return a.dst[i];
  else if constexpr (MODE == FPLAN_TOUCH) return a.count[i] > 0;
  else return a.count[i];
}

template <int MODE, typename T> DEV void plan_store(const FramePlanArgs& a, long long i, long long n, T excl, T x) {
  if constexpr (MODE == FPLAN_DST) {
    a.dst[i] = excl;
    if (i == n - 1) a.rec->total = excl + x;
  } else if constexpr (MODE == FPLAN_COUNT) {
    a.count[i] = excl + x;
  } else if constexpr (MODE == FPLAN_BASE) {
    a.cursor[i] = excl;
    if (i == n - 1) a.rec->npieces = excl + x;
  } else {
    if (x) {
      FrameTouch t;
      t.chunk = i; t.base = a.cursor[i]; t.count = a.count[i];
      a.touched[excl] = t;
    }
    if (i == n - 1) a.rec->ntouched = excl + x;
  }
}

/* Single pass with decoupled look-back: each CTA takes the next tile (PLAN_TILE items, PLAN_ITEMS consecutive ones
 * per thread) from a counter, so the tiles before it have started; it publishes its aggregate, then warp 0 walks back
 * 32 tiles at a time, summing aggregates up to the nearest tile that has published its inclusive prefix.  A is
 * PlanArgs or FramePlanArgs, whose tile states are indexed from PLAN_COVER and FPLAN_DST. */
template <int MODE, class A>
__global__ void __launch_bounds__(PLAN_THREADS) plan_scan_kernel(A a, long long n) {
  typedef typename PlanVal<MODE>::T T;
  const PlanScan& st = a.scan[MODE < FPLAN_DST ? MODE : MODE - FPLAN_DST];
  __shared__ T s_warp[PLAN_THREADS / 32];
  __shared__ T s_prefix;
  __shared__ unsigned s_tile;
  const int lane = lane_id(), warp = (int)(threadIdx.x >> 5);
  if (threadIdx.x == 0) s_tile = atomicAdd(st.ticket, 1u);
  __syncthreads();
  const long long tile = s_tile;
  const long long base = tile * PLAN_TILE + (long long)threadIdx.x * PLAN_ITEMS;
  T v[PLAN_ITEMS], sum = 0;
#pragma unroll
  for (int k = 0; k < PLAN_ITEMS; k++) {
    v[k] = base + k < n ? plan_load<MODE>(a, base + k) : (T)0;
    sum += v[k];
  }
  T inc = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const T t = __shfl_up_sync(FULLMASK, inc, d);
    if (lane >= d) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    T* agg = (T*)st.agg;
    T* incl = (T*)st.inc;
    volatile unsigned* flag = st.flag;
    const T w = lane < PLAN_THREADS / 32 ? s_warp[lane] : (T)0;
    T wi = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const T t = __shfl_up_sync(FULLMASK, wi, d);
      if (lane >= d) wi += t;
    }
    const T total = __shfl_sync(FULLMASK, wi, 31);
    if (lane < PLAN_THREADS / 32) s_warp[lane] = wi - w;
    if (lane == 0) {
      if (tile == 0) { incl[0] = total; __threadfence(); flag[0] = 2; }
      else { agg[tile] = total; __threadfence(); flag[tile] = 1; }
    }
    T prefix = 0;
    if (tile > 0) {
      for (long long p = tile - 1;; p -= 32) {
        const long long q = p - lane;
        unsigned f = 2;
        T val = 0;
        if (q >= 0) {
          while ((f = flag[q]) == 0) {}
          __threadfence();
          val = f == 2 ? ((volatile T*)incl)[q] : ((volatile T*)agg)[q];
        }
        const unsigned done = __ballot_sync(FULLMASK, f == 2);
        const int stop = done ? __ffs((int)done) - 1 : 31;     /* lanes up to the nearest inclusive prefix count */
        T c = lane <= stop ? val : (T)0;
#pragma unroll
        for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(FULLMASK, c, d);
        prefix += c;
        if (done) break;
      }
      if (lane == 0) { incl[tile] = prefix + total; __threadfence(); flag[tile] = 2; }
    }
    if (lane == 0) s_prefix = prefix;
  }
  __syncthreads();
  T excl = s_prefix + s_warp[warp] + inc - sum;
#pragma unroll
  for (int k = 0; k < PLAN_ITEMS; k++) {
    if (base + k < n) plan_store<MODE, T>(a, base + k, n, excl, v[k]);
    excl += v[k];
  }
}

#ifdef SIMT_EMU
/* The emulator's launcher of the plan kernels: a few CTAs for the per-range check, so that the grid-stride loop runs;
 * every tile of a scan is its own CTA, as on the GPU.  The emulator has one device. */
static long long g_emu_plan_launches = 0;
static unsigned emu_tiles(long long n) { return (unsigned)((n + PLAN_TILE - 1) / PLAN_TILE); }
static unsigned emu_range_ctas(long long n) { return (unsigned)(n > 2 * PLAN_THREADS ? 3 : (n + PLAN_THREADS - 1) / PLAN_THREADS); }
/* the PLAN_SLOT scan over a chunk plan's blocks, one plan launch */
static void emu_slot_scan(const PlanArgs& plan) {
  const long long nb = plan.nblocks;
  simt::launch(simt::Dim3(emu_tiles(nb)), simt::Dim3(PLAN_THREADS), 0, [&] { plan_scan_kernel<PLAN_SLOT>(plan, nb); });
  g_emu_plan_launches++;
}
extern "C" int b2_launch_plan(const PlanArgs* a, b2_stream_t) {
  if (a->nranges <= 0) return 0;
  PlanArgs args = *a;
  const long long nb = a->nblocks, nr = a->nranges;
  simt::launch(simt::Dim3(emu_range_ctas(nr)), simt::Dim3(PLAN_THREADS), 0, [&] { plan_check_kernel(args); });
  g_emu_plan_launches++;
  if (!a->in_place) {
    simt::launch(simt::Dim3(emu_tiles(nb)), simt::Dim3(PLAN_THREADS), 0, [&] { plan_scan_kernel<PLAN_COVER>(args, nb); });
    g_emu_plan_launches++;
    emu_slot_scan(args);
  }
  simt::launch(simt::Dim3(emu_tiles(nr)), simt::Dim3(PLAN_THREADS), 0, [&] { plan_scan_kernel<PLAN_POS>(args, nr); });
  g_emu_plan_launches++;
  return 0;
}

/* ... and of the frame plan's kernels, the same way; they count as plan launches */
extern "C" int b2_launch_fplan(const FramePlanArgs* a, b2_stream_t) {
  if (a->nranges <= 0) return 0;
  FramePlanArgs args = *a;
  const long long nr = a->nranges, nc = a->nchunks;
  simt::launch(simt::Dim3(emu_range_ctas(nr)), simt::Dim3(PLAN_THREADS), 0, [&] { fplan_check_kernel(args); });
  simt::launch(simt::Dim3(emu_tiles(nr)), simt::Dim3(PLAN_THREADS), 0, [&] { plan_scan_kernel<FPLAN_DST>(args, nr); });
  g_emu_plan_launches += 2;
  if (nc > 0) {
    simt::launch(simt::Dim3(emu_tiles(nc)), simt::Dim3(PLAN_THREADS), 0, [&] { plan_scan_kernel<FPLAN_COUNT>(args, nc); });
    simt::launch(simt::Dim3(emu_tiles(nc)), simt::Dim3(PLAN_THREADS), 0, [&] { plan_scan_kernel<FPLAN_BASE>(args, nc); });
    simt::launch(simt::Dim3(emu_tiles(nc)), simt::Dim3(PLAN_THREADS), 0, [&] { plan_scan_kernel<FPLAN_TOUCH>(args, nc); });
    g_emu_plan_launches += 3;
  }
  return 0;
}
extern "C" int b2_launch_fplan_scatter(const FramePlanArgs* a, b2_stream_t) {
  if (a->nranges <= 0) return 0;
  FramePlanArgs args = *a;
  simt::launch(simt::Dim3(emu_range_ctas(a->nranges)), simt::Dim3(PLAN_THREADS), 0, [&] { fplan_scatter_kernel(args); });
  g_emu_plan_launches++;
  return 0;
}
extern "C" int b2_ptr_device(const void*) { return 0; }
#endif


/* blosc_b200_getslice: a box of an N-d array (B2Box), planned and gathered from the box alone, with no per-run state.
 * Both kernels come in two instantiations, STEPPED = the box's `stepped`: the step-1 one compiles the box arithmetic
 * without its step code.  box_touch_kernel, one thread per block of the chunk: the block is touched when some box item
 * has a byte in it.  The test is on bytes, so it holds when the blocksize is not a multiple of the typesize, and a step
 * that jumps over whole blocks leaves them untouched. */
template <bool STEPPED>
__global__ void __launch_bounds__(PLAN_THREADS) box_touch_kernel(BoxPlanArgs a) {
  const long long ts = a.plan.typesize, bs = a.plan.blocksize;
  for (long long b = (long long)blockIdx.x * PLAN_THREADS + threadIdx.x; b < a.plan.nblocks;
       b += (long long)gridDim.x * PLAN_THREADS) {
    const long long lo = b * bs, hi = lo + bs < a.plan.nbytes ? lo + bs : a.plan.nbytes;
    a.plan.cover[b] = b2_box_next(&a.box, a.window + b2_box_div(lo, ts), STEPPED) < a.window + b2_box_div(hi + ts - 1, ts);
  }
}

/* box_gather_kernel: output-driven like gather_kernel, warp job k covering output bytes [k * GATHER_SPAN, (k + 1) *
 * GATHER_SPAN).  Runs of BOX_SHORT_RUN bytes or more are copied by the whole warp (slot_copy_warp).  Shorter runs are
 * copied by one lane each (slot_copy_lane): lane l takes every 32nd run that starts in the job's
 * bytes (the job of byte 0 also takes the run that the chunk's part starts inside), so no run is split between two
 * lanes.  Either way a run's source is the unrank of its first item.  With a step in the innermost dimension every run
 * is one item. */
#define BOX_SHORT_RUN 64
template <bool STEPPED>
__global__ void __launch_bounds__(GATHER_WARPS * 32) box_gather_kernel(BoxGatherArgs a) {
  if (a.status && ld_cg_i32(a.status) < 0) return;       /* a stream failed to decode: dest stays untouched */
  const long long ts = a.typesize, runb = a.box.run * ts, g0 = a.p0 * ts, end = g0 + a.total;
  const unsigned bs = (unsigned)a.blocksize;              /* chunk offsets are below 2^31 */
  const int lane = lane_id();
  const long long warps = (long long)gridDim.x * GATHER_WARPS;
  for (long long lo = ((long long)blockIdx.x * GATHER_WARPS + (threadIdx.x >> 5)) * GATHER_SPAN; lo < a.total;
       lo += warps * GATHER_SPAN) {
    const long long hi = lo + GATHER_SPAN < a.total ? lo + GATHER_SPAN : a.total;
    if (runb >= BOX_SHORT_RUN) {
      for (long long o = lo; o < hi;) {
        const long long g = g0 + o, k = b2_box_div(g, runb), u = g - k * runb;
        unsigned s = (unsigned)((b2_box_unrank(&a.box, k * a.box.run, STEPPED) - a.window) * ts + u);
        const long long n = runb - u < hi - o ? runb - u : hi - o;
        slot_copy_warp(a.dst + o, a.src, a.slot, bs, s, n);
        o += n;
      }
    } else {
      const long long ka = b2_box_div(lo == 0 ? g0 : g0 + lo + runb - 1, runb), kb = b2_box_div(g0 + hi + runb - 1, runb);
      for (long long k = ka + lane; k < kb; k += 32) {
        const long long gs = k * runb > g0 ? k * runb : g0, ge = (k + 1) * runb < end ? (k + 1) * runb : end;
        unsigned s = (unsigned)((b2_box_unrank(&a.box, k * a.box.run, STEPPED) - a.window) * ts + (gs - k * runb));
        slot_copy_lane(a.dst + (gs - g0), a.src, a.slot, bs, s, (int)(ge - gs));
      }
    }
  }
}

#ifdef SIMT_EMU
/* The emulator's launchers of the box kernels: a few CTAs each, so that the grid-stride loops run.  The plan's two
 * launches count as plan launches, the gather as a gather launch. */
extern "C" int b2_launch_box_plan(const BoxPlanArgs* a, b2_stream_t) {
  if (a->plan.nblocks <= 0) return 0;
  BoxPlanArgs args = *a;
  const long long nb = a->plan.nblocks;
  simt::launch(simt::Dim3(emu_range_ctas(nb)), simt::Dim3(PLAN_THREADS), 0, [&] {
    if (args.box.stepped) box_touch_kernel<true>(args); else box_touch_kernel<false>(args);
  });
  g_emu_plan_launches++;
  emu_slot_scan(args.plan);
  return 0;
}
extern "C" int b2_launch_box_gather(const BoxGatherArgs* a, b2_stream_t) {
  if (a->total <= 0) return 0;
  g_emu_gather_launches++;
  BoxGatherArgs args = *a;
  simt::launch(simt::Dim3(emu_gather_ctas(a->total)), simt::Dim3(GATHER_WARPS * 32), 0, [&] {
    if (args.box.stepped) box_gather_kernel<true>(args); else box_gather_kernel<false>(args);
  });
  return 0;
}
#endif


/* blosc_b200_getslices: K boxes of one extent, box i the origin box moved by off[i] flat items.  The first flat index
 * >= x (0 <= x <= nitems) of box i, or nitems when there is none: the origin box's answer for x - off[i], moved back. */
DEV long long box_next_at(const B2Box& b, long long off, long long x) {
  const long long n = b2_box_next(&b, x > off ? x - off : 0, 0);
  return n < b.nitems ? n + off : b.nitems;
}

__global__ void __launch_bounds__(PLAN_THREADS) box_check_kernel(BoxCheckArgs a) {
  for (long long i = (long long)blockIdx.x * PLAN_THREADS + threadIdx.x; i < a.nboxes;
       i += (long long)gridDim.x * PLAN_THREADS) {
    const long long* s = a.starts + i * a.ndim;
    long long f0 = 0;
    bool bad = false;
#pragma unroll
    for (int k = 0; k < B2_BOX_MAXDIM; k++)
      if (k < a.ndim) {
        const long long c = s[k];
        if (c < 0 || c > a.hi[k]) bad = true;
        f0 += c * a.stride[k];
      }
    if (bad) { atomicMin(a.bad, (unsigned long long)i); f0 = 0; }
    a.off[i] = f0;
    if (a.touched && !bad) {                     /* the chunks of the box's span that hold one of its items */
      for (long long ch = b2_box_div(f0, a.ipc), last = b2_box_div(f0 + a.span - 1, a.ipc); ch <= last; ch++) {
        const long long w1 = (ch + 1) * a.ipc < a.box.nitems ? (ch + 1) * a.ipc : a.box.nitems;
        if (box_next_at(a.box, f0, ch * a.ipc) < w1) a.touched[ch] = 1;
      }
    }
  }
}

/* boxes_touch_kernel, work item (box i, j): the j-th block of box i's span inside the chunk is touched when an item of
 * the box has a byte in it, the byte test of box_touch_kernel.  Boxes that share a block store the same 1. */
__global__ void __launch_bounds__(PLAN_THREADS) boxes_touch_kernel(BoxesPlanArgs a) {
  const long long ts = a.plan.typesize, bs = a.plan.blocksize, nb = a.plan.nbytes, wend = a.window + b2_box_div(nb, ts);
  for (long long t = (long long)blockIdx.x * PLAN_THREADS + threadIdx.x; t < a.nboxes * a.per_box;
       t += (long long)gridDim.x * PLAN_THREADS) {
    const long long i = b2_box_div(t, a.per_box), j = t - i * a.per_box, f0 = a.off[i];
    if (a.part && j == 0) {                      /* box i's items of flat index in [window, wend), as output bytes */
      const long long y0 = a.window > f0 ? a.window - f0 : 0, y1 = wend > f0 ? wend - f0 : 0;
      a.part[2 * i] = b2_box_rank(&a.box, y0 < a.box.nitems ? y0 : a.box.nitems, 0) * ts;
      a.part[2 * i + 1] = b2_box_rank(&a.box, y1 < a.box.nitems ? y1 : a.box.nitems, 0) * ts;
    }
    const long long x0 = f0 > a.window ? f0 : a.window, x1 = f0 + a.span < wend ? f0 + a.span : wend;
    if (a.in_place || x0 >= x1) continue;
    const long long lo = (b2_box_div((x0 - a.window) * ts, bs) + j) * bs;
    if (lo >= (x1 - a.window) * ts) continue;
    const long long hi = lo + bs < nb ? lo + bs : nb;
    if (box_next_at(a.box, f0, a.window + b2_box_div(lo, ts)) < a.window + b2_box_div(hi + ts - 1, ts))
      a.plan.cover[b2_box_div(lo, bs)] = 1;
  }
}

/* boxes_gather_kernel: box_gather_kernel's walk over the batch's output bytes, one warp job per GATHER_SPAN bytes.  Run
 * q belongs to box i = q / (count / run), and its source is the origin box's unrank of its first item plus off[i].
 * A lane reads box i's offset (and, on a frame, its part of the chunk) again only when its box changes.  The parts
 * come from the plan: ranking them here put two more division calls in the loop, and the kernel spilled. */
__global__ void __launch_bounds__(GATHER_WARPS * 32) boxes_gather_kernel(BoxesGatherArgs a) {
  if (a.status && ld_cg_i32(a.status) < 0) return;       /* a stream failed to decode: dest stays untouched */
  const long long ts = a.typesize, runb = a.box.run * ts, boxb = a.box.count * ts;
  const long long rpb = b2_box_div(a.box.count, a.box.run);      /* runs of a box */
  const unsigned bs = (unsigned)a.blocksize;              /* chunk offsets are below 2^31 */
  const int lane = lane_id();
  const long long warps = (long long)gridDim.x * GATHER_WARPS;
  long long cur = -1, f0 = 0, plo = 0, phi = boxb;       /* box cur's offset and its part [plo, phi) in bytes */
  auto use_box = [&](long long i) {
    if (i == cur) return;
    cur = i;
    f0 = a.off[i];
    if (a.part) { plo = a.part[2 * i]; phi = a.part[2 * i + 1]; }
  };
  for (long long lo = ((long long)blockIdx.x * GATHER_WARPS + (threadIdx.x >> 5)) * GATHER_SPAN; lo < a.total;
       lo += warps * GATHER_SPAN) {
    const long long hi = lo + GATHER_SPAN < a.total ? lo + GATHER_SPAN : a.total;
    if (runb >= BOX_SHORT_RUN) {
      for (long long o = lo; o < hi;) {
        const long long k = b2_box_div(o, runb), u = o - k * runb, i = b2_box_div(k, rpb);
        use_box(i);
        const long long gb = o - i * boxb;                 /* the byte's offset in its box */
        if (gb < plo) { o += plo - gb; continue; }
        if (gb >= phi) { o += boxb - gb; continue; }
        unsigned s = (unsigned)((b2_box_unrank(&a.box, (k - i * rpb) * a.box.run, 0) + f0 - a.window) * ts + u);
        long long n = runb - u < hi - o ? runb - u : hi - o;
        if (n > phi - gb) n = phi - gb;
        slot_copy_warp(a.dst + o, a.src, a.slot, bs, s, n);
        o += n;
      }
    } else {
      const long long ka = b2_box_div(lo + runb - 1, runb), kb = b2_box_div(hi + runb - 1, runb);
      for (long long k = ka + lane; k < kb; k += 32) {
        const long long i = b2_box_div(k, rpb);
        use_box(i);
        long long gs = k * runb, ge = (k + 1) * runb;
        if (gs < i * boxb + plo) gs = i * boxb + plo;
        if (ge > i * boxb + phi) ge = i * boxb + phi;
        if (gs >= ge) continue;
        unsigned s = (unsigned)((b2_box_unrank(&a.box, (k - i * rpb) * a.box.run, 0) + f0 - a.window) * ts + (gs - k * runb));
        slot_copy_lane(a.dst + gs, a.src, a.slot, bs, s, (int)(ge - gs));
      }
    }
  }
}

#ifdef SIMT_EMU
/* The emulator's launchers of the batch kernels, as those of the box kernels: the check and the plan's two launches
 * count as plan launches, the gather as a gather launch. */
extern "C" int b2_launch_box_check(const BoxCheckArgs* a, b2_stream_t) {
  if (a->nboxes <= 0) return 0;
  BoxCheckArgs args = *a;
  simt::launch(simt::Dim3(emu_range_ctas(a->nboxes)), simt::Dim3(PLAN_THREADS), 0, [&] { box_check_kernel(args); });
  g_emu_plan_launches++;
  return 0;
}
extern "C" int b2_launch_boxes_plan(const BoxesPlanArgs* a, b2_stream_t) {
  if (a->plan.nblocks <= 0) return 0;
  BoxesPlanArgs args = *a;
  simt::launch(simt::Dim3(emu_range_ctas(a->nboxes * a->per_box)), simt::Dim3(PLAN_THREADS), 0,
               [&] { boxes_touch_kernel(args); });
  g_emu_plan_launches++;
  emu_slot_scan(args.plan);
  return 0;
}
extern "C" int b2_launch_boxes_gather(const BoxesGatherArgs* a, b2_stream_t) {
  if (a->total <= 0) return 0;
  g_emu_gather_launches++;
  BoxesGatherArgs args = *a;
  simt::launch(simt::Dim3(emu_gather_ctas(a->total)), simt::Dim3(GATHER_WARPS * 32), 0, [&] { boxes_gather_kernel(args); });
  return 0;
}
#endif


/* blosc_b200_getoindex: an orthogonal index selection (B2OSel).  The lists need not be sorted, so there is no closed
 * form for "the next selected item >= x" and the touched blocks are planned forward: oindex_touch_kernel takes the
 * selection's runs, grid-stride, and marks the blocks (or, on a frame, the chunks) each run's source span overlaps, with
 * box_touch_kernel's byte test.  Its first work items check the list entries, so the check costs no launch of its own.
 * The work is proportional to the runs and the list entries, never to the shape. */
__global__ void __launch_bounds__(PLAN_THREADS) oindex_touch_kernel(OIndexPlanArgs a) {
  const long long ts = a.plan.typesize, bs = a.plan.blocksize, nb = a.plan.nbytes;
  const long long ne = a.check ? a.sel.nentries : 0, n = ne + a.r1 - a.r0;
  const long long wend = a.window + (a.touched ? 0 : b2_box_div(nb, ts));
  for (long long t = (long long)blockIdx.x * PLAN_THREADS + threadIdx.x; t < n; t += (long long)gridDim.x * PLAN_THREADS) {
    if (t < ne) {                                /* entry t: list d's position t - lbase[d] */
      int d = 0;
#pragma unroll
      for (int k = 0; k < B2_BOX_MAXDIM; k++)
        if (k < a.sel.ndim && a.sel.list[k] && t >= a.sel.lbase[k]) d = k;
      const long long q = t - a.sel.lbase[d], c = a.sel.list[d][q];
      if (c < 0 || c >= a.sel.shape[d]) atomicMin(a.bad, ((unsigned long long)a.sel.kdim[d] << 56) | (unsigned long long)q);
      continue;
    }
    const long long f = b2_osel_unrank(&a.sel, (a.r0 + t - ne) * a.sel.run);
    if (f < 0) continue;                         /* a bad entry: the check reports it */
    if (a.touched) {
      for (long long c = b2_box_div(f, a.ipc), last = b2_box_div(f + a.sel.run - 1, a.ipc); c <= last; c++)
        a.touched[c] = 1;
      continue;
    }
    const long long x0 = f > a.window ? f : a.window, x1 = f + a.sel.run < wend ? f + a.sel.run : wend;
    if (x0 >= x1) continue;
    for (long long b = b2_box_div((x0 - a.window) * ts, bs), e = (x1 - a.window) * ts; b * bs < e; b++)
      a.plan.cover[b] = 1;
  }
}

/* oindex_gather_kernel: box_gather_kernel's walk over the output bytes [g0, g1), one warp job per GATHER_SPAN bytes,
 * whole-warp copies for runs of BOX_SHORT_RUN bytes or more and one run per lane below that.  A run's source is the
 * unrank of its first item, list dimensions reading their entry; repeated and unsorted entries need nothing more.  On
 * a frame (clip) a run is first tested by its position of dimension 0 alone, one list lookup, and skipped with the
 * rest of that slab when the coordinate's rows miss the chunk; a run that crosses the window's edge is cut at it. */
__global__ void __launch_bounds__(GATHER_WARPS * 32) oindex_gather_kernel(OIndexGatherArgs a) {
  if (a.status && ld_cg_i32(a.status) < 0) return;       /* a stream failed to decode: dest stays untouched */
  const long long ts = a.typesize, run = a.sel.run, runb = run * ts, slabb = a.sel.slab * ts, total = a.g1 - a.g0;
  const unsigned bs = (unsigned)a.blocksize;              /* chunk offsets are below 2^31 */
  const int lane = lane_id();
  const long long warps = (long long)gridDim.x * GATHER_WARPS;
  /* whether slab i (a position of dimension 0) has rows inside the window */
  auto slab_in = [&](long long i) {
    const long long c = a.sel.list[0] ? a.sel.list[0][i] : a.sel.start[0] + i * a.sel.step[0];
    return c * a.sel.stride[0] < a.wend && (c + 1) * a.sel.stride[0] > a.window;
  };
  for (long long lo = ((long long)blockIdx.x * GATHER_WARPS + (threadIdx.x >> 5)) * GATHER_SPAN; lo < total;
       lo += warps * GATHER_SPAN) {
    const long long hi = lo + GATHER_SPAN < total ? lo + GATHER_SPAN : total;
    if (runb >= BOX_SHORT_RUN) {
      for (long long o = lo; o < hi;) {
        const long long g = a.g0 + o, k = b2_box_div(g, runb);
        long long u = g - k * runb, n = runb - u < hi - o ? runb - u : hi - o;
        if (a.clip) {
          const long long i = b2_box_div(g, slabb);
          if (!slab_in(i)) { o = (i + 1) * slabb - a.g0 < hi ? (i + 1) * slabb - a.g0 : hi; continue; }
        }
        const long long f = b2_osel_unrank(&a.sel, k * run);
        if (a.clip) {                            /* the run's bytes [alo, ahi) whose items lie in the window */
          const long long alo = (f < a.window ? a.window - f : 0) * ts;
          const long long ahi = (f + run > a.wend ? a.wend - f : run) * ts;
          if (u < alo) { o += alo - u < n ? alo - u : n; continue; }
          if (u >= ahi) { o += n; continue; }
          if (n > ahi - u) n = ahi - u;
        }
        slot_copy_warp(a.dst + a.g0 + o, a.src, a.slot, bs, (unsigned)((f - a.window) * ts + u), n);
        o += n;
      }
    } else {
      const long long ka = b2_box_div(a.g0 + lo + runb - 1, runb), kb = b2_box_div(a.g0 + hi + runb - 1, runb);
      for (long long k = ka + lane; k < kb; k += 32) {
        if (a.clip && !slab_in(b2_box_div(k * run, a.sel.slab))) continue;
        const long long f = b2_osel_unrank(&a.sel, k * run);
        long long x0 = 0, x1 = run;              /* the run's items inside the window */
        if (a.clip) {
          if (f < a.window) x0 = a.window - f;
          if (f + run > a.wend) x1 = a.wend - f;
        }
        slot_copy_lane(a.dst + (k * run + x0) * ts, a.src, a.slot, bs, (unsigned)((f + x0 - a.window) * ts),
                       (int)((x1 - x0) * ts));
      }
    }
  }
}

#ifdef SIMT_EMU
/* The emulator's launchers of the index-selection kernels, as those of the box kernels: the touch (and, on a chunk
 * that is not read in place, the slot scan) count as plan launches, the gather as a gather launch. */
extern "C" int b2_launch_oindex_plan(const OIndexPlanArgs* a, b2_stream_t) {
  const long long n = (a->check ? a->sel.nentries : 0) + a->r1 - a->r0, nb = a->plan.nblocks;
  OIndexPlanArgs args = *a;
  if (n > 0) {
    simt::launch(simt::Dim3(emu_range_ctas(n)), simt::Dim3(PLAN_THREADS), 0, [&] { oindex_touch_kernel(args); });
    g_emu_plan_launches++;
  }
  if (!a->touched && a->r1 > a->r0 && nb > 0) emu_slot_scan(args.plan);
  return 0;
}
extern "C" int b2_launch_oindex_gather(const OIndexGatherArgs* a, b2_stream_t) {
  const long long total = a->g1 - a->g0;
  if (total <= 0) return 0;
  g_emu_gather_launches++;
  OIndexGatherArgs args = *a;
  simt::launch(simt::Dim3(emu_gather_ctas(total)), simt::Dim3(GATHER_WARPS * 32), 0, [&] { oindex_gather_kernel(args); });
  return 0;
}
#endif


/* blosc_b200_grid_getslice: a touched chunk's part written straight into its place in the output (PlacedGatherArgs).
 * The walk is box_gather_kernel's over the part's bytes [0, total), one warp job per GATHER_SPAN bytes, with the run's
 * source the chunk box's unrank and its destination the output box's.  The part starts at a run edge and holds whole
 * runs, so a lane-per-run job takes exactly the runs that start in its bytes.  STEPPED = the chunk box's `stepped`;
 * the output box has step 1. */
template <bool STEPPED>
__global__ void __launch_bounds__(GATHER_WARPS * 32) placed_gather_kernel(PlacedGatherArgs a) {
  if (a.status && ld_cg_i32(a.status) < 0) return;       /* a stream failed to decode: dest stays untouched */
  const long long ts = a.itemsize, runb = a.run * ts;
  const unsigned bs = (unsigned)a.blocksize;              /* chunk offsets are below 2^31 */
  const int lane = lane_id();
  const long long warps = (long long)gridDim.x * GATHER_WARPS;
  for (long long lo = ((long long)blockIdx.x * GATHER_WARPS + (threadIdx.x >> 5)) * GATHER_SPAN; lo < a.total;
       lo += warps * GATHER_SPAN) {
    const long long hi = lo + GATHER_SPAN < a.total ? lo + GATHER_SPAN : a.total;
    if (runb >= BOX_SHORT_RUN) {
      for (long long o = lo; o < hi;) {
        const long long k = b2_box_div(o, runb), u = o - k * runb;
        u8* out = a.dst + b2_box_unrank(&a.out, k * a.run, 0) * ts + u;
        const unsigned s = (unsigned)(b2_box_unrank(&a.box, k * a.run, STEPPED) * ts + u);
        const long long n = runb - u < hi - o ? runb - u : hi - o;
        slot_copy_warp(out, a.src, a.slot, bs, s, n);
        o += n;
      }
    } else {
      const long long ka = b2_box_div(lo + runb - 1, runb), kb = b2_box_div(hi + runb - 1, runb);
      for (long long k = ka + lane; k < kb; k += 32)
        slot_copy_lane(a.dst + b2_box_unrank(&a.out, k * a.run, 0) * ts, a.src, a.slot, bs,
                       (unsigned)(b2_box_unrank(&a.box, k * a.run, STEPPED) * ts), (int)runb);
    }
  }
}

/* placed_fill_kernel: a missing chunk's part of the output, the output box `out`, filled with the item pattern.  Warp
 * job k covers the part's bytes [k * GATHER_SPAN, (k + 1) * GATHER_SPAN), cut at run edges; the lanes store each
 * piece's consecutive bytes.  A run starts at an item edge, so byte u of a run is byte u % itemsize of the pattern. */
__global__ void __launch_bounds__(GATHER_WARPS * 32) placed_fill_kernel(PlacedGatherArgs a) {
  const long long runb = a.run * a.itemsize;
  const unsigned ts = (unsigned)a.itemsize;               /* a part's bytes are below 2^31 */
  const int lane = lane_id();
  const long long warps = (long long)gridDim.x * GATHER_WARPS;
  for (long long lo = ((long long)blockIdx.x * GATHER_WARPS + (threadIdx.x >> 5)) * GATHER_SPAN; lo < a.total;
       lo += warps * GATHER_SPAN) {
    const long long hi = lo + GATHER_SPAN < a.total ? lo + GATHER_SPAN : a.total;
    for (long long o = lo; o < hi;) {
      const long long k = b2_box_div(o, runb), u = o - k * runb;
      u8* out = a.dst + b2_box_unrank(&a.out, k * a.run, 0) * a.itemsize + u;
      const int n = (int)(runb - u < hi - o ? runb - u : hi - o);
      for (int x = lane; x < n; x += 32) out[x] = a.fill ? a.fill[((unsigned)u + (unsigned)x) % ts] : 0;
      o += n;
    }
  }
}

/* warp_copy_vec that also compares: byte x of the piece is held against byte (u0 + x) % ts of the pattern `fill`
 * (zeros when NULL).  Returns nonzero in a lane that copied a byte other than the pattern's. */
DEV unsigned warp_copy_cmp(u8* __restrict__ dst, const u8* __restrict__ src, int n, const u8* fill, unsigned ts,
                           unsigned u0) {
  const int lane = lane_id();
  unsigned d = 0;
  int i = lane;
  if ((((uintptr_t)dst ^ (uintptr_t)src) & 15u) == 0 && n >= 32) {
    const int head = (int)((16u - ((uintptr_t)dst & 15u)) & 15u);
    const int nv = (n - head) >> 4;
    const uint4* s4 = (const uint4*)(src + head);
    uint4* d4 = (uint4*)(dst + head);
    if (lane < head) { const u8 v = src[lane]; dst[lane] = v; d |= v ^ (fill ? fill[(u0 + lane) % ts] : 0); }
    for (int q = lane; q < nv; q += 32) {
      const uint4 v = s4[q];
      d4[q] = v;
      if (!fill) d |= v.x | v.y | v.z | v.w;
      else {
        const unsigned w[4] = {v.x, v.y, v.z, v.w}, at = u0 + (unsigned)head + 16u * (unsigned)q;
#pragma unroll
        for (int b = 0; b < 16; b++) d |= ((w[b >> 2] >> (8 * (b & 3))) & 0xffu) ^ fill[(at + b) % ts];
      }
    }
    i = head + (nv << 4) + lane;
  }
  for (; i < n; i += 32) { const u8 v = src[i]; dst[i] = v; d |= v ^ (fill ? fill[(u0 + i) % ts] : 0); }
  return d;
}

/* blosc_b200_grid_compress: one chunk's sub-array packed out of the array into the chunk's input (GridPackArgs).  The
 * walk is placed_gather_kernel's over the part's bytes [0, total), with the run's source the array box's unrank and its
 * destination the chunk box's; both boxes have step 1.  Source offsets are 64-bit: the array may exceed 4 GiB.  CMP =
 * a.diff != NULL: each lane compares the bytes it stores with the fill pattern and sets *diff once at the end; without
 * it the kernel only copies. */
template <bool CMP>
__global__ void __launch_bounds__(GATHER_WARPS * 32) grid_pack_kernel(GridPackArgs a) {
  const long long ts = a.itemsize, runb = a.run * ts;
  const unsigned its = (unsigned)a.itemsize;              /* a chunk's bytes are below 2^31 */
  const int lane = lane_id();
  const long long warps = (long long)gridDim.x * GATHER_WARPS;
  unsigned d = 0;
  for (long long lo = ((long long)blockIdx.x * GATHER_WARPS + (threadIdx.x >> 5)) * GATHER_SPAN; lo < a.total;
       lo += warps * GATHER_SPAN) {
    const long long hi = lo + GATHER_SPAN < a.total ? lo + GATHER_SPAN : a.total;
    if (runb >= BOX_SHORT_RUN) {
      for (long long o = lo; o < hi;) {
        const long long k = b2_box_div(o, runb), u = o - k * runb;
        const u8* from = a.src + b2_box_unrank(&a.box, k * a.run, 0) * ts + u;
        u8* out = a.dst + b2_box_unrank(&a.out, k * a.run, 0) * ts + u;
        const int n = (int)(runb - u < hi - o ? runb - u : hi - o);
        if (CMP) d |= warp_copy_cmp(out, from, n, a.fill, its, (unsigned)u);
        else warp_copy_vec(out, from, n);
        o += n;
      }
    } else {
      const long long ka = b2_box_div(lo + runb - 1, runb), kb = b2_box_div(hi + runb - 1, runb);
      for (long long k = ka + lane; k < kb; k += 32) {
        const u8* from = a.src + b2_box_unrank(&a.box, k * a.run, 0) * ts;
        u8* out = a.dst + b2_box_unrank(&a.out, k * a.run, 0) * ts;
        for (int x = 0; x < (int)runb; x++) {
          const u8 v = from[x];
          out[x] = v;
          if (CMP) d |= v ^ (a.fill ? a.fill[(unsigned)x % its] : 0);
        }
      }
    }
  }
  if (CMP && d) *a.diff = 1;
}

#ifdef SIMT_EMU
/* The emulator's launchers of the placed kernels, as those of the box kernels; both count as gather launches */
extern "C" int b2_launch_placed_gather(const PlacedGatherArgs* a, b2_stream_t) {
  if (a->total <= 0) return 0;
  g_emu_gather_launches++;
  PlacedGatherArgs args = *a;
  simt::launch(simt::Dim3(emu_gather_ctas(a->total)), simt::Dim3(GATHER_WARPS * 32), 0, [&] {
    if (args.box.stepped) placed_gather_kernel<true>(args); else placed_gather_kernel<false>(args);
  });
  return 0;
}
extern "C" int b2_launch_placed_fill(const PlacedGatherArgs* a, b2_stream_t) {
  if (a->total <= 0) return 0;
  g_emu_gather_launches++;
  PlacedGatherArgs args = *a;
  simt::launch(simt::Dim3(emu_gather_ctas(a->total)), simt::Dim3(GATHER_WARPS * 32), 0, [&] { placed_fill_kernel(args); });
  return 0;
}
extern "C" int b2_launch_grid_pack(const GridPackArgs* a, b2_stream_t) {
  if (a->total <= 0) return 0;
  g_emu_gather_launches++;
  GridPackArgs args = *a;
  simt::launch(simt::Dim3(emu_gather_ctas(a->total)), simt::Dim3(GATHER_WARPS * 32), 0, [&] {
    if (args.diff) grid_pack_kernel<true>(args); else grid_pack_kernel<false>(args);
  });
  return 0;
}
#endif


/* LZ4 chunks: one CTA of two warps per stream -- a parser that walks the tokens and a copier that owns the output
 * (dev_lz4dpair.cuh).  The parser warp alone draws tickets, checks the size prefixes, counts finished streams and
 * publishes the verdict, exactly as a warp of decode_kernel does. */
#define PAIR_CTAS_PER_SM 12
__global__ void __launch_bounds__(64) decode_pair_kernel(DecodeArgs a) {
#ifdef SIMT_EMU
  u8* smem = simt::g_dynsmem;
#else
  extern __shared__ __align__(16) u8 smem[];
#endif
  Lz4pSlot* slots = (Lz4pSlot*)(smem + LZ4D_RING);
  if ((threadIdx.x >> 5) == 1) { lz4_pair_copier(smem, slots); return; }
  decode_streams(a, [&](const u8* src, int cs, u8* out, int len) { return lz4_pair_parse(src, cs, out, len, slots); });
  lz4_pair_quit(slots);
}

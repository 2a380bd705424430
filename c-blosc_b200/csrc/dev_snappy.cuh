/*
 * dev_snappy.cuh -- Blosc's "snappy" codec, sm_90a: a one-warp decoder and the encoder's stream writer.
 *
 * A snappy stream (snappy's format_description.txt) is the uncompressed length as a varint, then elements, each
 * starting with a tag byte whose low two bits give its kind:
 *   00 literal   lengths 1..60 in the tag (tag >> 2 = length - 1); 61..64 in the tag mean 1..4 little-endian length
 *                bytes follow (length - 1)
 *   01 copy-1    length 4..11 (bits 2-4), offset 0..2047 (bits 5-7 of the tag, then one byte)
 *   10 copy-2    length 1..64 (tag >> 2), 16-bit little-endian offset
 *   11 copy-4    length 1..64 (tag >> 2), 32-bit little-endian offset
 * Copies may overlap their own output (offset < length).
 *
 * Decoder (decode_kernel<B2_CODEC_SNAPPY>, one warp per stream, the LZ4 decoder's LZ4D_SMEM ring of recent output):
 *   dense step   byte-planes of shuffled data encode to long runs of 3-byte copy-2 tags.  Lane l parses the tag at
 *                ip + 3l; the leading lanes that all see a copy-2 are the run, a prefix sum of their lengths places
 *                each copy, and every copy whose source lies before the step's first output byte is made by its own
 *                lane, 4 bytes at a time (sn_copy_dense, lz4d_copy_dense with lengths up to 64 instead of 18).
 *   one element  everything else, one element at a time: literals and copies through lz4d_copy_general.
 * The checks are snappy_uncompress's: the preamble must be a varint of at most 5 bytes that fits in 32 bits and
 * equal the split's length (blosc_d checks the size); offset 0 and offsets past the output produced so far, any tag,
 * length or offset past the input, any element past the output, input left over when the output is full and input
 * that ends early are rejected (-1, which decode_streams reports as it does for a refused LZ4 split).
 *
 * Stream writer (senc_kernel, dev_chunk.cuh; one warp per stream), on the zstd encoder's parse records
 * (dev_zstdenc.cuh zse_parse_lane: offsets <= 65535, so every copy is a copy-1 or a copy-2):
 *   - lane 0 stitches the records of the stream's segments into elements in the stream's part of prev[] (dead once
 *     the parse is done): literals pending across segments go in front of the next match, a match that the next
 *     segment continues with the same offset is merged, and matches are cut into the fewest copies of 1..64 bytes
 *     (every piece of a cut is >= 4 bytes; a 4..11-byte piece with an offset below 2048 is a copy-1).  It sums the
 *     elements' sizes on the way, so the stream's size is known before anything is written;
 *   - if the stream would not be smaller than its split the split is stored raw and nothing is written;
 *   - otherwise the warp writes the preamble and then 32 elements at a time: an exclusive scan of the element sizes
 *     places the tags, one of the decoded lengths places the literals' sources, and the warp copies each literal run.
 * Nothing depends on the order in which warps or lanes run, so the device bytes equal the emulator's.
 */
#pragma once
#include "b2_args.h"
#include "dev_common.cuh"
#include "dev_lz4.cuh"
#include "dev_lz4fast.cuh"
#include "dev_zstdenc.cuh"

/* ---- decoder ---- */
enum {
  SN_H_DENSE = 0,                            /* a dense step of copy-2 tags */
  SN_H_DENSE_RING, SN_H_DENSE_GLOBAL,        /* a dense copy's source */
  SN_H_DENSE_BAD,                            /* a copy that reads the step's own output (or is invalid) ended the run */
  SN_H_DENSE_FEW,                            /* too short a run: one element at a time */
  SN_H_LIT_TAG,                              /* literal, length in the tag */
  SN_H_LIT_1, SN_H_LIT_2, SN_H_LIT_3, SN_H_LIT_4,   /* literal, 1..4 length bytes */
  SN_H_LIT_BUMP,                             /* a literal run longer than the ring moves ring_lo */
  SN_H_COPY1, SN_H_COPY2, SN_H_COPY4,
  SN_H_RING, SN_H_GLOBAL,                    /* a one-element copy's source */
  SN_H_OVERLAP,                              /* a copy that overlaps its own output */
  SN_NHIT
};
#ifdef SIMT_EMU
static int g_sn_fail_line = 0;               /* emulator builds remember the first check that rejected the stream */
#define SN_FAIL (g_sn_fail_line = g_sn_fail_line ? g_sn_fail_line : __LINE__, -1)
static long long g_sn_hit[SN_NHIT];
#define SN_HIT(id) do { if (lane == 0) g_sn_hit[id]++; } while (0)           /* warp-uniform branch */
#define SN_HITL(id, c) do { if (c) g_sn_hit[id]++; } while (0)              /* per lane */
#else
#define SN_FAIL (-1)
#define SN_HIT(id) do {} while (0)
#define SN_HITL(id, c) do {} while (0)
#endif
#define SN_DENSE_OUT (32 * 64)               /* a dense step writes <= 32 copies of <= 64 bytes */
#define SN_DENSE_MIN 4                       /* fewer chained copy-2 tags than this: one element at a time */

/* dense step: lanes [0, cnt) hold one copy each, ml <= 64 bytes to out + dst from off bytes back -- before the step's
 * first output byte.  4 bytes per step, from the ring (two aligned words + funnel shift) or, for far sources, from the
 * output in global memory. */
DEV void sn_copy_dense(u8* out, smem_addr_t ring, int dst, int off, int ml, bool from_ring, int cnt) {
  const int lane = lane_id();
  const int match = dst - off;
  const int mls = lane < cnt ? ml : 0;
  const int mlmax = __ballot_sync(FULLMASK, mls > 32) ? 64 : (__ballot_sync(FULLMASK, mls > 16) ? 32 : 16);
  u8* o = out + dst;
#pragma unroll 1
  for (int k = 0; k < mlmax; k += 4) {
    if (k < mls) {
      u32 v;
      if (from_ring) {
        const u32 m = (u32)(match + k);
        v = __funnelshift_r(smem_ld_u32(ring, m & (LZ4D_RMASK & ~3u)), smem_ld_u32(ring, (m + 4u) & (LZ4D_RMASK & ~3u)), (m & 3u) * 8u);
      } else v = ld_u32(out + match + k);       /* may read a few bytes past the source: they are not used */
      const int nb = mls - k;
      const u32 r = (u32)(dst + k);
      o[k] = (u8)v; smem_st_u8(ring, r & LZ4D_RMASK, v);
      if (nb > 1) { o[k + 1] = (u8)(v >> 8); smem_st_u8(ring, (r + 1u) & LZ4D_RMASK, v >> 8); }
      if (nb > 2) { o[k + 2] = (u8)(v >> 16); smem_st_u8(ring, (r + 2u) & LZ4D_RMASK, v >> 16); }
      if (nb > 3) { o[k + 3] = (u8)(v >> 24); smem_st_u8(ring, (r + 3u) & LZ4D_RMASK, v >> 24); }
    }
  }
}

/* snappy_uncompress for one stream of csize bytes into out[0, cap); `ring_ptr`: LZ4D_SMEM bytes of warp-private
 * shared memory.  Returns cap or -1. */
DEV int snappy_decode_warp(const u8* __restrict__ in, const int csize, u8* out, const int cap, u8* ring_ptr) {
  const int lane = lane_id();
  const smem_addr_t ring = smem_addr(ring_ptr);
  const int iend = csize, oend = cap;
  int ip = 0, op = 0, ring_lo = 0, result = 0;
  /* preamble: varint32 (snappy's Varint::Parse32WithLimit: at most 5 bytes, the fifth < 16) */
  {
    u32 v = 0;
    int k = 0;
    for (;; k++) {
      if (k == 5 || ip >= iend) return SN_FAIL;
      const u32 b = in[ip++];
      if (k == 4 && b >= 16u) return SN_FAIL;
      v |= (b & 127u) << (7 * k);
      if (b < 128u) break;
    }
    if (v != (u32)cap) return SN_FAIL;
  }
  int dense_skip = 0, dense_back = 0;
  while (op < oend) {
    if (ip >= iend) { result = SN_FAIL; break; }                     /* the input ends before the output is full */
    /* ---- dense step: a run of 3-byte copy-2 tags, one per lane ---- */
    if (dense_skip > 0) dense_skip--;
    else if (ip + 96 <= iend && op + SN_DENSE_OUT <= oend) {
      const int q = ip + 3 * lane;
      const u32 tag = in[q];
      const bool is2 = (tag & 3u) == 2u;
      const unsigned okm = __ballot_sync(FULLMASK, is2);
      int cnt = okm == FULLMASK ? 32 : __ffs((int)~okm) - 1;         /* lanes [0, cnt) see copy-2 tags */
      const int ml = lane < cnt ? (int)(tag >> 2) + 1 : 0;
      const int off = lane < cnt ? ((int)in[q + 1] | ((int)in[q + 2] << 8)) : 0;
      int incl = ml;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(FULLMASK, incl, d);
        if (lane >= d) incl += t;
      }
      const int dst = op + incl - ml, match = dst - off;
      /* the first copy that reads the step's own output (or is invalid: offset 0, before the stream) ends the run;
       * 8 bytes of slack because the word-wise copy reads up to 7 bytes past the end of its source */
      const unsigned bad = __ballot_sync(FULLMASK, lane < cnt && (off < incl + 8 || match < 0));
      if (bad) { cnt = __ffs((int)bad) - 1; SN_HIT(SN_H_DENSE_BAD); }
      if (cnt >= SN_DENSE_MIN) {
        const int total = __shfl_sync(FULLMASK, incl, cnt - 1);
        const bool from_ring = off <= LZ4D_RING - SN_DENSE_OUT - 64 && match >= ring_lo;
        SN_HIT(SN_H_DENSE);
        SN_HITL(from_ring ? SN_H_DENSE_RING : SN_H_DENSE_GLOBAL, lane < cnt);
        sn_copy_dense(out, ring, dst, off, ml, from_ring, cnt);
        __syncwarp();
        ip += 3 * cnt; op += total;
        dense_back = 0;
        continue;
      }
      SN_HIT(SN_H_DENSE_FEW);
      dense_back = dense_back < 8 ? dense_back + 1 : 8;              /* not that kind of data right here: back off */
      dense_skip = dense_back;
    }
    /* ---- one element ---- */
    const u32 tag = in[ip++];
    if ((tag & 3u) == 0u) {                                          /* literal */
      long long len = (long long)(tag >> 2) + 1;
      if (len > 60) {
        const int nb = (int)len - 60;
        if (ip + nb > iend) { result = SN_FAIL; break; }
        u32 v = 0;
        for (int k = 0; k < nb; k++) v |= (u32)in[ip + k] << (8 * k);
        ip += nb;
        len = (long long)v + 1;
        SN_HIT(SN_H_LIT_1 + nb - 1);
      } else SN_HIT(SN_H_LIT_TAG);
      if (len > iend - ip) { result = SN_FAIL; break; }            /* runs past the input */
      if (len > oend - op) { result = SN_FAIL; break; }            /* runs past the output */
      const int l = (int)len;
      lz4d_copy_general(in, out, ring, ip, op, l, 0, 0, LZ4D_ZERO);
      __syncwarp();
      if (l > LZ4D_RING - 64) { ring_lo = op + l - (LZ4D_RING - 64) > ring_lo ? op + l - (LZ4D_RING - 64) : ring_lo; SN_HIT(SN_H_LIT_BUMP); }
      ip += l; op += l;
      continue;
    }
    int len;
    long long off;
    if ((tag & 3u) == 1u) {                                          /* copy-1 */
      if (ip + 1 > iend) { result = SN_FAIL; break; }
      len = 4 + (int)((tag >> 2) & 7u);
      off = (long long)(((tag >> 5) << 8) | in[ip]);
      ip += 1;
      SN_HIT(SN_H_COPY1);
    } else if ((tag & 3u) == 2u) {                                   /* copy-2 */
      if (ip + 2 > iend) { result = SN_FAIL; break; }
      len = 1 + (int)(tag >> 2);
      off = (long long)((u32)in[ip] | ((u32)in[ip + 1] << 8));
      ip += 2;
      SN_HIT(SN_H_COPY2);
    } else {                                                         /* copy-4 */
      if (ip + 4 > iend) { result = SN_FAIL; break; }
      len = 1 + (int)(tag >> 2);
      off = (long long)((u32)in[ip] | ((u32)in[ip + 1] << 8) | ((u32)in[ip + 2] << 16) | ((u32)in[ip + 3] << 24));
      ip += 4;
      SN_HIT(SN_H_COPY4);
    }
    if (off == 0 || off > op) { result = SN_FAIL; break; }          /* offset 0, or before the stream */
    if (len > oend - op) { result = SN_FAIL; break; }               /* runs past the output */
    const int o = (int)off;
    const int how = o <= LZ4D_RING - 64 && op - o >= ring_lo ? LZ4D_FROM_RING : LZ4D_FROM_GLOBAL;
    SN_HIT(how == LZ4D_FROM_RING ? SN_H_RING : SN_H_GLOBAL);
    if (o < len) SN_HIT(SN_H_OVERLAP);
    lz4d_copy_general(in, out, ring, 0, op, 0, len, o, how);
    __syncwarp();
    op += len;
  }
  if (result == 0 && ip != iend) result = SN_FAIL;                   /* input left over once the output is full */
  __syncwarp();
  return result < 0 ? result : op;
}

/* ---- stream writer ---- */
#define SN_LIT 0x80000000u                   /* element: SN_LIT | length (literal), or length << 16 | offset (copy) */

DEV int sn_varint_len(u32 v) { return v < (1u << 7) ? 1 : (v < (1u << 14) ? 2 : (v < (1u << 21) ? 3 : (v < (1u << 28) ? 4 : 5))); }
/* bytes of an element: tag (+ length bytes) + literals, or the copy's 2 / 3 bytes */
DEV int sn_elem_size(u32 e) {
  if (e & SN_LIT) {
    const u32 l = e & ~SN_LIT;
    return (int)l + (l <= 60u ? 1 : (l <= 256u ? 2 : (l <= 65536u ? 3 : (l <= (1u << 24) ? 4 : 5))));
  }
  const u32 l = e >> 16, o = e & 0xffffu;
  return (l >= 4u && l <= 11u && o < 2048u) ? 2 : 3;
}

/* a match of l bytes at offset d as the fewest copies of <= 64 bytes, none shorter than 4 (as snappy cuts them) */
DEV void sn_put_match(u32* item, int& ni, long long& size, int l, int d) {
  while (l > 64) {
    const int take = l - 64 >= 4 ? 64 : l - 4;
    item[ni] = (u32)take << 16 | (u32)d; size += sn_elem_size(item[ni]); ni++;
    l -= take;
  }
  item[ni] = (u32)l << 16 | (u32)d; size += sn_elem_size(item[ni]); ni++;
}
DEV void sn_put_lits(u32* item, int& ni, long long& size, int l) {
  if (l <= 0) return;
  item[ni] = SN_LIT | (u32)l; size += sn_elem_size(item[ni]); ni++;
}

/* Lane 0: the elements of the stream s[0, n) from the records of its segments; returns their count, *size the
 * stream's size with the preamble */
DEV int sn_stitch(const u32* __restrict__ rec, const u32* __restrict__ cnt, const int n, u32* item, long long* size) {
  const int nseg = (n + FAST_SEG - 1) / FAST_SEG;
  int from = 0, pl = 0, pd = 0, pend = -1, ni = 0;            /* literals start at `from`; the pending match */
  long long sz = sn_varint_len((u32)n);
  for (int k = 0; k < nseg; k++) {
    const int c = (int)cnt[k], ss = k * FAST_SEG;
    int p = ss;
    for (int r = 0; r < c; r++) {
      const u32 x = rec[(long long)k * ZE_SEG_RECS + r];
      const int ll = (int)(x & 0xffu), ml = (int)((x >> 8) & 0xffu) + 4, off = (int)(x >> 16);
      if (r == 0 && ll == 0 && pl > 0 && pend == ss && pd == off) {    /* the match goes on */
        pl += ml; pend = ss + ml; p = pend; from = pend;
        continue;
      }
      const int ms = p + ll;
      if (pl > 0) sn_put_match(item, ni, sz, pl, pd);
      sn_put_lits(item, ni, sz, ms - from);
      pl = ml; pd = off; pend = ms + ml; p = pend; from = pend;
    }
  }
  if (pl > 0) sn_put_match(item, ni, sz, pl, pd);
  sn_put_lits(item, ni, sz, n - from);
  *size = sz;
  return ni;
}

/* The whole warp: the snappy stream of s[0, n) into out[0, n) (records rec / cnt per segment, scratch = the stream's 2n
 * bytes of prev[]).  Returns its size, or n (nothing written) when it would not be smaller than the input. */
DEV int sn_stream(const u8* __restrict__ s, const int n, const u32* __restrict__ rec, const u32* __restrict__ cnt,
                  u8* scratch, u8* out) {
  const int lane = lane_id();
  if (n < 16) return n;
  /* the elements, on the first 4-byte boundary of the scratch (a stream's part of prev[] starts on an odd u16 when
   * the split length is odd).  Each element covers >= 1 byte and no two literal runs are adjacent: 4 x elements + 3
   * <= 1.6 n + 7 <= 2 n bytes for n >= 16 */
  u32* item = (u32*)(((uintptr_t)scratch + 3u) & ~(uintptr_t)3u);
  int ni = 0;
  long long size = 0;
  if (lane == 0) ni = sn_stitch(rec, cnt, n, item, &size);
  ni = __shfl_sync(FULLMASK, ni, 0);
  size = __shfl_sync(FULLMASK, size, 0);
  if (size >= n) return n;                                        /* would not be smaller: stored raw */
  __syncwarp();
  const int pre = sn_varint_len((u32)n);
  if (lane < pre) out[lane] = (u8)(((u32)n >> (7 * lane)) & 127u) | (lane < pre - 1 ? 128u : 0u);
  int ob = pre, ib = 0;
  for (int t0 = 0; t0 < ni; t0 += 32) {
    const int i = t0 + lane;
    const u32 e = i < ni ? item[i] : 0u;
    const bool lit = i < ni && (e & SN_LIT);
    const int es = i < ni ? sn_elem_size(e) : 0;
    const int dl = i < ni ? (lit ? (int)(e & ~SN_LIT) : (int)(e >> 16)) : 0;
    int eo = es, di = dl;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(FULLMASK, eo, d), u = __shfl_up_sync(FULLMASK, di, d);
      if (lane >= d) { eo += t; di += u; }
    }
    const int etot = __shfl_sync(FULLMASK, eo, 31), dtot = __shfl_sync(FULLMASK, di, 31);
    const int p = ob + eo - es, src = ib + di - dl;
    int th = 0;                                                    /* tag and length bytes */
    if (lit) {
      const u32 l1 = (e & ~SN_LIT) - 1u;
      if (l1 < 60u) { out[p] = (u8)(l1 << 2); th = 1; }
      else {
        const int nb = l1 < 256u ? 1 : (l1 < 65536u ? 2 : (l1 < (1u << 24) ? 3 : 4));
        out[p] = (u8)((59 + nb) << 2);
        for (int k = 0; k < nb; k++) out[p + 1 + k] = (u8)(l1 >> (8 * k));
        th = 1 + nb;
      }
    } else if (i < ni) {
      const u32 l = e >> 16, o = e & 0xffffu;
      if (es == 2) { out[p] = (u8)(1u | ((l - 4u) << 2) | ((o >> 8) << 5)); out[p + 1] = (u8)o; }
      else { out[p] = (u8)(2u | ((l - 1u) << 2)); out[p + 1] = (u8)o; out[p + 2] = (u8)(o >> 8); }
    }
    /* the literal runs, each by the whole warp */
    for (unsigned lm = __ballot_sync(FULLMASK, lit); lm; lm &= lm - 1u) {
      const int t = __ffs((int)lm) - 1;
      const int tp = __shfl_sync(FULLMASK, p + th, t), ts = __shfl_sync(FULLMASK, src, t), tl = __shfl_sync(FULLMASK, dl, t);
      for (int k = lane; k < tl; k += 32) out[tp + k] = s[ts + k];
    }
    ob += etot; ib += dtot;
  }
  __syncwarp();
  return ob;
}

/*
 * dev_lz4dpair.cuh -- LZ4 block decoder as a PAIR of warps per stream, sm_90a.
 *
 * lz4_decode_warp (dev_lz4.cuh) is one warp per stream and, on the hard byte-plane of shuffled data, a chain of
 * ~150 k dependent instructions: every step parses up to 32 sequences and then copies them, and a lone warp issues
 * one instruction every ~6 cycles.  Parsing step k+1 needs nothing from the copies of step k -- only the byte counts,
 * which the parse itself produces -- so the two halves run in two warps:
 *
 *   parser  walks the tokens exactly as lz4_decode_warp does (same four tiers, same LZ4_decompress_safe checks,
 *           lz4.c:2022-2445), keeps ip / op / ring_lo, and instead of copying writes a descriptor of the step
 *           (destination, source and length of every sequence) into a queue of LZ4P_Q slots in shared memory;
 *   copier  owns the output and the 16 KiB ring that mirrors it, takes the descriptors in order and performs the
 *           copies with the very same code the single-warp decoder uses.
 *
 * Hand-over with named barriers (bar.sync / bar.arrive, 64 threads): FULL(s) parser -> copier, EMPTY(s) back.
 * The decoded bytes and every verdict on damaged input are identical to lz4_decode_warp's (tests run both).
 */
#pragma once
#include "dev_lz4.cuh"

#define LZ4P_Q 4                               /* descriptor slots */
#define LZ4P_BAR_FULL(s) (1 + (s))
#define LZ4P_BAR_EMPTY(s) (1 + LZ4P_Q + (s))
enum { LZ4P_END = 0, LZ4P_DENSE = 1, LZ4P_LONE = 2, LZ4P_BATCH = 3, LZ4P_SINGLE = 4, LZ4P_GENERAL = 5, LZ4P_START = 6, LZ4P_QUIT = 7 };

struct Lz4pSlot {
  u32 type;
  u32 p[7];                                    /* scalars of the step */
  u32 w[64];                                   /* DENSE: two words per lane; BATCH: 22 table words + 10 start-bit words */
};
#define LZ4P_SMEM (LZ4D_RING + LZ4P_Q * (int)sizeof(Lz4pSlot))

/* ---- parser side: slot management ---- */
DEV Lz4pSlot* lz4p_acquire(Lz4pSlot* slots, int k) {
  const int s = k & (LZ4P_Q - 1);
  if (k >= LZ4P_Q) bar_sync(LZ4P_BAR_EMPTY(s), 64);        /* the copier is done with descriptor k - Q */
  return &slots[s];
}
DEV void lz4p_publish(int& k) {
  __syncwarp();
  __threadfence_block();
  bar_arrive(LZ4P_BAR_FULL(k & (LZ4P_Q - 1)), 64);
  k++;
}
/* the EMPTY arrivals of the last descriptors have no acquire that consumes them: take them, so that both warps start
 * the next stream with every barrier idle */
DEV void lz4p_drain(int k) {
  for (int j = k > LZ4P_Q ? k - LZ4P_Q : 0; j < k; j++) bar_sync(LZ4P_BAR_EMPTY(j & (LZ4P_Q - 1)), 64);
}

/* ---- copier ---- */
DEV void lz4_pair_copier(u8* ring_ptr, Lz4pSlot* slots) {
  const int lane = lane_id();
  const smem_addr_t ring = smem_addr(ring_ptr);
  const u8* in = nullptr;
  u8* out = nullptr;
  int k = 0;
  for (;;) {
    const int s = k & (LZ4P_Q - 1);
    bar_sync(LZ4P_BAR_FULL(s), 64);
    const Lz4pSlot* q = &slots[s];
    const u32 type = *(const volatile u32*)&q->type;
    if (type == LZ4P_QUIT) return;
    const u32 p0 = *(const volatile u32*)&q->p[0], p1 = *(const volatile u32*)&q->p[1], p2 = *(const volatile u32*)&q->p[2],
              p3 = *(const volatile u32*)&q->p[3], p4 = *(const volatile u32*)&q->p[4], p5 = *(const volatile u32*)&q->p[5];
    if (type == LZ4P_START) {
      in = (const u8*)(((u64)p1 << 32) | p0);
      out = (u8*)(((u64)p3 << 32) | p2);
    } else if (type == LZ4P_DENSE) {
      /* p0 = cnt, p1 = mask of the long matches; lane: w[2l] = dst, w[2l+1] = off | ml << 16 | kind << 28 | from_ring << 31 */
      const int cnt = (int)p0;
      const unsigned longm = p1;
      const u32 wd = *(const volatile u32*)&q->w[2 * lane], wx = *(const volatile u32*)&q->w[2 * lane + 1];
      const int dst = (int)wd, off = (int)(wx & 0xffffu), ml = (int)((wx >> 16) & 0xfffu), kind = (int)((wx >> 28) & 3u);
      const bool from_ring = (wx >> 31) != 0u;
      const int match = dst - off;
      {
        const int mls = (lane < cnt && kind == 1) ? ml : 0;
        const int mlmax = __ballot_sync(FULLMASK, mls > 16) ? 18 : (__ballot_sync(FULLMASK, mls > 8) ? 16 : 8);
        u8* o = out + dst;
#pragma unroll 1
        for (int kk = 0; kk < mlmax; kk += 4) {
          if (kk < mls) {
            u32 v;
            if (from_ring) {
              const u32 m = (u32)(match + kk);
              v = __funnelshift_r(smem_ld_u32(ring, m & (LZ4D_RMASK & ~3u)), smem_ld_u32(ring, (m + 4u) & (LZ4D_RMASK & ~3u)), (m & 3u) * 8u);
            } else v = ld_u32(out + match + kk);
            const int nb = mls - kk;
            const u32 r = (u32)(dst + kk);
            o[kk] = (u8)v; smem_st_u8(ring, r & LZ4D_RMASK, v);
            if (nb > 1) { o[kk + 1] = (u8)(v >> 8); smem_st_u8(ring, (r + 1u) & LZ4D_RMASK, v >> 8); }
            if (nb > 2) { o[kk + 2] = (u8)(v >> 16); smem_st_u8(ring, (r + 2u) & LZ4D_RMASK, v >> 16); }
            if (nb > 3) { o[kk + 3] = (u8)(v >> 24); smem_st_u8(ring, (r + 3u) & LZ4D_RMASK, v >> 24); }
          }
        }
      }
      for (unsigned tm = longm; tm; tm &= tm - 1u) {
        const int t = __ffs((int)tm) - 1;
        const int td = __shfl_sync(FULLMASK, dst, t), tmt = __shfl_sync(FULLMASK, match, t), tl = __shfl_sync(FULLMASK, ml, t);
        const bool tring = __shfl_sync(FULLMASK, (int)from_ring, t) != 0;
        for (int kk = lane; kk < tl; kk += 32) {
          const u32 v = tring ? smem_ld_u8(ring, (u32)(tmt + kk) & LZ4D_RMASK) : (u32)out[tmt + kk];
          out[td + kk] = (u8)v;
          smem_st_u8(ring, (u32)(td + kk) & LZ4D_RMASK, v);
        }
      }
    } else if (type == LZ4P_LONE) {
      /* one long match whose source overlaps its own output: p0 = op, p1 = length, p2 = offset, p3 = from ring */
      const int op = (int)p0, tlen = (int)p1, toff = (int)p2, tmatch = op - toff;
      const bool tring = p3 != 0u;
      for (int kk = lane; kk < tlen; kk += 32) {
        const int src = tmatch + (toff >= tlen ? kk : kk % toff);
        const u32 v = tring ? smem_ld_u8(ring, (u32)src & LZ4D_RMASK) : (u32)out[src];
        out[op + kk] = (u8)v;
        smem_st_u8(ring, (u32)(op + kk) & LZ4D_RMASK, v);
      }
    } else if (type == LZ4P_BATCH) {
      /* p0 = ip, p1 = op, p2 = total, p3 = ring_lo; w[0..21] = {info, off} of up to 11 sequences, w[22..31] start bits */
      const int ip = (int)p0, op = (int)p1, total = (int)p2, ring_lo = (int)p3;
      const volatile u32* tbl = q->w;
      const volatile u32* smask = q->w + 22;
      int kbase = 0;
      for (int r = 0; r * 32 < total; r++) {
        const u32 wv = smask[r];
        const int y = r * 32 + lane;
        if (y < total) {
          const int kq = kbase + __popc(wv & ((2u << lane) - 1u)) - 1;
          const u32 e0 = tbl[2 * kq], offk = tbl[2 * kq + 1];
          const int opre = (int)(e0 & 511u), litk = (int)((e0 >> 9) & 15u), lanek = (int)(e0 >> 13);
          const int j = y - opre;
          u32 v;
          if (j < litk) v = in[ip + lanek + 1 + j];
          else {
            const int src = op + opre + litk - (int)offk + (j - litk);
            const int m0 = op + opre + litk - (int)offk;
            if ((int)offk <= LZ4D_RING - LZ4D_BATCH_OUT - 64 && m0 >= ring_lo) v = smem_ld_u8(ring, (u32)src & LZ4D_RMASK);
            else v = out[src];
          }
          out[op + y] = (u8)v;
          smem_st_u8(ring, (u32)(op + y) & LZ4D_RMASK, v);
        }
        kbase += __popc(wv);
      }
    } else if (type == LZ4P_SINGLE) {
      /* p0 = ip, p1 = op, p2 = lit, p3 = total, p4 = offset, p5 = use ring */
      const int ip = (int)p0, op = (int)p1, lit = (int)p2, total = (int)p3, match = op + lit - (int)p4;
      if (lane < total) {
        u32 v;
        if (lane < lit) v = in[ip + 1 + lane];
        else if (p5) v = smem_ld_u8(ring, (u32)(match + lane - lit) & LZ4D_RMASK);
        else v = out[match + lane - lit];
        out[op + lane] = (u8)v;
        smem_st_u8(ring, (u32)(op + lane) & LZ4D_RMASK, v);
      }
    } else if (type == LZ4P_GENERAL) {
      /* p0 = literal source, p1 = op, p2 = literal count, p3 = match length (0: literals only), p4 = offset,
       * p5 = how to copy the match: 0 zero fill (offset 0), 1 ring-mirrored from the ring, 2 ring-mirrored from global, 3 long */
      const int lsrc = (int)p0, len = (int)p2, mlen = (int)p3, off = (int)p4;
      int op = (int)p1;
      for (int kk = lane; kk < len; kk += 32) {
        const u32 v = in[lsrc + kk];
        out[op + kk] = (u8)v;
        smem_st_u8(ring, (u32)(op + kk) & LZ4D_RMASK, v);
      }
      if (mlen > 0) {
        op += len;
        const int match = op - off;
        __syncwarp();
        if (p5 == 0u) {
          for (int kk = lane; kk < mlen; kk += 32) out[op + kk] = 0;
        } else if (p5 <= 2u) {
          const bool from_ring = p5 == 1u;
          for (int k0 = 0; k0 < mlen; k0 += 32) {
            const int kk = k0 + lane;
            if (kk < mlen) {
              const int src = match + (off >= mlen ? kk : kk % off);
              const u32 v = from_ring ? smem_ld_u8(ring, (u32)src & LZ4D_RMASK) : (u32)out[src];
              out[op + kk] = (u8)v;
              smem_st_u8(ring, (u32)(op + kk) & LZ4D_RMASK, v);
            }
          }
        } else warp_copy_match(out, op, match, mlen);
      }
    }
    __syncwarp();
    bar_arrive(LZ4P_BAR_EMPTY(s), 64);
    k = type == LZ4P_END ? 0 : k + 1;
  }
}

/* ---- parser: LZ4_decompress_safe for one stream, copies delegated.  Returns the number of bytes the stream decodes to
 * or -1; the copier has finished with the stream when this returns. ---- */
DEV int lz4_pair_parse(const u8* __restrict__ in, const int csize, u8* out, const int cap, Lz4pSlot* slots) {
  const int iend = csize, oend = cap;
  const int lane = lane_id();
  const StreamBase ib = make_stream_base(in);
  int ip = 0, op = 0, k = 0, result = 0;
  int ring_lo = 0;
  if (cap == 0) return (csize == 1 && in[0] == 0) ? 0 : LZ4D_FAIL;   /* lz4.c:2062-2066 */
  if (csize == 0) return LZ4D_FAIL;
  {
    Lz4pSlot* q = lz4p_acquire(slots, k);
    if (lane == 0) {
      q->type = LZ4P_START;
      q->p[0] = (u32)(u64)(uintptr_t)in; q->p[1] = (u32)((u64)(uintptr_t)in >> 32);
      q->p[2] = (u32)(u64)(uintptr_t)out; q->p[3] = (u32)((u64)(uintptr_t)out >> 32);
    }
    lz4p_publish(k);
  }
  int dense_skip = 0, dense_back = 0;
  for (;;) {
    /* ---- dense path (see lz4_decode_warp) ---- */
    if (dense_skip > 0) dense_skip--;
    else if (ip + 112 <= iend && op + LZ4D_DENSE_OUT <= oend - LZ4_MFLIMIT) {
      u32 b0, b1, b2;
      ldp_win12(ib, ip + 3 * lane, b0, b1, b2);
      lz4d_prefetch(in, ip + 256 + 128 * lane, lane < 2 ? iend : 0);
      int kind = 0, ml = 0, off = 0, c = 0, sft = 0;
      u32 w = b0;
      for (;;) {
        const u32 tok = w & 0xffu;
        const unsigned okm = __ballot_sync(FULLMASK, lane >= c && (tok >> 4) == 0u && (tok & 15u) != 15u);
        const unsigned stop = ~okm & ~((1u << c) - 1u);
        const int e = stop ? __ffs((int)stop) - 1 : 32;
        if (lane >= c && lane < e) { kind = 1; ml = (int)(tok & 15u) + 4; off = (int)((w >> 8) & 0xffffu); }
        c = e;
        if (e >= 32 || sft == LZ4D_DENSE_LONG) break;
        const u32 tw = __shfl_sync(FULLMASK, w, e);
        if ((tw & 0xffu) != 0x0fu || (tw >> 24) == 255u) break;
        if (lane == e) { kind = 2; ml = 19 + (int)(tw >> 24); off = (int)((tw >> 8) & 0xffffu); }
        c = e + 1; sft++;
        if (c >= 32) break;
        w = sft < 4 ? __funnelshift_r(b0, b1, 8u * (u32)sft) : (sft == 4 ? b1 : (sft < 8 ? __funnelshift_r(b1, b2, 8u * (u32)(sft - 4)) : b2));
      }
      int cnt = c;
      int incl = ml;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(FULLMASK, incl, d);
        if (lane >= d) incl += t;
      }
      const int dst = op + incl - ml, match = dst - off;
      const unsigned bad = __ballot_sync(FULLMASK, lane < cnt && (off < incl + 8 || match < 0));
      if (bad) cnt = __ffs((int)bad) - 1;
      if (bad) LZ4D_HIT(cnt == 0 ? LZ4D_H_DENSE_BAD0 : LZ4D_H_DENSE_BAD);
      const unsigned longm = __ballot_sync(FULLMASK, lane < cnt && kind == 2);
      if (cnt >= LZ4D_DENSE_MIN || longm) {
        const int total = __shfl_sync(FULLMASK, incl, cnt - 1);
        const bool from_ring = off <= LZ4D_RING - LZ4D_DENSE_OUT - 64 && match >= ring_lo;
        LZ4D_HIT(LZ4D_H_DENSE_SHIFT + sft);
        if (sft == LZ4D_DENSE_LONG && c < 32) LZ4D_HIT(LZ4D_H_DENSE_LONGCAP);
        LZ4D_HITL(from_ring ? LZ4D_H_DENSE_RING : LZ4D_H_DENSE_GLOBAL, lane < cnt);
        Lz4pSlot* q = lz4p_acquire(slots, k);
        q->w[2 * lane] = (u32)dst;
        q->w[2 * lane + 1] = (u32)off | ((u32)ml << 16) | ((u32)kind << 28) | (from_ring ? 0x80000000u : 0u);
        if (lane == 0) { q->type = LZ4P_DENSE; q->p[0] = (u32)cnt; q->p[1] = longm; }
        lz4p_publish(k);
        ip += 3 * cnt + __popc(longm); op += total;
        LZ4D_DBGN(g_dbg_lz4d_dense_seqs, cnt);
        dense_back = 0;
        continue;
      }
      {
        const u32 tw = __shfl_sync(FULLMASK, b0, 0);
        const int tlen = 19 + (int)(tw >> 24), toff = (int)((tw >> 8) & 0xffffu), tmatch = op - toff;
        if ((tw & 0xffu) == 0x0fu && (tw >> 24) != 255u && toff != 0 && tmatch >= 0 && op + tlen <= oend - LZ4_MFLIMIT) {
          const bool tring = toff <= LZ4D_RING - 512 && tmatch >= ring_lo;
          LZ4D_HIT(tring ? LZ4D_H_LONE_RING : LZ4D_H_LONE_GLOBAL);
          if (toff < tlen) LZ4D_HIT(LZ4D_H_LONE_PERIOD);
          Lz4pSlot* q = lz4p_acquire(slots, k);
          if (lane == 0) { q->type = LZ4P_LONE; q->p[0] = (u32)op; q->p[1] = (u32)tlen; q->p[2] = (u32)toff; q->p[3] = tring ? 1u : 0u; }
          lz4p_publish(k);
          ip += 4; op += tlen;
          LZ4D_DBG(g_dbg_lz4d_dense_seqs);
          dense_back = 0;
          continue;
        }
      }
      if (cnt > 0) LZ4D_HIT(LZ4D_H_DENSE_FEW);
      dense_back = dense_back < 8 ? dense_back + 1 : 8;
      dense_skip = dense_back;
    }
    /* ---- batch path ---- */
    if (ip + 49 <= iend && op + LZ4D_BATCH_OUT <= oend - LZ4_MFLIMIT) {
      u32 b0, b1, b2;
      ldp_win12(ib, ip + lane, b0, b1, b2);
      const u32 token = b0 & 0xffu;
      const int lit = (int)(token >> 4), mln = (int)(token & 15u);
      const int ob = 1 + lit;
      const u32 ow = ob < 4 ? __funnelshift_r(b0, b1, 8u * ob) : (ob < 8 ? __funnelshift_r(b1, b2, 8u * (ob - 4)) : b2 >> (8u * ((ob - 8) & 3)));
      const int off = (int)(ow & 0xffffu);
      const int L = 3 + lit, O = lit + mln + 4;
      const bool good = lit <= 9 && mln != 15 && off >= LZ4D_BATCH_OUT;
      int nseq = 0, consumed = 0, total = 0, my_rank = -1, my_opre = 0;
      const unsigned g3 = __ballot_sync(FULLMASK, good && lit == 0);
      if ((g3 & 0x49249249u) == 0x49249249u) {
        const bool real = (lane % 3) == 0;
        const int v = real ? O : 0;
        int incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int t = __shfl_up_sync(FULLMASK, incl, d);
          if (lane >= d) incl += t;
        }
        if (real) { my_rank = lane / 3; my_opre = incl - v; }
        nseq = 11; consumed = 33;
        total = __shfl_sync(FULLMASK, incl, 31);
      } else {
        const u32 packed = (good ? 1u : 0u) | ((u32)L << 1) | ((u32)O << 5);
        int cur = 0;
        while (cur < 32) {
          const u32 pk = __shfl_sync(FULLMASK, packed, cur);
          if (!(pk & 1u)) break;
          if (lane == cur) { my_rank = nseq; my_opre = total; }
          total += (int)((pk >> 5) & 31u);
          cur += (int)((pk >> 1) & 15u);
          nseq++;
        }
        consumed = cur;
      }
      if (nseq > 0) {
        const int match = op + my_opre + lit - off;
        if (__ballot_sync(FULLMASK, my_rank >= 0 && match < 0)) { result = LZ4D_FAIL; break; }   /* lz4.c:2356 */
        LZ4D_HIT((g3 & 0x49249249u) == 0x49249249u ? LZ4D_H_BATCH_FAST : LZ4D_H_BATCH_WALK);
        LZ4D_HITL(off <= LZ4D_RING - LZ4D_BATCH_OUT - 64 && match >= ring_lo ? LZ4D_H_BATCH_RING : LZ4D_H_BATCH_GLOBAL, my_rank >= 0);
        Lz4pSlot* q = lz4p_acquire(slots, k);
        if (lane < 10) q->w[22 + lane] = 0;
        __syncwarp();
        if (my_rank >= 0) {
          q->w[2 * my_rank] = (u32)my_opre | ((u32)lit << 9) | ((u32)lane << 13);
          q->w[2 * my_rank + 1] = (u32)off;
          atomicOr(&q->w[22 + (my_opre >> 5)], 1u << (my_opre & 31));
        }
        if (lane == 0) { q->type = LZ4P_BATCH; q->p[0] = (u32)ip; q->p[1] = (u32)op; q->p[2] = (u32)total; q->p[3] = (u32)ring_lo; }
        lz4p_publish(k);
        ip += consumed; op += total;
        LZ4D_DBGN(g_dbg_lz4d_batch_seqs, nseq);
        continue;
      }
    }
    /* ---- single-sequence fast path ---- */
    if (ip + 20 <= iend) {
      u32 b0, b1, b2;
      ldp_win12(ib, ip, b0, b1, b2);
      const u32 token = b0 & 0xffu;
      const int lit = (int)(token >> 4), mln = (int)(token & 15u);
      if (lit <= 9 && mln != 15) {
        const int ml = mln + 4, total = lit + ml;
        const int ob = 1 + lit;
        const u32 ow = ob < 4 ? __funnelshift_r(b0, b1, 8u * ob) : (ob < 8 ? __funnelshift_r(b1, b2, 8u * (ob - 4)) : b2 >> (8u * (ob - 8)));
        const int off = (int)(ow & 0xffffu);
        const int match = op + lit - off;
        if (off >= total && op + total <= oend - LZ4_MFLIMIT) {
          if (match < 0) { result = LZ4D_FAIL; break; }       /* lz4.c:2356 */
          const bool use_ring = off <= LZ4D_RING - 64 && match >= ring_lo;
          LZ4D_HIT(use_ring ? LZ4D_H_SINGLE_RING : LZ4D_H_SINGLE_GLOBAL);
          Lz4pSlot* q = lz4p_acquire(slots, k);
          if (lane == 0) {
            q->type = LZ4P_SINGLE; q->p[0] = (u32)ip; q->p[1] = (u32)op; q->p[2] = (u32)lit; q->p[3] = (u32)total; q->p[4] = (u32)off;
            q->p[5] = use_ring ? 1u : 0u;
          }
          lz4p_publish(k);
          ip += 3 + lit; op += total;
          LZ4D_DBG(g_dbg_lz4d_fast_seqs);
          continue;
        }
      }
    }
    /* ---- general path ---- */
    LZ4D_DBG(g_dbg_lz4d_general_seqs);
    const u32 token = in[ip++];
    int len = (int)(token >> 4);
    if (len == 15) {                                          /* read_variable_length(ip, iend-15, 1) */
      u32 sb;
      if (ip >= iend - 15) { result = LZ4D_FAIL; break; }
      do {
        sb = in[ip++];
        len += (int)sb;
        if (ip > iend - 15) { result = LZ4D_FAIL; break; }
        if (len > oend) { result = LZ4D_FAIL; break; }
      } while (sb == 255);
      if (result < 0) break;
    }
    int cpy = op + len;
    const bool last = cpy > oend - LZ4_MFLIMIT || ip + len > iend - (2 + 1 + LZ4_LASTLITERALS);   /* lz4.c:2289-2331 */
    if (last && (ip + len != iend || cpy > oend)) { result = LZ4D_FAIL; break; }
    const int lsrc = ip, lop = op;
    if (len > LZ4D_RING - 64) { ring_lo = cpy - (LZ4D_RING - 64) > ring_lo ? cpy - (LZ4D_RING - 64) : ring_lo; LZ4D_HIT(LZ4D_H_GEN_LITBUMP); }
    if (last) {
      LZ4D_HIT(LZ4D_H_GEN_LAST);
      Lz4pSlot* q = lz4p_acquire(slots, k);
      if (lane == 0) { q->type = LZ4P_GENERAL; q->p[0] = (u32)lsrc; q->p[1] = (u32)lop; q->p[2] = (u32)len; q->p[3] = 0u; q->p[4] = 0u; q->p[5] = 0u; }
      lz4p_publish(k);
      op += len;
      result = op;
      break;
    }
    ip += len; op = cpy;
    const int off = (int)in[ip] | ((int)in[ip + 1] << 8);
    ip += 2;
    const int match = op - off;
    int mlen = (int)(token & 15u);
    if (mlen == 15) {                                         /* read_variable_length(ip, iend-4, 0) */
      u32 sb;
      do {
        sb = in[ip++];
        mlen += (int)sb;
        if (ip > iend - LZ4_LASTLITERALS + 1) { result = LZ4D_FAIL; break; }
        if (mlen > oend) { result = LZ4D_FAIL; break; }
      } while (sb == 255);
      if (result < 0) break;
    }
    mlen += 4;
    /* the literals of a sequence that turns out to be damaged are still copied, as lz4_decode_warp does before it
     * looks at the match */
    int how = 0;
    bool ok = true;
    if (match < 0) { ok = false; LZ4D_FAIL_NOTE(); }          /* lz4.c:2356 */
    cpy = op + mlen;
    if (ok && cpy > oend - LZ4_LASTLITERALS) { ok = false; LZ4D_FAIL_NOTE(); }   /* lz4.c:2423 */
    if (ok) {
      if (off == 0) { how = 0; ring_lo = cpy; }
      else if (mlen <= 2048) how = (off <= LZ4D_RING - 2048 - 64 && match >= ring_lo) ? 1 : 2;
      else { how = 3; ring_lo = cpy; }
      LZ4D_HIT(how == 0 ? LZ4D_H_GEN_OFF0 : how == 1 ? LZ4D_H_GEN_RING : how == 2 ? LZ4D_H_GEN_GLOBAL : LZ4D_H_GEN_LONG);
    }
    {
      Lz4pSlot* q = lz4p_acquire(slots, k);
      if (lane == 0) {
        q->type = LZ4P_GENERAL; q->p[0] = (u32)lsrc; q->p[1] = (u32)lop; q->p[2] = (u32)len; q->p[3] = ok ? (u32)mlen : 0u;
        q->p[4] = (u32)off; q->p[5] = (u32)how;
      }
      lz4p_publish(k);
    }
    if (!ok) { result = -1; break; }
    op = cpy;
  }
  /* end of the stream: the copier takes END, and the parser waits until everything before it has been copied */
  {
    Lz4pSlot* q = lz4p_acquire(slots, k);
    if (lane == 0) q->type = LZ4P_END;
    lz4p_publish(k);
    lz4p_drain(k);
  }
  __syncwarp();
  return result;
}

/* tell the copier that there are no more streams */
DEV void lz4_pair_quit(Lz4pSlot* slots) {
  if (lane_id() == 0) slots[0].type = LZ4P_QUIT;
  __syncwarp();
  __threadfence_block();
  bar_arrive(LZ4P_BAR_FULL(0), 64);
}

/*
 * dev_lz4fast.cuh -- the segment-parallel LZ4 encoder (BLOSC_B200_PARSE=fast), sm_90a.
 *
 * dev_lz4.cuh replays LZ4_compress_fast's greedy parse bit for bit, which makes every stream one
 * serial dependency chain (one warp, ~10 k dependent steps on the hard byte-plane of bench.c data).
 * This file is the GPU-native alternative: it writes the same FORMAT -- LZ4 blocks that
 * LZ4_decompress_safe (reference internal-complibs/lz4-1.10.0/lz4.c:2022-2445, called from
 * blosc/blosc.c:435-439) decodes -- but not the same bytes, and it has no serial chain longer than
 * one kilobyte of input:
 *
 *   index   one warp per stream walks the stream 128 positions at a time and records, for EVERY
 *           position p, the distance to the most recent earlier position (before this batch of 128)
 *           whose 5 bytes hash alike: prev[p] (u16, 0 = none).  Followed repeatedly, prev[] is the
 *           hash chain of LZ4HC (lz4hc.c chainTable), complete and read-only.
 *   parse   the stream is cut into segments of FAST_SEG bytes; every LANE parses one segment on its
 *           own (32 segments per warp, thousands of warps): at each position it follows the chain
 *           for up to `depth` candidates, keeps the longest match, and emits LZ4 sequences into the
 *           segment's slot.  Matches may reach back across segment boundaries (the input is all
 *           there); they never run past the end of their own segment.
 *   stitch  a segment's leading / trailing literals belong to a sequence that straddles the boundary:
 *           they are not written by the parser but recorded (FastSeg), a per-stream scan turns the
 *           records into output offsets and the stream's compressed size, and compact_kernel writes
 *           the merged token / literal-length bytes while it copies the pieces to their final place.
 *
 * The chain search finds longer matches than LZ4_compress_fast's single probe, so on the bench.c
 * planes the ratio is better than the reference's (DESIGN.md has the table).
 */
#pragma once
#include "b2_args.h"
#include "dev_common.cuh"

#define FAST_SEG B2_FAST_SEG          /* bytes per segment (one lane) */
#define FAST_HLOG 12
#define FAST_TAB_BYTES (4 << FAST_HLOG)   /* index kernel: 4096 x u32 per warp */
#define FAST_BATCH 128                /* positions per index step (4 per lane) */
#ifndef FAST_SMALL
#define FAST_SMALL 4
#endif
#ifndef FAST_BUDGET
#define FAST_BUDGET 12
#endif
#define FAST_NICE 4096                  /* a match this long is taken without walking the chain */
#define FAST_MFLIMIT 12               /* lz4.c:239-243: the last match starts >= 12 bytes before the end ... */
#define FAST_LASTLITERALS 5           /* ... and the last 5 bytes are literals */

/* aligned-word view of a byte stream: never touches a word that lies entirely outside [s, s+n) */
struct FastView {
  const u32* w;      /* aligned word holding s[0] */
  int sal;           /* s - (const u8*)w */
  int nwords;        /* words that overlap the stream */
  const u32* sm;     /* words [sm_lo, sm_hi) of the stream are also in shared memory, at sm[i - sm_lo] */
  int sm_lo, sm_hi;
  int lo_pos;        /* positions >= lo_pos (and below the end of the window) can be read from shared memory ... */
  int bias;          /* ... at byte p + bias of `sm` */
};
DEV FastView fast_view(const u8* s, int n) {
  FastView v;
  v.sal = (int)((uintptr_t)s & 3u);
  v.w = (const u32*)(s - v.sal);
  v.nwords = (n + v.sal + 3) >> 2;
  v.sm = nullptr; v.sm_lo = 0; v.sm_hi = 0; v.lo_pos = 0x7fffffff; v.bias = 0;
  return v;
}
DEV u32 fast_word(const FastView& v, int i) {
  if (i >= v.sm_lo && i < v.sm_hi) return v.sm[i - v.sm_lo];
  return i < v.nwords ? __ldg(v.w + i) : 0u;
}
/* 4 bytes at position p (p >= 0); bytes past the end of the stream read as zero */
DEV u32 fast_ld32(const FastView& v, int p) {
  if (p >= v.lo_pos) {                             /* the common case: inside the window */
    const u32 x = (u32)(p + v.bias);
    const u32* w = v.sm + (x >> 2);
    return __funnelshift_r(w[0], w[1], (x & 3u) * 8u);
  }
  const int q = p + v.sal;
  const u32 lo = fast_word(v, q >> 2);
  const u32 sh = (u32)(q & 3) * 8u;
  if (sh == 0) return lo;
  return __funnelshift_r(lo, fast_word(v, (q >> 2) + 1), sh);
}
DEV u32 fast_ld8(const FastView& v, int p) {
  const int q = p + v.sal;
  return (fast_word(v, q >> 2) >> ((u32)(q & 3) * 8u)) & 0xffu;
}

/* hash of the 4..6 bytes word | b45 << 32 (b45 = the bytes that follow the word, masked: 0xffff = 6-byte hash, the LZ4 fast
 * setting; 0 = 4-byte hash = LZ4's MINMATCH, the "lz4hc" setting) */
DEV u32 fast_hash(u32 word, u32 b45) { return ((word * 2654435761u) ^ (b45 * 2246822519u)) >> (32 - FAST_HLOG); }

/* ---- index: prev[p] for every position of one stream, by one warp ----
 * Every step takes FAST_BATCH = 128 positions (4 consecutive ones per lane): hash, look the table up (state as of
 * the end of the previous step), then enter the 128 positions (atomicMax: the highest position wins, whatever the
 * order of the lanes).  A lane loads ONE aligned word per step -- its neighbours' words arrive by shuffle -- and the
 * words of the next two steps are requested before this step's table work, so the only latency on the step-to-step
 * chain is the shared-memory round trip.  Table entries are positions; "empty" is a position so far back that
 * the distance test rejects it. */
#define FAST_EMPTY (-(1 << 20))
DEV void lz4f_index_warp(const u8* __restrict__ s, const int n, u16* __restrict__ prev, u32* tabmem, const u32 hmask) {
  int* tab = (int*)tabmem;
  const int lane = lane_id();
  for (int i = lane; i < (1 << FAST_HLOG); i += 32) tab[i] = FAST_EMPTY;
  __syncwarp();
  const FastView v = fast_view(s, n);
  const bool vec = (((uintptr_t)prev) & 7u) == 0;
  const u32 sh = (u32)v.sal * 8u;
  /* lane's word of a step: (base + 4 lane + sal) >> 2 = base/4 + lane.  The step uses its own words and three words
   * of the next step: both were requested at least a step ago, and one lane pulls the line of eight steps ahead
   * into L1, so that no step waits for DRAM. */
  u32 cur = fast_word(v, lane), nxt = fast_word(v, (FAST_BATCH >> 2) + lane);
  for (int base = 0; base < n; base += FAST_BATCH) {
    const int p0 = base + 4 * lane;
    const u32 w0 = cur;
    cur = nxt;
    nxt = fast_word(v, ((base + 2 * FAST_BATCH) >> 2) + lane);
#ifndef SIMT_EMU
    if (lane == 0 && base + 10 * FAST_BATCH < n) asm volatile("prefetch.global.L1 [%0];" :: "l"(s + base + 8 * FAST_BATCH));
#endif
    /* the three words behind the lane's own: the next lanes' words, or the first words of the next step */
    const u32 d1 = __shfl_down_sync(FULLMASK, w0, 1), d2 = __shfl_down_sync(FULLMASK, w0, 2), d3 = __shfl_down_sync(FULLMASK, w0, 3);
    const u32 e1 = __shfl_sync(FULLMASK, cur, (lane + 1) & 31), e2 = __shfl_sync(FULLMASK, cur, (lane + 2) & 31),
              e3 = __shfl_sync(FULLMASK, cur, (lane + 3) & 31);
    const u32 w1 = lane < 31 ? d1 : e1, w2 = lane < 30 ? d2 : e2, w3 = lane < 29 ? d3 : e3;
    /* bytes p0 .. p0+11 */
    const u32 v0 = __funnelshift_r(w0, w1, sh), v1 = __funnelshift_r(w1, w2, sh), v2 = __funnelshift_r(w2, w3, sh);
    u32 h[4];
    int c[4];
    /* a step inside a run of one byte value (the zero planes of shuffled data are nothing else): every position has
     * the same hash, one lookup and one table store serve the whole step */
    const u32 b0 = __shfl_sync(FULLMASK, v0, 0);
    const bool runstep = base != 0 && base + FAST_BATCH + 8 <= n &&
                         __all_sync(FULLMASK, v0 == b0 && v1 == b0 && v2 == b0 && b0 == __funnelshift_r(b0, b0, 8));
    if (runstep) {
      const u32 hr = fast_hash(b0, b0 & hmask);
      const int cr = tab[hr];
      __syncwarp();
      if (lane == 31) tab[hr] = p0 + 3;
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 4; j++) c[j] = cr;
    } else {
#pragma unroll
    for (int j = 0; j < 4; j++)
      h[j] = fast_hash(__funnelshift_r(v0, v1, 8u * j), __funnelshift_r(v1, v2, 8u * j) & hmask);
    if (base == 0) {
      /* the first batch has nothing in front of it: resolve it position by position, so that a run or a
       * short period at the very start of a stream is found from its second occurrence on */
      for (int m = 0; m < 32; m++) {
        if (lane == m) {
#pragma unroll
          for (int j = 0; j < 4; j++) {
            c[j] = FAST_EMPTY;
            if (p0 + j + 8 <= n) { c[j] = tab[h[j]]; tab[h[j]] = p0 + j; }
          }
        }
        __syncwarp();
      }
    } else if (base + FAST_BATCH + 8 <= n) {        /* every position of the step has its 8 bytes inside the stream */
#pragma unroll
      for (int j = 0; j < 4; j++) c[j] = tab[h[j]];
      __syncwarp();
      /* a run (every position of the step hashes alike -- the zero planes of shuffled data) would make the
       * 128 atomics collide on one word: the last position enters it alone */
      const u32 hl = __shfl_sync(FULLMASK, h[3], 0);
      const bool same = h[0] == h[1] && h[1] == h[2] && h[2] == h[3] && h[3] == hl;
      if (__all_sync(FULLMASK, same)) {
        if (lane == 31) tab[h[3]] = p0 + 3;
      } else {
#pragma unroll
        for (int j = 0; j < 4; j++)
          if (j == 3 || h[j] != h[j + 1]) atomicMax(&tab[h[j]], p0 + j);
      }
      __syncwarp();
    } else {                                          /* the last step(s) of the stream */
#pragma unroll
      for (int j = 0; j < 4; j++) c[j] = p0 + j + 8 <= n ? tab[h[j]] : FAST_EMPTY;
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 4; j++)
        if (p0 + j + 8 <= n) atomicMax(&tab[h[j]], p0 + j);
      __syncwarp();
    }
    }
    u32 d[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const u32 delta = (u32)(p0 + j - c[j]);
      d[j] = delta <= 65535u ? delta : 0u;
    }
    if (p0 + 4 <= n && vec) *(uint2*)(prev + p0) = make_uint2(d[0] | (d[1] << 16), d[2] | (d[3] << 16));
    else {
#pragma unroll
      for (int j = 0; j < 4; j++) if (p0 + j < n) prev[p0 + j] = (u16)d[j];
    }
  }
}

/* number of equal bytes of s[p..] and s[q..] (q < p), at most `lim`: one new aligned word per side and 4 bytes */
DEV int fast_count(const FastView& v, int p, int q, int lim) {
  if (lim <= 0) return 0;
  int c = 0;
  if (q >= v.lo_pos) {                                          /* both sides inside the shared-memory window */
    const u32 px = (u32)(p + v.bias), qx = (u32)(q + v.bias);
    const u32 psh = (px & 3u) * 8u, qsh = (qx & 3u) * 8u;
    const u32* ps = v.sm + (px >> 2);
    const u32* qs = v.sm + (qx >> 2);
    u32 pl = ps[0], ql = qs[0];
    for (;;) {
      const u32 ph = *++ps, qh = *++qs;
      const u32 x = __funnelshift_r(pl, ph, psh) ^ __funnelshift_r(ql, qh, qsh);
      if (x) { c += (__ffs((int)x) - 1) >> 3; break; }
      c += 4;
      if (c >= lim) break;
      pl = ph; ql = qh;
    }
  } else {
    int pi = (p + v.sal) >> 2, qi = (q + v.sal) >> 2;
    const u32 psh = (u32)((p + v.sal) & 3) * 8u, qsh = (u32)((q + v.sal) & 3) * 8u;
    u32 pl = fast_word(v, pi), ql = fast_word(v, qi);
    for (;;) {
      const u32 ph = fast_word(v, ++pi), qh = fast_word(v, ++qi);
      const u32 x = __funnelshift_r(pl, ph, psh) ^ __funnelshift_r(ql, qh, qsh);
      if (x) { c += (__ffs((int)x) - 1) >> 3; break; }
      c += 4;
      if (c >= lim) break;
      pl = ph; ql = qh;
    }
  }
  return c < lim ? c : lim;
}

DEV int fast_lit_ext(int lit) { return lit >= 15 ? 1 + (lit - 15) / 255 : 0; }

/* Longest match for position ip among: the offset `rep`, the offsets 1..4, and up to `de` candidates of the hash
 * chain no farther than MAXD (DEFLATE's window is 32768).  Returns its length (0: none) and *off. */
template <int MAXD = 65535>
DEV int lz4f_search(const FastView& v, const u16* __restrict__ prev, const int ip, const int mlim, const int rep, const int rep_len,
                    const int de, int* off) {
  const u32 wip = fast_ld32(v, ip);
  int best = 0, boff = 0, q = ip;
  if (rep_len) { best = rep_len; boff = rep; }            /* already counted by the caller */
  else if (rep && fast_ld32(v, ip - rep) == wip) {
    best = 4 + fast_count(v, ip + 4, ip - rep + 4, mlim - (ip + 4));
    boff = rep;
  }
  if (ip + best < mlim && best < FAST_NICE) {
    u32 wend = best >= 4 ? fast_ld32(v, ip + best - 3) : 0u;   /* bytes [best-3, best] of the position: the first one a longer match adds */
    for (int d = 0; d < de; d++) {
      const int dl = (int)prev[q];
      if (dl == 0) break;
      q -= dl;
      if (ip - q > MAXD) break;
      /* a candidate can only win if it also matches where the best match so far ends (the LZ4HC test,
       * lz4hc.c LZ4HC_InsertAndGetWiderMatch): most candidates are turned down by this one compare */
      if (best >= 4 && fast_ld32(v, q + best - 3) != wend) continue;
      if (fast_ld32(v, q) == wip) {
        const int len = 4 + fast_count(v, ip + 4, q + 4, mlim - (ip + 4));
        if (len > best) {
          best = len; boff = ip - q;
          if (ip + len >= mlim) break;           /* cannot get longer */
          wend = fast_ld32(v, ip + best - 3);
        }
      }
    }
  }
  if (best < FAST_SMALL && ip >= 4) {
    /* offsets 1..4 straight from the bytes in front of ip: the index only knows occurrences that are at least a
     * batch (<= FAST_BATCH positions) old, so the start of a run or of a short period would otherwise stay literal */
    const u32 wb = fast_ld32(v, ip - 4);
    int o = 0;
    if (__funnelshift_r(wb, wip, 24) == wip) o = 1;
    else if (__funnelshift_r(wb, wip, 16) == wip) o = 2;
    else if (__funnelshift_r(wb, wip, 8) == wip) o = 3;
    else if (wb == wip) o = 4;
    if (o) {
      const int len = 4 + fast_count(v, ip + 4, ip - o + 4, mlim - (ip + 4));
      if (len > best) { best = len; boff = o; }
    }
  }
  if (ip + best > mlim) best = 0;
  *off = boff;
  return best;
}

/* ---- parse: one lane, one segment [a, b) of the stream ----
 * Slot layout: the segment's sequences back to back, except that (1) the first sequence has no literal-length
 * bytes and no literals (the stitcher merges them with what the previous segments left pending) and (2) the
 * LAST sequence has no match-length extension bytes: a match that ends exactly at the end of the segment may
 * be continued by the segments that follow (runs, periodic data), so its final length is only known to the
 * stream scan. */
DEV void lz4f_parse_lane(const FastView& v, const int n, const u16* __restrict__ prev, const int a, const int b,
                         u8* __restrict__ slot, FastSeg* rec, const int depth, const int accel, const int lazy) {
  int mfl = b - 4, mlim = b;                     /* last position a match may start at; first byte it may not cover */
  if (mfl > n - FAST_MFLIMIT) mfl = n - FAST_MFLIMIT;
  if (mlim > n - FAST_LASTLITERALS) mlim = n - FAST_LASTLITERALS;
  int ip = a, anchor = a, op = 0, l1 = 0, miss = 0;
  int lt = 0, lm = 0, lo = 0;                    /* last sequence: token position in the slot, match length, offset */
  int step = 1, snb = accel << 6;                /* LZ4's skip schedule (lz4.c:1043-1053) */
  int nsearch = 0;
  bool first = true;
  /* `rep`: an offset worth trying before the chain.  Inside a segment it is the offset of the last match (periodic
   * data: the match that a glitch ended resumes right behind it).  At the start of a segment it is whichever chain
   * candidate of the byte in FRONT of the segment continues best into it -- normally the offset the previous
   * segment's lane ends with, so that a match which covers this whole segment can simply be continued. */
  int rep = 0, pre = 0;
  if (a > 0 && a <= mfl) {
    const u32 wa = fast_ld32(v, a);
    int q = a - 1, bl = 0;
    for (int d = 0; d < 8; d++) {
      const int dl = (int)prev[q];
      if (dl == 0) break;
      q -= dl;
      const int o = a - 1 - q;
      if (o > 65535) break;
      if (fast_ld32(v, a - o) == wa) {
        const int len = 4 + fast_count(v, a + 4, a - o + 4, mlim - (a + 4));
        if (len > bl) { bl = len; rep = o; }
        if (a + len >= mlim) break;
      }
    }
    pre = bl;
  }
  while (ip <= mfl) {
    int de = depth >> ((miss >> 3) < 5 ? (miss >> 3) : 5);   /* a run of misses (incompressible data) shortens the chain walk */
    if (nsearch >= FAST_BUDGET) de >>= 1;                     /* the slowest segment of a window sets its time: a segment that needs many searches walks shorter chains */
    if (nsearch >= 2 * FAST_BUDGET) de >>= 1;
    nsearch++;
    if (de < 2) de = 2;
    int boff = 0;
    int best = lz4f_search(v, prev, ip, mlim, rep, ip == a ? pre : 0, de, &boff);
    if (best >= 4 && best < lazy && ip + 1 <= mfl) {
      /* lazy evaluation (as LZ4HC / zlib): a short match is given up for a literal when the next position
       * starts a longer one */
      int boff2 = 0;
      const int best2 = lz4f_search(v, prev, ip + 1, mlim, rep, 0, de, &boff2);
      if (best2 > best + 1) { ip++; best = best2; boff = boff2; }
    }
    const int lit = ip - anchor;
    if (best >= 4 && ip + best <= mlim && !(lit >= 15 && best < 9)) {   /* a sequence never takes more bytes than it covers */
      const int mc = best - 4;
      if (first) {
        l1 = lit;
        first = false;
        lt = op;
        slot[op++] = (u8)(mc < 15 ? mc : 15);
      } else {
        if (lm - 4 >= 15) {                      /* the previous sequence was not the last one: its length bytes */
          int r = lm - 4 - 15;
          while (r >= 255) { slot[op++] = 255; r -= 255; }
          slot[op++] = (u8)r;
        }
        lt = op;
        slot[op++] = (u8)(((lit < 15 ? lit : 15) << 4) | (mc < 15 ? mc : 15));
        if (lit >= 15) {
          int r = lit - 15;
          while (r >= 255) { slot[op++] = 255; r -= 255; }
          slot[op++] = (u8)r;
        }
        for (int k = 0; k < lit; k++) slot[op + k] = (u8)fast_ld8(v, anchor + k);
        op += lit;
      }
      slot[op++] = (u8)boff; slot[op++] = (u8)(boff >> 8);
      lm = best; lo = boff; rep = boff;
      ip += best; anchor = ip;
      miss = 0; step = 1; snb = accel << 6;
    } else {
      ip += step; step = (snb++) >> 6;
      miss++;
    }
  }
  rec->nbytes = (u16)op; rec->l1 = (u16)l1; rec->tail = (u16)(b - anchor); rec->lt = (u16)lt;
  rec->lm = (u16)lm; rec->lo = (u16)lo; rec->pad0 = 0; rec->pad1 = 0;
}

DEV int fast_ml_ext(int ml) { return ml - 4 >= 15 ? 1 + (ml - 4 - 15) / 255 : 0; }

/* ---- per-stream scan of the segment records: pending literals, continued matches, output offsets, size ----
 * Run by one warp once every segment of the stream has been parsed; the walk over the K records is sequential
 * (a few instructions per record, every lane computes the same state; records are fetched 32 at a time and
 * broadcast by shuffles).  A segment that is ONE match over all its bytes, with the offset of the match that
 * ends the segment before it, is swallowed: that match simply goes on.  Returns the size of the merged LZ4
 * block (uniform); *ptail = literals after the stream's last match. */
DEV int lz4f_stream_scan(FastSeg* segs, const int K, const int n, int* ptail) {
  const int lane = lane_id();
  long long pos = 0;
  int carry = 0;                      /* literals since the last match */
  int head = -1, head_total = 0, head_lo = 0;   /* open sequence: last match of segment `head` ends at a segment boundary */
  for (int k0 = 0; k0 < K; k0 += 32) {
    u32 r0 = 0, r1 = 0, r2 = 0;
    if (k0 + lane < K) {
#ifdef SIMT_EMU
      const FastSeg* r = &segs[k0 + lane];
      r0 = (u32)r->nbytes | ((u32)r->l1 << 16); r1 = (u32)r->tail | ((u32)r->lt << 16); r2 = (u32)r->lm | ((u32)r->lo << 16);
#else
      const uint4 q = __ldcg((const uint4*)&segs[k0 + lane]);     /* written by other SMs during this launch */
      r0 = q.x; r1 = q.y; r2 = q.z;
#endif
    }
    const int cnt = K - k0 < 32 ? K - k0 : 32;
    for (int j = 0; j < cnt; j++) {
      const u32 x0 = __shfl_sync(FULLMASK, r0, j), x1 = __shfl_sync(FULLMASK, r1, j), x2 = __shfl_sync(FULLMASK, r2, j);
      const int nb = (int)(x0 & 0xffffu), l1 = (int)(x0 >> 16), tl = (int)(x1 & 0xffffu), lt = (int)(x1 >> 16);
      const int lm = (int)(x2 & 0xffffu), lo = (int)(x2 >> 16);
      const int k = k0 + j;
      const int a = k * FAST_SEG, len = (a + FAST_SEG < n ? a + FAST_SEG : n) - a;
      if (nb == 0) {                                                   /* all literals */
        if (head >= 0) { pos += fast_ml_ext(head_total); if (lane == 0) segs[head].run = (u32)head_total; head = -1; }
        carry += tl;
        continue;
      }
      if (head >= 0 && lt == 0 && l1 == 0 && tl == 0 && lm == len && lo == head_lo) {   /* swallowed */
        head_total += len;
        if (lane == 0) segs[k].dst = 0xffffffffu;
        continue;
      }
      if (head >= 0) { pos += fast_ml_ext(head_total); if (lane == 0) segs[head].run = (u32)head_total; head = -1; }
      const int lit = carry + l1;
      if (lane == 0) { segs[k].dst = (u32)pos; segs[k].pin = (u32)carry; }
      pos += 1 + fast_lit_ext(lit) + lit + (nb - 1);
      if (tl == 0) { head = k; head_total = lm; head_lo = lo; carry = 0; }
      else { pos += fast_ml_ext(lm); if (lane == 0) segs[k].run = (u32)lm; carry = tl; }
    }
  }
  if (head >= 0) { pos += fast_ml_ext(head_total); if (lane == 0) segs[head].run = (u32)head_total; }
  pos += 1 + fast_lit_ext(carry) + carry;
  *ptail = carry;
  return pos > 0x7fffffffll ? 0x7fffffff : (int)pos;
}

/* `cnt` length bytes of a literal / match length `r` = value - 15 at o[0..): 255 ... 255, remainder */
DEV void fast_put_ext(u8* o, int r, int lane) {
  const int nff = r / 255;
  for (int i = lane; i < nff; i += 32) o[i] = 255;
  if (lane == 0) o[nff] = (u8)(r - nff * 255);
}

/* ---- stitch: copy one fast-parsed stream to its final place (called by compact_kernel, whole CTA) ----
 * `dst` receives `c` bytes.  One warp per segment that was not swallowed: the merged first token, the
 * literal-length bytes, the pending + leading literals (straight from the input), the rest of the slot with the
 * last token's match nibble brought up to date, and the length bytes of the last match; then the last literals. */
DEV void lz4f_stitch_cta(u8* __restrict__ dst, const int c, const u8* __restrict__ s, const int n,
                         const u8* __restrict__ slots, const FastSeg* __restrict__ segs, const int K, const int ptail) {
  const int lane = lane_id();
  const int warp = (int)(threadIdx.x >> 5), nwarps = (int)(blockDim.x >> 5);
  if (warp == 0) {                                /* last literals (lz4.c:1302-1329) */
    const int lit = ptail;
    u8* o = dst + (c - (1 + fast_lit_ext(lit) + lit));
    if (lane == 0) o[0] = (u8)((lit < 15 ? lit : 15) << 4);
    int h = 1;
    if (lit >= 15) { fast_put_ext(o + 1, lit - 15, lane); h += fast_lit_ext(lit); }
    for (int i = lane; i < lit; i += 32) o[h + i] = s[n - lit + i];
  }
  /* a warp takes 32 records at a time (one per lane, two 16-byte loads each) and then walks the ones that have
   * something to copy: one record load per segment and warp would leave the kernel waiting for L2 */
  for (int k0 = warp * 32; k0 < K; k0 += nwarps * 32) {
    u32 g0 = 0, g1 = 0, gd = 0xffffffffu, gp = 0, gr = 0;
    if (k0 + lane < K) {
      const FastSeg* r = &segs[k0 + lane];
      g0 = (u32)r->nbytes | ((u32)r->l1 << 16); g1 = (u32)r->lt;
      gd = r->dst; gp = r->pin; gr = r->run;
    }
    unsigned act = __ballot_sync(FULLMASK, (g0 & 0xffffu) != 0u && gd != 0xffffffffu);
    for (; act; act &= act - 1u) {
      const int j = __ffs((int)act) - 1;
      const int k = k0 + j;
      const u32 x0 = __shfl_sync(FULLMASK, g0, j), x1 = __shfl_sync(FULLMASK, g1, j);
      const u32 xd = __shfl_sync(FULLMASK, gd, j), xp = __shfl_sync(FULLMASK, gp, j), xr = __shfl_sync(FULLMASK, gr, j);
      const int nb = (int)(x0 & 0xffffu), l1 = (int)(x0 >> 16), lt = (int)x1, total = (int)xr;
      const int a = k * FAST_SEG;
      const int lit = (int)xp + l1;
      const u32 mn = (u32)(total - 4 < 15 ? total - 4 : 15);
      const u8* sl = slots + a;
      u8* o = dst + xd;
      if (lane == 0) o[0] = (u8)(((lit < 15 ? lit : 15) << 4) | (lt == 0 ? mn : (u32)(sl[0] & 15u)));
      int h = 1;
      if (lit >= 15) { fast_put_ext(o + 1, lit - 15, lane); h += fast_lit_ext(lit); }
      const u8* ls = s + a + l1 - lit;              /* the literals are contiguous in the input and end at the first match */
      for (int i = lane; i < lit; i += 32) o[h + i] = ls[i];
      h += lit;
      for (int i = 1 + lane; i < nb; i += 32) {
        u32 b = sl[i];
        if (i == lt) b = (b & 0xf0u) | mn;
        o[h + i - 1] = (u8)b;
      }
      if (total - 4 >= 15) fast_put_ext(o + h + nb - 1, total - 4 - 15, lane);
    }
  }
}

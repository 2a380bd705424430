/*
 * dev_zstdenc.cuh -- the segment-parallel zstd encoder (Blosc's "zstd" codec), sm_90a.
 *
 * It writes one zstd frame (RFC 8878) per stream that ZSTD_decompress (reference blosc/blosc.c:517-529) and
 * dev_zstd.cuh both accept -- not ZSTD_compress's bytes.  Three launches after index_kernel (dev_lz4fast.cuh, whose
 * prev[] hash chains and lz4f_search are used as they are):
 *
 *   zparse   every THREAD parses one segment of FAST_SEG bytes against the hash chains (the same search as the
 *            "lz4hc" parse) and writes plain sequence records -- literal length, match length, offset -- instead of
 *            LZ4 bytes.  Matches never cross a segment boundary.
 *   zenc     one warp per stream, the work on lane 0: per 128 KiB zstd block (a whole number of segments) stitch
 *            the records in order -- literals pending across segments go in front of the next match, a match that
 *            continues across a boundary with the same offset is merged -- resolve the repeat offsets (their
 *            history runs on across the blocks of the frame), then entropy code the block: Huffman literals
 *            (direct or FSE-coded weights, codes <= 11 bits, 1 or 4 streams), LL/ML/OF codes in predefined, RLE
 *            or FSE_Compressed mode, whichever is smallest.  A block that does not shrink is stored raw.
 *   (scan / compact as for every codec: csizes[] -> bstarts -> the chunk)
 *
 * Scratch: the records go to a buffer of 256 bytes per segment (64 records of 4 bytes: a match is >= 4 bytes),
 * the stitched sequences and the gathered literals of the block being coded to the stream's own part of prev[]
 * (2 bytes per input byte, dead once zparse is done), the frame to the stream's slot.  Nothing depends on the
 * order in which warps or threads run, so the device bytes equal the emulator's.
 */
#pragma once
#include "b2_args.h"
#include "dev_common.cuh"
#include "dev_lz4fast.cuh"
#include "dev_zstd.cuh"

#define ZE_SEG_RECS (FAST_SEG / 4)                   /* records per segment */
#define ZE_BLOCK_SEGS (ZS_BLOCKMAX / FAST_SEG)       /* segments per zstd block */
#define ZE_WARPS 4

/* ---- zparse: one lane, one segment [a, b) of the stream ----
 * record = literal length (8 bits, from the end of the previous match or the segment start) | (match length - 4) << 8
 * | offset << 16, offsets <= MAXD (the DEFLATE encoder, dev_deflate.cuh, parses with 32768).  Returns the number of
 * records. */
template <int MAXD = 65535>
DEV int zse_parse_lane(const FastView& v, const int n, const u16* __restrict__ prev, const int a, const int b,
                       u32* __restrict__ rec, const int depth, const int lazy) {
  const int mlim = b < n ? b : n, mfl = mlim - 4;    /* a match lies inside the segment and has >= 4 bytes */
  int ip = a, anchor = a, cnt = 0, miss = 0, nsearch = 0;
  int step = 1, snb = 1 << 6;                         /* long runs of misses are skipped faster (lz4.c:1043-1053) */
  int rep = 0, pre = 0;
  if (a > 0 && a <= mfl) {                            /* the offset the previous segment most likely ends with */
    const u32 wa = fast_ld32(v, a);
    int q = a - 1, bl = 0;
    for (int d = 0; d < 8; d++) {
      const int dl = (int)prev[q];
      if (dl == 0) break;
      q -= dl;
      const int o = a - 1 - q;
      if (o > MAXD) break;
      if (fast_ld32(v, a - o) == wa) {
        const int len = 4 + fast_count(v, a + 4, a - o + 4, mlim - (a + 4));
        if (len > bl) { bl = len; rep = o; }
        if (a + len >= mlim) break;
      }
    }
    pre = bl;
  }
  while (ip <= mfl && cnt < ZE_SEG_RECS) {
    int de = depth >> ((miss >> 3) < 5 ? (miss >> 3) : 5);
    if (nsearch >= FAST_BUDGET) de >>= 1;
    if (nsearch >= 2 * FAST_BUDGET) de >>= 1;
    nsearch++;
    if (de < 2) de = 2;
    int boff = 0;
    int best = lz4f_search<MAXD>(v, prev, ip, mlim, rep, ip == a ? pre : 0, de, &boff);
    if (best >= 4 && best < lazy && ip + 1 <= mfl) {
      int boff2 = 0;
      const int best2 = lz4f_search<MAXD>(v, prev, ip + 1, mlim, rep, 0, de, &boff2);
      if (best2 > best + 1) { ip++; best = best2; boff = boff2; }
    }
    if (best >= 4 && ip + best <= mlim) {
      rec[cnt++] = (u32)(ip - anchor) | ((u32)(best - 4) << 8) | ((u32)boff << 16);
      rep = boff;
      ip += best; anchor = ip;
      miss = 0; step = 1; snb = 1 << 6;
    } else {
      ip += step; step = (snb++) >> 6;
      miss++;
    }
  }
  return cnt;
}

/* ---- entropy stage: tables in the warp's shared memory ---- */
struct ZeCT {                 /* FSE encoding table (zstd fse_compress.c layout) */
  u16 st[512];                /* state table */
  u32 dnb[64];                /* per symbol: deltaNbBits */
  int dfs[64];                /* per symbol: deltaFindState */
  int log;
};
struct ZeSm {
  ZeCT ct[3];                 /* LL, OF, ML */
  ZeCT wt;                    /* Huffman weights */
  u32 hist[256];              /* literal counts */
  u32 cnt[3][64];             /* LL / OF / ML code counts */
  short norm[4][64];
  u16 hcode[256];
  u8 hlen[256];
  u32 nc[512];                /* Huffman tree: node weights, then parents */
  u16 par[512];
  u16 leaf[256];              /* symbols sorted by count */
  u8 tsym[512];
  u8 w[256];                  /* Huffman weights as written */
};
#define ZE_SMEM_BYTES ((int)((sizeof(ZeSm) + 15) & ~(size_t)15))

/* forward bit writer (LSB first, as zstd's BIT_CStream), bounded by `cap` */
struct ZeBW { u8* p; int pos, cap; u64 acc; int nb; bool over; };
DEV void zbw_init(ZeBW& w, u8* p, int cap) { w.p = p; w.pos = 0; w.cap = cap; w.acc = 0; w.nb = 0; w.over = false; }
DEV void zbw_add(ZeBW& w, u32 v, int n) {
  if (n == 0) return;
  w.acc |= (u64)(v & (n == 32 ? 0xffffffffu : ((1u << n) - 1u))) << w.nb;
  w.nb += n;
  while (w.nb >= 8) {
    if (w.pos < w.cap) w.p[w.pos] = (u8)w.acc; else w.over = true;
    w.pos++; w.acc >>= 8; w.nb -= 8;
  }
}
DEV int zbw_close(ZeBW& w) {                       /* end mark, last partial byte; returns the bytes written */
  zbw_add(w, 1, 1);
  if (w.nb > 0) { if (w.pos < w.cap) w.p[w.pos] = (u8)w.acc; else w.over = true; w.pos++; w.acc = 0; w.nb = 0; }
  return w.pos;
}

DEV int ze_hb(u32 v) { return 31 - __clz((int)v); }         /* v != 0 */
/* log2 with 8 fractional bits, linear between powers of two (integer only: the same on host and device) */
DEV int ze_log2fix(u32 v) { const int h = ze_hb(v); return (h << 8) + (int)(((u64)v << 8 >> h) - 256u); }

DEV int ze_llcode(u32 ll) {
  if (ll < 16) return (int)ll;
  if (ll >= 64) return ze_hb(ll) + 19;
  int c = 16;
  while (c < 35 && k_zs_ll_base[c + 1] <= ll) c++;
  return c;
}
DEV int ze_mlcode(u32 ml) {                         /* ml >= 3 */
  const u32 mb = ml - 3;
  if (mb < 32) return (int)mb;
  if (mb >= 128) return ze_hb(mb) + 36;
  int c = 32;
  while (c < 52 && k_zs_ml_base[c + 1] <= ml) c++;
  return c;
}

/* FSE_optimalTableLog */
DEV int ze_table_log(int maxlog, u32 total, int maxsym) {
  int tl = maxlog;
  const int maxsrc = ze_hb(total - 1) - 2;
  const int minsrc = ze_hb(total) + 1, minsym = ze_hb((u32)(maxsym > 0 ? maxsym : 1)) + 2;
  const int minb = minsrc < minsym ? minsrc : minsym;
  if (maxsrc < tl) tl = maxsrc;
  if (minb > tl) tl = minb;
  if (tl < 5) tl = 5;
  if (tl > maxlog) tl = maxlog;
  return tl;
}

/* counts -> normalised counts summing to 2^log, every present symbol >= 1 */
DEV void ze_normalize(const u32* cnt, int nsym, u32 total, int log, short* norm) {
  const int scale = 1 << log;
  int sum = 0, big = 0;
  for (int s = 0; s < nsym; s++) {
    int v = 0;
    if (cnt[s]) { v = (int)(((u64)cnt[s] << log) / total); if (v < 1) v = 1; }
    norm[s] = (short)v;
    sum += v;
    if (cnt[s] > cnt[big]) big = s;
  }
  while (sum > scale) {                             /* the rounding up of rare symbols: taken from the largest */
    int m = -1;
    for (int s = 0; s < nsym; s++) if (norm[s] > 1 && (m < 0 || norm[s] > norm[m])) m = s;
    norm[m]--; sum--;
  }
  norm[big] = (short)(norm[big] + (scale - sum));
}

/* FSE table description (FSE_writeNCount); returns bytes or -1 when it does not fit */
DEV int ze_write_ncount(u8* o, int cap, const short* norm, int nsym, int log) {
  const int size = 1 << log;
  u32 bs = 0;
  int bc = 0, out = 0;
  bs = (u32)(log - 5);
  bc = 4;
  int remaining = size + 1, threshold = size, nbits = log + 1, s = 0;
  bool prev0 = false;
  while (s < nsym && remaining > 1) {
    if (prev0) {
      int start = s;
      while (s < nsym && norm[s] == 0) s++;
      if (s == nsym) break;
      while (s >= start + 24) {
        start += 24;
        bs += 0xffffu << bc;
        if (out + 2 > cap) return -1;
        o[out++] = (u8)bs; o[out++] = (u8)(bs >> 8);
        bs >>= 16;
      }
      while (s >= start + 3) { start += 3; bs += 3u << bc; bc += 2; }
      bs += (u32)(s - start) << bc;
      bc += 2;
      if (bc > 16) {
        if (out + 2 > cap) return -1;
        o[out++] = (u8)bs; o[out++] = (u8)(bs >> 8);
        bs >>= 16; bc -= 16;
      }
    }
    {
      int count = norm[s++];
      const int max = (2 * threshold - 1) - remaining;
      remaining -= count < 0 ? -count : count;
      count++;
      if (count >= threshold) count += max;
      bs += (u32)count << bc;
      bc += nbits;
      bc -= (count < max);
      prev0 = (count == 1);
      while (remaining < threshold) { nbits--; threshold >>= 1; }
    }
    if (bc > 16) {
      if (out + 2 > cap) return -1;
      o[out++] = (u8)bs; o[out++] = (u8)(bs >> 8);
      bs >>= 16; bc -= 16;
    }
  }
  if (remaining != 1) return -1;
  while (bc > 0) { if (out >= cap) return -1; o[out++] = (u8)bs; bs >>= 8; bc -= 8; }
  return out;
}

/* FSE_buildCTable: the symbol spread is the decoder's (zs_fse_build) */
DEV void ze_build_ct(ZeCT& ct, const short* norm, int nsym, int log, u8* tsym) {
  const int size = 1 << log, mask = size - 1;
  int high = size - 1;
  u16 cum[65];
  cum[0] = 0;
  for (int u = 1; u <= nsym; u++) {
    if (norm[u - 1] == -1) { cum[u] = (u16)(cum[u - 1] + 1); tsym[high--] = (u8)(u - 1); }
    else cum[u] = (u16)(cum[u - 1] + (norm[u - 1] > 0 ? norm[u - 1] : 0));
  }
  const int step = (size >> 1) + (size >> 3) + 3;
  int pos = 0;
  for (int s = 0; s < nsym; s++)
    for (int i = 0; i < norm[s]; i++) {
      tsym[pos] = (u8)s;
      do pos = (pos + step) & mask; while (pos > high);
    }
  for (int u = 0; u < size; u++) { const int s = tsym[u]; ct.st[cum[s]++] = (u16)(size + u); }
  int total = 0;
  for (int s = 0; s < nsym; s++) {
    const int nv = norm[s];
    if (nv == 0) { ct.dnb[s] = ((u32)(log + 1) << 16) - (u32)size; ct.dfs[s] = 0; }
    else if (nv == -1 || nv == 1) { ct.dnb[s] = ((u32)log << 16) - (u32)size; ct.dfs[s] = total - 1; total++; }
    else {
      const int mbo = log - ze_hb((u32)(nv - 1));
      const u32 msp = (u32)nv << mbo;
      ct.dnb[s] = ((u32)mbo << 16) - msp;
      ct.dfs[s] = total - nv;
      total += nv;
    }
  }
  ct.log = log;
}
DEV u32 ze_fse_init(const ZeCT& ct, int s) {
  const u32 nbo = (ct.dnb[s] + (1u << 15)) >> 16;
  const u32 val = (nbo << 16) - ct.dnb[s];
  return ct.st[(int)(val >> nbo) + ct.dfs[s]];
}
DEV void ze_fse_enc(ZeBW& w, const ZeCT& ct, u32& state, int s) {
  const u32 nbo = (state + ct.dnb[s]) >> 16;
  zbw_add(w, state, (int)nbo);
  state = ct.st[(int)(state >> nbo) + ct.dfs[s]];
}

/* cost in 1/256 bits of coding `cnt` with normalised counts `norm` of table log `log`; -1: a symbol has no slot */
DEV long long ze_cost(const u32* cnt, int nsym, const short* norm, int nnorm, int log) {
  long long c = 0;
  for (int s = 0; s < nsym; s++) {
    if (!cnt[s]) continue;
    if (s >= nnorm || norm[s] == 0) return -1;
    const int nv = norm[s] < 0 ? 1 : norm[s];
    c += (long long)cnt[s] * ((log << 8) - ze_log2fix((u32)nv));
  }
  return c;
}

/* ---- length-limited Huffman code lengths, shared with the DEFLATE encoder (dev_deflate.cuh) ----
 * hist[0, nsym) -> len[0, nsym), every length <= maxlen and the code complete (Kraft sum exactly 1).  Scratch: leaf[nsym]
 * (the present symbols by ascending count, then symbol), nc / par[2 nsym].  Returns the number of present symbols; when
 * that is below 2 nothing is written to len. */
DEV int huf_limited_lengths(const u32* hist, const int nsym, const int maxlen, u16* leaf, u32* nc, u16* par, u8* len) {
  int n = 0;
  for (int s = 0; s < nsym; s++) if (hist[s]) leaf[n++] = (u16)s;
  if (n < 2) return n;
  for (int i = 1; i < n; i++) {                     /* by count, then symbol: ascending */
    const u16 x = leaf[i];
    int j = i - 1;
    while (j >= 0 && hist[leaf[j]] > hist[x]) { leaf[j + 1] = leaf[j]; j--; }
    leaf[j + 1] = x;
  }
  /* two-queue Huffman: leaves 0..n-1, internal nodes n..2n-2 (created in non-decreasing weight order) */
  for (int i = 0; i < n; i++) nc[i] = hist[leaf[i]];
  int li = 0, ni = n, nn = n;
  for (int k = 0; k < n - 1; k++) {
    int pick[2];
    for (int t = 0; t < 2; t++) {
      if (li < n && (ni >= nn || nc[li] <= nc[ni])) pick[t] = li++;
      else pick[t] = ni++;
    }
    nc[nn] = nc[pick[0]] + nc[pick[1]];
    par[pick[0]] = (u16)nn; par[pick[1]] = (u16)nn;
    nn++;
  }
  /* depths, root (nn-1) first: reuse nc[] for them */
  nc[nn - 1] = 0;
  for (int k = nn - 2; k >= 0; k--) nc[k] = nc[par[k]] + 1;
  for (int s = 0; s < nsym; s++) len[s] = 0;
  int kraft = 0;                                     /* sum of 2^(maxlen - len) */
  for (int i = 0; i < n; i++) {
    int l = (int)nc[i];
    if (l > maxlen) l = maxlen;
    len[leaf[i]] = (u8)l;
    kraft += 1 << (maxlen - l);
  }
  while (kraft > (1 << maxlen)) {                    /* too many codes after the clamp: lengthen the rarest */
    for (int i = 0; i < n && kraft > (1 << maxlen); i++) {
      const int s = leaf[i];
      if (len[s] < maxlen) { kraft -= 1 << (maxlen - 1 - len[s]); len[s]++; }
    }
  }
  while (kraft < (1 << maxlen)) {                    /* room left: shorten the most frequent that fit */
    for (int i = n - 1; i >= 0 && kraft < (1 << maxlen); i--) {
      const int s = leaf[i];
      const int add = 1 << (maxlen - len[s]);
      if (len[s] > 1 && add <= (1 << maxlen) - kraft) { kraft += add; len[s]--; }
    }
  }
  return n;
}

/* ---- Huffman code lengths <= 11 for the present literals; returns the longest code (0: fewer than two symbols) ---- */
DEV int ze_huf_lengths(ZeSm& S) {
  const int n = huf_limited_lengths(S.hist, 256, ZS_HUFLOG, S.leaf, S.nc, S.par, S.hlen);
  if (n < 2) return 0;
  int maxb = 0;
  for (int i = 0; i < n; i++) if (S.hlen[S.leaf[i]] > maxb) maxb = S.hlen[S.leaf[i]];
  /* canonical codes in the decoder's order (zs_huf_table): longer codes first, within a length by symbol */
  int start[ZS_HUFLOG + 2], at = 0;
  int rank[ZS_HUFLOG + 2];
  for (int wt = 0; wt <= ZS_HUFLOG + 1; wt++) rank[wt] = 0;
  for (int s = 0; s < 256; s++) if (S.hlen[s]) rank[maxb + 1 - S.hlen[s]]++;
  for (int wt = 1; wt <= maxb; wt++) { start[wt] = at; at += rank[wt] << (wt - 1); }
  for (int s = 0; s < 256; s++) {
    if (!S.hlen[s]) { S.w[s] = 0; continue; }
    const int wt = maxb + 1 - S.hlen[s];
    S.w[s] = (u8)wt;
    S.hcode[s] = (u16)(start[wt] >> (wt - 1));
    start[wt] += 1 << (wt - 1);
  }
  return maxb;
}

/* Huffman tree description (RFC 8878 4.2.1.1): FSE-coded weights when that is smaller, else 4-bit weights.
 * Returns bytes, 0 when neither form can describe the table. */
DEV int ze_huf_desc(ZeSm& S, int last, u8* o, int cap) {
  const int nw = last;                               /* weights of symbols 0 .. last-1; last's is implied */
  int best = 0;
  if (nw <= 128 && 1 + (nw + 1) / 2 <= cap) best = 1 + (nw + 1) / 2;
  /* FSE-coded (HUF_compressWeights): two interleaved states, table log <= 6 */
  u32 wc[13];
  for (int i = 0; i < 13; i++) wc[i] = 0;
  int maxw = 0;
  u32 mc = 0;
  for (int i = 0; i < nw; i++) { wc[S.w[i]]++; if (S.w[i] > maxw) maxw = S.w[i]; }
  for (int i = 0; i <= maxw; i++) if (wc[i] > mc) mc = wc[i];
  if (nw >= 2 && mc != (u32)nw && mc > 1 && cap >= 128) {
    const int log = ze_table_log(6, (u32)nw, maxw);
    short* norm = S.norm[3];
    ze_normalize(wc, maxw + 1, (u32)nw, log, norm);
    const int h = ze_write_ncount(o + 1, 127, norm, maxw + 1, log);
    if (h > 0) {
      ze_build_ct(S.wt, norm, maxw + 1, log, S.tsym);
      ZeBW bw;
      zbw_init(bw, o + 1 + h, 127 - h);
      u32 st[2];
      st[(nw - 1) & 1] = ze_fse_init(S.wt, S.w[nw - 1]);
      st[(nw - 2) & 1] = ze_fse_init(S.wt, S.w[nw - 2]);
      for (int i = nw - 3; i >= 0; i--) ze_fse_enc(bw, S.wt, st[i & 1], S.w[i]);
      zbw_add(bw, st[1], log);
      zbw_add(bw, st[0], log);
      const int b = zbw_close(bw);
      if (!bw.over && h + b < 128 && (best == 0 || 1 + h + b < best)) { o[0] = (u8)(h + b); return 1 + h + b; }
    }
  }
  if (!best) return 0;
  o[0] = (u8)(127 + nw);
  for (int i = 0; i < nw; i += 2) o[1 + i / 2] = (u8)((S.w[i] << 4) | (i + 1 < nw ? S.w[i + 1] : 0));
  return best;
}

/* one Huffman stream: literals lit[a, b) last first, then the end mark */
DEV int ze_huf_stream(const ZeSm& S, const u8* lit, int a, int b, u8* o, int cap) {
  ZeBW bw;
  zbw_init(bw, o, cap);
  for (int i = b - 1; i >= a; i--) { const int s = lit[i]; zbw_add(bw, S.hcode[s], S.hlen[s]); }
  const int r = zbw_close(bw);
  return bw.over ? -1 : r;
}

/* Literals section of a block (RFC 8878 3.1.1.3.1) for lit[0, nlit); histogram in S.hist.  Returns bytes or -1. */
DEV int ze_literals(ZeSm& S, const u8* lit, int nlit, u8* o, int cap) {
  int maxs = 0, last = 0;
  for (int s = 0; s < 256; s++) if (S.hist[s]) { last = s; if (S.hist[s] > S.hist[maxs]) maxs = s; }
  const int rawh = nlit < 32 ? 1 : (nlit < 4096 ? 2 : 3);
  if (nlit > 0 && S.hist[maxs] == (u32)nlit && nlit > 2) {           /* RLE */
    if (rawh + 1 > cap) return -1;
    const u32 h = 1u | (rawh == 1 ? ((u32)nlit << 3) : (rawh == 2 ? (1u << 2) | ((u32)nlit << 4) : (3u << 2) | ((u32)nlit << 4)));
    for (int i = 0; i < rawh; i++) o[i] = (u8)(h >> (8 * i));
    o[rawh] = lit[0];
    return rawh + 1;
  }
  if (nlit >= 64) {
    const int maxb = ze_huf_lengths(S);
    if (maxb > 0) {
      const bool one = nlit < 1024;
      const int seg = (nlit + 3) / 4;
      int sb[4] = {0, 0, 0, 0};                    /* exact bytes of each stream */
      {
        long long bits[4] = {0, 0, 0, 0};
        for (int i = 0; i < nlit; i++) bits[one ? 0 : i / seg] += S.hlen[lit[i]];
        for (int k = 0; k < (one ? 1 : 4); k++) sb[k] = (int)((bits[k] + 1 + 7) >> 3);
      }
      u8 desc[140];
      const int dn = ze_huf_desc(S, last, desc, 140);
      if (dn > 0) {
        const int comp = dn + (one ? sb[0] : 6 + sb[0] + sb[1] + sb[2] + sb[3]);
        const int sf = one ? 0 : ((nlit < 16384 && comp < 16384) ? 2 : 3);
        const int hh = sf < 2 ? 3 : sf + 2;
        if (comp < 16384 * 16 && hh + comp < rawh + nlit && !(one && comp >= 1024) && hh + comp <= cap) {
          const u64 h = 2u | ((u64)sf << 2) | ((u64)nlit << 4) | ((u64)comp << (sf < 2 ? 14 : (sf == 2 ? 18 : 22)));
          for (int i = 0; i < hh; i++) o[i] = (u8)(h >> (8 * i));
          int p = hh;
          for (int i = 0; i < dn; i++) o[p + i] = desc[i];
          p += dn;
          if (one) {
            if (ze_huf_stream(S, lit, 0, nlit, o + p, sb[0]) != sb[0]) return -1;
            p += sb[0];
          } else {
            o[p] = (u8)sb[0]; o[p + 1] = (u8)(sb[0] >> 8); o[p + 2] = (u8)sb[1]; o[p + 3] = (u8)(sb[1] >> 8);
            o[p + 4] = (u8)sb[2]; o[p + 5] = (u8)(sb[2] >> 8);
            p += 6;
            for (int k = 0; k < 4; k++) {
              const int a = k * seg, b = k < 3 ? a + seg : nlit;
              if (ze_huf_stream(S, lit, a, b, o + p, sb[k]) != sb[k]) return -1;
              p += sb[k];
            }
          }
          return p;
        }
      }
    }
  }
  if (rawh + nlit > cap) return -1;                                  /* raw */
  const u32 h = rawh == 1 ? ((u32)nlit << 3) : (rawh == 2 ? (1u << 2) | ((u32)nlit << 4) : (3u << 2) | ((u32)nlit << 4));
  for (int i = 0; i < rawh; i++) o[i] = (u8)(h >> (8 * i));
  for (int i = 0; i < nlit; i++) o[rawh + i] = lit[i];
  return rawh + nlit;
}

/* a stitched sequence: ll | ofv low 14 bits << 18, ml | ofv >> 14 << 18 (ll, ml < 2^18, ofv < 2^17) */
DEV void ze_seq_get(const uint2* q, int i, u32& ll, u32& ml, u32& ofv) {
  const uint2 x = q[i];
  ll = x.x & 0x3ffffu; ml = x.y & 0x3ffffu; ofv = (x.x >> 18) | ((x.y >> 18) << 14);
}

/* Sequences section for q[0, ns) (RFC 8878 3.1.1.3.2).  Returns bytes or -1. */
DEV int ze_sequences(ZeSm& S, const uint2* q, int ns, u8* o, int cap) {
  int p = 0;
  if (cap < 4) return -1;
  if (ns < 128) o[p++] = (u8)ns;
  else if (ns < 0x7f00) { o[p++] = (u8)((ns >> 8) + 128); o[p++] = (u8)ns; }
  else { o[p++] = 255; o[p++] = (u8)(ns - 0x7f00); o[p++] = (u8)((ns - 0x7f00) >> 8); }
  if (ns == 0) return p;
  const int nsym[3] = {36, 32, 53}, maxlog[3] = {9, 8, 9}, dlog[3] = {6, 5, 6}, dn[3] = {36, 29, 53};
  const short* dnorm[3] = {k_zs_ll_norm, k_zs_of_norm, k_zs_ml_norm};
  for (int t = 0; t < 3; t++) for (int s = 0; s < 64; s++) S.cnt[t][s] = 0;
  for (int i = 0; i < ns; i++) {
    u32 ll, ml, ofv;
    ze_seq_get(q, i, ll, ml, ofv);
    S.cnt[0][ze_llcode(ll)]++; S.cnt[1][ze_hb(ofv)]++; S.cnt[2][ze_mlcode(ml)]++;
  }
  int mode[3];
  const int mp = p++;
  for (int t = 0; t < 3; t++) {
    int maxs = 0, nz = 0, one = 0;
    for (int s = 0; s < nsym[t]; s++) if (S.cnt[t][s]) { maxs = s; nz++; one = s; }
    long long best = -1;
    int bm = 0;
    /* predefined */
    const long long cp = ze_cost(S.cnt[t], nsym[t], dnorm[t], dn[t], dlog[t]);
    if (cp >= 0) { best = cp; bm = 0; }
    if (nz == 1 && (best < 0 || 8 * 256 < best)) { best = 8 * 256; bm = 1; }
    /* FSE_Compressed */
    u8 hdr[128];
    int hn = -1, flog = 0;
    if (nz > 1) {
      flog = ze_table_log(maxlog[t], (u32)ns, maxs);
      ze_normalize(S.cnt[t], maxs + 1, (u32)ns, flog, S.norm[t]);
      hn = ze_write_ncount(hdr, 128, S.norm[t], maxs + 1, flog);
      if (hn > 0) {
        const long long cf = ze_cost(S.cnt[t], nsym[t], S.norm[t], maxs + 1, flog) + (long long)hn * 8 * 256;
        if (best < 0 || cf < best) { best = cf; bm = 2; }
      }
    }
    if (best < 0) return -1;
    mode[t] = bm;
    if (bm == 0) ze_build_ct(S.ct[t], dnorm[t], dn[t], dlog[t], S.tsym);
    else if (bm == 1) { if (p + 1 > cap) return -1; o[p++] = (u8)one; }
    else {
      if (p + hn > cap) return -1;
      for (int i = 0; i < hn; i++) o[p + i] = hdr[i];
      p += hn;
      ze_build_ct(S.ct[t], S.norm[t], maxs + 1, flog, S.tsym);
    }
  }
  o[mp] = (u8)((mode[0] << 6) | (mode[1] << 4) | (mode[2] << 2));
  /* the bitstream: last sequence first (ZSTD_encodeSequences) */
  ZeBW bw;
  zbw_init(bw, o + p, cap - p);
  u32 sll = 0, sof = 0, sml = 0;
  {
    u32 ll, ml, ofv;
    ze_seq_get(q, ns - 1, ll, ml, ofv);
    const int lc = ze_llcode(ll), oc = ze_hb(ofv), mc = ze_mlcode(ml);
    if (mode[2] != 1) sml = ze_fse_init(S.ct[2], mc);
    if (mode[1] != 1) sof = ze_fse_init(S.ct[1], oc);
    if (mode[0] != 1) sll = ze_fse_init(S.ct[0], lc);
    zbw_add(bw, ll - k_zs_ll_base[lc], k_zs_ll_bits[lc]);
    zbw_add(bw, ml - k_zs_ml_base[mc], k_zs_ml_bits[mc]);
    zbw_add(bw, ofv - (1u << oc), oc);
  }
  for (int i = ns - 2; i >= 0; i--) {
    u32 ll, ml, ofv;
    ze_seq_get(q, i, ll, ml, ofv);
    const int lc = ze_llcode(ll), oc = ze_hb(ofv), mc = ze_mlcode(ml);
    if (mode[1] != 1) ze_fse_enc(bw, S.ct[1], sof, oc);
    if (mode[2] != 1) ze_fse_enc(bw, S.ct[2], sml, mc);
    if (mode[0] != 1) ze_fse_enc(bw, S.ct[0], sll, lc);
    zbw_add(bw, ll - k_zs_ll_base[lc], k_zs_ll_bits[lc]);
    zbw_add(bw, ml - k_zs_ml_base[mc], k_zs_ml_bits[mc]);
    zbw_add(bw, ofv - (1u << oc), oc);
    if (bw.over) return -1;
  }
  if (mode[2] != 1) zbw_add(bw, sml, S.ct[2].log);
  if (mode[1] != 1) zbw_add(bw, sof, S.ct[1].log);
  if (mode[0] != 1) zbw_add(bw, sll, S.ct[0].log);
  const int b = zbw_close(bw);
  if (bw.over) return -1;
  return p + b;
}

/* Runs on ONE lane: the frame of stream s[0, n) into out[0, n) (records rec / cnt per segment, scratch = the stream's
 * 2n bytes of prev[]).  Returns the frame size, or n when the frame would not be smaller than the stream. */
DEV int zse_frame_serial(ZeSm& S, const u8* __restrict__ s, const int n, const u32* __restrict__ rec, const u32* __restrict__ cnt,
                         u8* scratch, u8* out) {
  if (n < 16) return n;
  const uintptr_t sb = ((uintptr_t)scratch + 7) & ~(uintptr_t)7;
  uint2* q = (uint2*)sb;
  const u8* send = scratch + 2 * (long long)n;
  const int qcap = (int)(((uintptr_t)send - sb) / 8);
  /* frame header: magic, single segment with the content size, no checksum, no dictionary */
  int op = 0;
  out[0] = 0x28; out[1] = 0xB5; out[2] = 0x2F; out[3] = 0xFD;
  if (n < 256) { out[4] = 0x20; out[5] = (u8)n; op = 6; }
  else if (n < 65536 + 256) { out[4] = 0x60; out[5] = (u8)(n - 256); out[6] = (u8)((n - 256) >> 8); op = 7; }
  else { out[4] = 0xA0; st_u32_bytes(out + 5, (u32)n); op = 9; }
  u32 r1 = 1, r2 = 4, r3 = 8;
  const int nseg = (n + FAST_SEG - 1) / FAST_SEG;
  for (int k0 = 0; k0 < nseg; k0 += ZE_BLOCK_SEGS) {
    const int k1 = k0 + ZE_BLOCK_SEGS < nseg ? k0 + ZE_BLOCK_SEGS : nseg;
    const int bpos = k0 * FAST_SEG, bend = k1 * FAST_SEG < n ? k1 * FAST_SEG : n, blen = bend - bpos;
    const bool lastb = k1 == nseg;
    if (op + 3 + 1 > n) return n;
    const u32 s1 = r1, s2 = r2, s3 = r3;
    /* stitch the block's records into sequences */
    int ns = 0, carry = 0, lme = -1, covered = 0;
    u32 loff = 0;
    bool ok = true;
    for (int k = k0; k < k1 && ok; k++) {
      const int c = (int)cnt[k], ss = k * FAST_SEG, se = ss + FAST_SEG < n ? ss + FAST_SEG : n;
      int p = ss;
      for (int r = 0; r < c; r++) {
        const u32 x = rec[(long long)k * ZE_SEG_RECS + r];
        const int ll = (int)(x & 0xffu), ml = (int)((x >> 8) & 0xffu) + 4;
        const u32 off = x >> 16;
        if (r == 0 && ll == 0 && carry == 0 && ns > 0 && lme == ss && loff == off) {    /* the match goes on */
          q[ns - 1].y += (u32)ml;
          p = ss + ml; lme = p; covered += ml;
          continue;
        }
        if (ns >= qcap) { ok = false; break; }
        const u32 tl = (u32)(carry + ll);
        u32 ofv;                                     /* repeat offsets (RFC 8878 3.1.2.5) */
        if (tl > 0) ofv = off == r1 ? 1u : (off == r2 ? 2u : (off == r3 ? 3u : off + 3u));
        else ofv = off == r2 ? 1u : (off == r3 ? 2u : (off == r1 - 1u ? 3u : off + 3u));
        if (ofv > 3) { r3 = r2; r2 = r1; r1 = off; }
        else {
          const u32 idx = ofv + (tl == 0 ? 1u : 0u);
          if (idx != 1) { if (idx != 2) r3 = r2; r2 = r1; r1 = off; }
        }
        q[ns++] = make_uint2(tl | ((ofv & 0x3fffu) << 18), (u32)ml | ((ofv >> 14) << 18));
        carry = 0;
        p = ss + ll + (p - ss) + ml;
        lme = p; loff = off; covered += ml;
      }
      carry += se - p;
    }
    /* gather the literals behind the sequences */
    u8* lit = (u8*)(q + ns);
    int nlit = 0, blk = -1;
    if (ok && (const u8*)lit + (blen - covered) <= send) {     /* 8 ns + literals <= 2 blen: a match covers >= 4 bytes */
      for (int i = 0; i < 256; i++) S.hist[i] = 0;
      int pos = bpos;
      for (int i = 0; i < ns; i++) {
        u32 ll, ml, ofv;
        ze_seq_get(q, i, ll, ml, ofv);
        for (u32 j = 0; j < ll; j++) { const u8 b = s[pos + j]; lit[nlit++] = b; S.hist[b]++; }
        pos += (int)(ll + ml);
      }
      for (; pos < bend; pos++) { const u8 b = s[pos]; lit[nlit++] = b; S.hist[b]++; }
      /* the compressed block, if it is smaller than the raw one */
      const int cap = (n - op - 3) < blen - 1 ? (n - op - 3) : blen - 1;
      if (cap > 2) {
        const int a = ze_literals(S, lit, nlit, out + op + 3, cap);
        if (a > 0) {
          const int b = ze_sequences(S, q, ns, out + op + 3 + a, cap - a);
          if (b > 0 && a + b < blen) blk = a + b;
        }
      }
    }
    if (blk > 0) {
      const u32 bh = (lastb ? 1u : 0u) | (2u << 1) | ((u32)blk << 3);
      out[op] = (u8)bh; out[op + 1] = (u8)(bh >> 8); out[op + 2] = (u8)(bh >> 16);
      op += 3 + blk;
    } else {                                         /* raw block: the decoder's repeat offsets stay as they were */
      r1 = s1; r2 = s2; r3 = s3;
      if (op + 3 + blen >= n) return n;
      const u32 bh = (lastb ? 1u : 0u) | ((u32)blen << 3);
      out[op] = (u8)bh; out[op + 1] = (u8)(bh >> 8); out[op + 2] = (u8)(bh >> 16);
      for (int i = 0; i < blen; i++) out[op + 3 + i] = s[bpos + i];
      op += 3 + blen;
    }
  }
  return op < n ? op : n;
}

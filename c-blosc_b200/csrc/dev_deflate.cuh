/*
 * dev_deflate.cuh -- the segment-parallel DEFLATE encoder (Blosc's "zlib" codec), sm_90a.
 *
 * It writes one zlib stream (RFC 1950 around RFC 1951 blocks) per stream of the chunk, the form compress2() writes
 * (reference blosc/blosc.c:472-483), that every inflate() and dev_inflate.cuh accept -- not compress2's bytes.  The
 * front half is the zstd encoder's (dev_zstdenc.cuh):
 *
 *   index_kernel  the prev[] hash chains (dev_lz4fast.cuh), unchanged.
 *   dparse        zparse with DEFLATE's window: every THREAD parses one segment of FAST_SEG bytes into sequence
 *                 records, offsets <= 32768.  A match lies inside its segment, so it is at most 256 bytes long.
 *   denc          one warp per stream.  Per DEFLATE block of up to 128 KiB (a whole number of segments):
 *                   - lane 0 stitches the records into items -- literal bytes, and matches cut into pieces of 3..258
 *                     bytes where a match continues across segments with the same offset -- in the stream's part of
 *                     prev[] (2 bytes per input byte, dead once the parse is done): u16 items from the front, the
 *                     u16 distances of the matches from the back (2 per literal + 4 per match <= 2 bytes per byte);
 *                   - the warp counts the 286 literal/length and 30 distance symbols;
 *                   - lane 0 builds the dynamic code (lengths <= 15, the code-length code <= 7, every code complete),
 *                     costs dynamic, fixed and stored blocks exactly and writes the header of the cheapest;
 *                   - the warp writes the symbols 32 at a time: each lane forms its item's bits (code and extra
 *                     bits, <= 48), an exclusive scan gives each lane its bit offset, the lanes OR their bits into a
 *                     shared-memory window that is flushed to the slot in whole words.
 *                 Stored blocks are copied by the warp.  The Adler-32 of the stream is computed by the warp.
 *   (scan / compact as for every codec: csizes[] -> bstarts -> the chunk)
 *
 * The block costs are exact, so a stream that would not be smaller than its input is known before its bytes are
 * written: nothing is written past the stream's slot.  Nothing depends on the order in which warps or lanes run, so
 * the device bytes equal the emulator's.
 */
#pragma once
#include "b2_args.h"
#include "dev_common.cuh"
#include "dev_lz4fast.cuh"
#include "dev_inflate.cuh"
#include "dev_zstdenc.cuh"

#define DZ_MAXD 32768                 /* DEFLATE's window */
#define DZ_WARPS 4
#define DZ_NL 286                     /* literal/length symbols that may occur (286, 287 never do) */
#define DZ_ND 30
#define DZ_DOFF 288                   /* distance lengths / codes follow the 288 literal/length ones */
#define DZ_WIN 128                    /* staging window: words */
#define DZ_WIN_BITS (DZ_WIN * 32 - 64)  /* bits the window may hold before a write (a write spans <= 3 words) */

struct DzSm {
  u32 win[DZ_WIN + 4];        /* the bits not yet in the slot; bit j of word w is stream bit 32 w + j past obyte */
  u32 lhist[DZ_NL];
  u32 dhist[DZ_ND];
  u32 clhist[19];
  u32 nc[2 * DZ_NL];          /* Huffman builder (huf_limited_lengths) */
  u16 par[2 * DZ_NL];
  u16 leaf[DZ_NL];
  u16 code[DZ_DOFF + DZ_ND];  /* bit-reversed codes: literal/length, then distance */
  u16 clcode[19];
  u16 clit[DZ_NL + DZ_ND];    /* the run-length coded code lengths: code-length symbol | extra bits << 5 */
  u8 len[DZ_DOFF + DZ_ND];    /* code lengths: literal/length, then distance */
  u8 cllen[19];
  int ni, nm, btype, wbits, obyte, raw;    /* lane 0 -> the warp */
  int nci, hdr;               /* dynamic header: code-length items; HLIT | HDIST << 9 | HCLEN << 14 */
};
#define DZ_SMEM_BYTES ((int)((sizeof(DzSm) + 15) & ~(size_t)15))

/* length 3..258 -> length code 0..28 (symbol 257 + code); distance 1..32768 -> distance code 0..29 (RFC 1951 3.2.5) */
DEV int dz_lcode(int l) {
  const int x = l - 3;
  if (x < 8) return x;
  if (x == 255) return 28;
  const int h = ze_hb((u32)x);
  return 4 * (h - 1) + ((x >> (h - 2)) & 3);
}
DEV int dz_dcode(int d) {
  const int x = d - 1;
  if (x < 4) return x;
  const int h = ze_hb((u32)x);
  return 2 * h + ((x >> (h - 1)) & 1);
}
DEV int dz_clext(int sym) { return sym < 16 ? 0 : (sym == 16 ? 2 : (sym == 17 ? 3 : 7)); }

/* canonical codes of len[0, n) (RFC 1951 3.2.2), bit-reversed: the stream is written LSB first */
DEV void dz_codes(const u8* len, int n, u16* code) {
  int cnt[16], next[16];
  for (int b = 0; b < 16; b++) cnt[b] = 0;
  for (int s = 0; s < n; s++) cnt[len[s]]++;
  cnt[0] = 0;
  int c = 0;
  for (int b = 1; b < 16; b++) { c = (c + cnt[b - 1]) << 1; next[b] = c; }
  for (int s = 0; s < n; s++)
    code[s] = len[s] ? (u16)(__brev((u32)next[len[s]]++) >> (32 - len[s])) : (u16)0;
}

/* move the window to out + ob: its whole words, or (all) every bit, the last byte padded with zeros.  Run by `nl`
 * lanes: 32 (the warp) or 1 (lane 0 alone). */
DEV void dz_flush(u32* win, u8* out, int& wb, int& ob, int lane, int nl, bool all) {
  const int nbytes = all ? (wb + 7) >> 3 : (wb >> 5) << 2;
  const int used = (wb + 31) >> 5, nw = nbytes >> 2;
  for (int i = lane; i < nbytes; i += nl) out[ob + i] = (u8)(win[i >> 2] >> (8 * (i & 3)));
  const u32 keep = all ? 0u : win[nw];
  if (nl > 1) __syncwarp();
  for (int i = lane; i < used; i += nl) win[i] = 0;
  if (nl > 1) __syncwarp();
  if (lane == 0) win[0] = keep;
  if (nl > 1) __syncwarp();
  ob += nbytes;
  wb = all ? 0 : wb & 31;
}

/* n <= 32 bits, lane 0 alone */
DEV void dz_put(u32* win, u8* out, int& wb, int& ob, u32 v, int n) {
  if (n == 0) return;
  if (wb + n > DZ_WIN_BITS) dz_flush(win, out, wb, ob, 0, 1, false);
  const u64 x = (u64)(n == 32 ? v : (v & ((1u << n) - 1u))) << (wb & 31);
  win[wb >> 5] |= (u32)x;
  win[(wb >> 5) + 1] |= (u32)(x >> 32);
  wb += n;
}

/* Lane 0: items of the block [bpos, bend) from the records of its segments [k0, k1).  Literal: the byte; match piece:
 * 256 + length - 3, its distance in dend[-1 - ordinal].  A match that the next segment continues with the same offset
 * is merged, and a merged run longer than 258 bytes is cut into pieces of 3..258 bytes (259 -> 256 + 3). */
DEV void dz_put_match(u16* item, u16* dend, int& ni, int& nm, int l, int d) {
  while (l > 258) {
    const int take = l - 258 >= 3 ? 258 : l - 3;
    item[ni++] = (u16)(256 + take - 3); dend[-1 - nm] = (u16)d; nm++;
    l -= take;
  }
  item[ni++] = (u16)(256 + l - 3); dend[-1 - nm] = (u16)d; nm++;
}
DEV void dz_stitch(const u8* __restrict__ s, const u32* __restrict__ rec, const u32* __restrict__ cnt,
                   const int k0, const int k1, const int bend, u16* item, u16* dend, int& ni, int& nm) {
  int from = k0 * FAST_SEG, pl = 0, pd = 0, pend = -1;     /* literals start at `from`; the pending match */
  ni = 0; nm = 0;
  for (int k = k0; k < k1; k++) {
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
      if (pl > 0) dz_put_match(item, dend, ni, nm, pl, pd);
      for (int j = from; j < ms; j++) item[ni++] = s[j];
      pl = ml; pd = off; pend = ms + ml; p = pend; from = pend;
    }
  }
  if (pl > 0) dz_put_match(item, dend, ni, nm, pl, pd);
  for (int j = from; j < bend; j++) item[ni++] = s[j];
}

/* Lane 0: the block's codes and its cheapest type, costed exactly; writes its header bits.  Returns the type (0 stored,
 * 1 fixed, 2 dynamic) and *bits, the block's size in bits starting at bit position `wb` of the window. */
DEV int dz_plan(DzSm& S, const int blen, const int wb, long long* bits) {
  S.lhist[256] = 1;
  long long extra = 0, fixed = 3, dyn = 3 + 5 + 5 + 4;
  for (int c = 0; c < 29; c++) extra += (long long)S.lhist[257 + c] * k_inf_lext[c];
  for (int c = 0; c < DZ_ND; c++) extra += (long long)S.dhist[c] * k_inf_dext[c];
  for (int s = 0; s < DZ_NL; s++) fixed += (long long)S.lhist[s] * (s < 144 ? 8 : (s < 256 ? 9 : (s < 280 ? 7 : 8)));
  for (int c = 0; c < DZ_ND; c++) fixed += (long long)S.dhist[c] * 5;
  fixed += extra;
  /* dynamic: literal/length lengths (EOB and at least one item: two symbols or more), distance lengths */
  for (int s = DZ_NL; s < DZ_DOFF; s++) S.len[s] = 0;
  huf_limited_lengths(S.lhist, DZ_NL, 15, S.leaf, S.nc, S.par, S.len);
  const int nd = huf_limited_lengths(S.dhist, DZ_ND, 15, S.leaf, S.nc, S.par, S.len + DZ_DOFF);
  if (nd < 2) {                     /* one distance code of length 1 (zlib accepts that incomplete code) */
    for (int c = 0; c < DZ_ND; c++) S.len[DZ_DOFF + c] = 0;
    S.len[DZ_DOFF + (nd == 1 ? S.leaf[0] : 0)] = 1;
  }
  int hlit = DZ_NL, hdist = DZ_ND;
  while (hlit > 257 && S.len[hlit - 1] == 0) hlit--;
  while (hdist > 1 && S.len[DZ_DOFF + hdist - 1] == 0) hdist--;
  /* run-length code the hlit + hdist lengths: 16 repeats the previous length 3..6 times, 17 / 18 code 3..10 / 11..138
   * zeros */
  for (int i = 0; i < 19; i++) S.clhist[i] = 0;
  int nci = 0;
  const int total = hlit + hdist;
  for (int i = 0; i < total;) {
    const int v = S.len[i < hlit ? i : DZ_DOFF + i - hlit];
    int run = 1;
    while (i + run < total && S.len[i + run < hlit ? i + run : DZ_DOFF + i + run - hlit] == v) run++;
    i += run;
    if (v == 0) {
      while (run >= 11) { const int r = run < 138 ? run : 138; S.clit[nci++] = (u16)(18 | (r - 11) << 5); S.clhist[18]++; run -= r; }
      if (run >= 3) { S.clit[nci++] = (u16)(17 | (run - 3) << 5); S.clhist[17]++; run = 0; }
    } else {
      S.clit[nci++] = (u16)v; S.clhist[v]++; run--;
      while (run >= 3) { const int r = run < 6 ? run : 6; S.clit[nci++] = (u16)(16 | (r - 3) << 5); S.clhist[16]++; run -= r; }
    }
    for (; run > 0; run--) { S.clit[nci++] = (u16)v; S.clhist[v]++; }
  }
  const int ncl = huf_limited_lengths(S.clhist, 19, 7, S.leaf, S.nc, S.par, S.cllen);
  if (ncl < 2) {                    /* the code-length code must be complete: a second 1-bit code */
    for (int i = 0; i < 19; i++) S.cllen[i] = 0;
    S.cllen[S.leaf[0]] = 1;
    S.cllen[S.leaf[0] == 0 ? 1 : 0] = 1;
  }
  int hclen = 19;
  while (hclen > 4 && S.cllen[k_inf_order[hclen - 1]] == 0) hclen--;
  dyn += 3 * hclen + extra;
  for (int i = 0; i < nci; i++) { const int sym = S.clit[i] & 31; dyn += S.cllen[sym] + dz_clext(sym); }
  for (int s = 0; s < DZ_NL; s++) dyn += (long long)S.lhist[s] * S.len[s];
  for (int c = 0; c < DZ_ND; c++) dyn += (long long)S.dhist[c] * S.len[DZ_DOFF + c];
  /* stored: pieces of <= 65535 bytes, each header padded to a byte boundary */
  long long stored = 0;
  int pos = wb & 7;
  for (int left = blen; left > 0;) {
    const int piece = left < 65535 ? left : 65535;
    stored += 3 + ((8 - ((pos + 3) & 7)) & 7) + 32 + 8LL * piece;
    pos = 0; left -= piece;
  }
  const int type = dyn < fixed ? 2 : 1;
  const long long huff = dyn < fixed ? dyn : fixed;
  if (huff >= stored) { *bits = stored; return 0; }
  *bits = huff;
  if (type == 1) {                  /* RFC 1951 3.2.6 */
    for (int s = 0; s < DZ_DOFF; s++) S.len[s] = (u8)(s < 144 ? 8 : (s < 256 ? 9 : (s < 280 ? 7 : 8)));
    for (int c = 0; c < DZ_ND; c++) S.len[DZ_DOFF + c] = 5;
  } else {
    S.nci = nci;
    S.hdr = hlit | hdist << 9 | hclen << 14;
  }
  dz_codes(S.len, DZ_DOFF, S.code);
  dz_codes(S.len + DZ_DOFF, DZ_ND, S.code + DZ_DOFF);
  dz_codes(S.cllen, 19, S.clcode);
  return type;
}

/* Lane 0: the dynamic header after BFINAL / BTYPE (RFC 1951 3.2.7), as dz_plan left it */
DEV void dz_dyn_header(DzSm& S, u8* out, int& wb, int& ob) {
  const int hlit = S.hdr & 511, hdist = (S.hdr >> 9) & 31, hclen = S.hdr >> 14, nci = S.nci;
  dz_put(S.win, out, wb, ob, (u32)(hlit - 257), 5);
  dz_put(S.win, out, wb, ob, (u32)(hdist - 1), 5);
  dz_put(S.win, out, wb, ob, (u32)(hclen - 4), 4);
  for (int i = 0; i < hclen; i++) dz_put(S.win, out, wb, ob, S.cllen[k_inf_order[i]], 3);
  for (int i = 0; i < nci; i++) {
    const int sym = S.clit[i] & 31;
    dz_put(S.win, out, wb, ob, S.clcode[sym], S.cllen[sym]);
    dz_put(S.win, out, wb, ob, (u32)(S.clit[i] >> 5), dz_clext(sym));
  }
}

/* Adler-32 of s[0, n) by the warp (the combine of dev_inflate.cuh's check) */
DEV u32 dz_adler32_warp(const u8* __restrict__ s, const int n) {
  const int lane = lane_id();
  const int per = (n + 31) / 32;
  const int lo = lane * per < n ? lane * per : n, hi = lo + per < n ? lo + per : n;
  u32 a = 0, b = 0;
  for (int k = lo; k < hi;) {
    const int run = hi - k < 3800 ? hi - k : 3800;          /* keeps b below 2^32 before the modulo */
    for (const int e = k + run; k < e; k++) { a += s[k]; b += a; }
    a %= 65521u; b %= 65521u;
  }
  u32 pa = a;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u32 t = __shfl_up_sync(FULLMASK, pa, d);
    if (lane >= d) pa = (pa + t) % 65521u;
  }
  const u32 before = (pa + 65521u - a) % 65521u;
  u32 tb = (b + (u32)(((u64)(before + 1u) * (u64)(hi - lo)) % 65521u)) % 65521u;
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) tb = (tb + __shfl_xor_sync(FULLMASK, tb, d)) % 65521u;
  const u32 ta = (__shfl_sync(FULLMASK, pa, 31) + 1u) % 65521u;
  return (tb << 16) | ta;
}

/* The whole warp: the zlib stream of s[0, n) into out[0, n) (records rec / cnt per segment, scratch = the stream's 2n
 * bytes of prev[]).  Returns its size, or n when it would not be smaller than the input. */
DEV int dz_stream(DzSm& S, const u8* __restrict__ s, const int n, const u32* __restrict__ rec, const u32* __restrict__ cnt,
                  u8* scratch, u8* out, const int flevel) {
  const int lane = lane_id();
  if (n < 16) return n;
  for (int i = lane; i < DZ_WIN + 4; i += 32) S.win[i] = 0;
  if (lane == 0) {                                 /* CMF: deflate, 32 KiB window; FLG: FLEVEL and FCHECK (deflate.c) */
    const u32 h = 0x7800u | ((u32)flevel << 6);
    out[0] = 0x78; out[1] = (u8)((h | (31u - h % 31u)) & 0xffu);
  }
  int wb = 0, ob = 2;
  const int nseg = (n + FAST_SEG - 1) / FAST_SEG;
  u16* item = (u16*)scratch;
  for (int k0 = 0; k0 < nseg; k0 += ZE_BLOCK_SEGS) {
    const int k1 = k0 + ZE_BLOCK_SEGS < nseg ? k0 + ZE_BLOCK_SEGS : nseg;
    const int bpos = k0 * FAST_SEG, bend = k1 * FAST_SEG < n ? k1 * FAST_SEG : n, blen = bend - bpos;
    const bool lastb = k1 == nseg;
    u16* dend = (u16*)(scratch + 2 * (long long)blen);
    __syncwarp();
    if (lane == 0) { int ni, nm; dz_stitch(s, rec, cnt, k0, k1, bend, item, dend, ni, nm); S.ni = ni; S.nm = nm; }
    for (int i = lane; i < DZ_NL; i += 32) S.lhist[i] = 0;
    if (lane < DZ_ND) S.dhist[lane] = 0;
    __syncwarp();
    const int ni = S.ni, nm = S.nm;
    for (int i = lane; i < ni; i += 32) {          /* the histograms, by the warp */
      const int it = item[i];
      atomicAdd(&S.lhist[it < 256 ? it : 257 + dz_lcode(it - 253)], 1u);
    }
    for (int j = lane; j < nm; j += 32) atomicAdd(&S.dhist[dz_dcode(dend[-1 - j])], 1u);
    __syncwarp();
    if (lane == 0) {
      long long bits = 0;
      const int type = dz_plan(S, blen, wb, &bits);
      S.raw = ((long long)ob * 8 + wb + bits + 7) / 8 + 4 >= n;   /* the stream would not be smaller */
      if (!S.raw && type > 0) {
        dz_put(S.win, out, wb, ob, lastb ? 1u : 0u, 1);
        dz_put(S.win, out, wb, ob, (u32)type, 2);
        if (type == 2) dz_dyn_header(S, out, wb, ob);
      }
      S.wbits = wb; S.obyte = ob; S.btype = type;
    }
    __syncwarp();
    if (S.raw) return n;
    const int type = S.btype;
    wb = S.wbits; ob = S.obyte;
    __syncwarp();
    if (type == 0) {                               /* stored pieces, copied by the warp */
      for (int pos = bpos; pos < bend;) {
        const int piece = bend - pos < 65535 ? bend - pos : 65535;
        if (lane == 0) {
          dz_put(S.win, out, wb, ob, (lastb && pos + piece == bend) ? 1u : 0u, 1);
          dz_put(S.win, out, wb, ob, 0u, 2);
          wb = (wb + 7) & ~7;
          dz_put(S.win, out, wb, ob, (u32)piece, 16);
          dz_put(S.win, out, wb, ob, (u32)piece ^ 0xffffu, 16);
        }
        wb = __shfl_sync(FULLMASK, wb, 0); ob = __shfl_sync(FULLMASK, ob, 0);
        __syncwarp();
        dz_flush(S.win, out, wb, ob, lane, 32, true);
        for (int j = lane; j < piece; j += 32) out[ob + j] = s[pos + j];
        ob += piece; pos += piece;
      }
      continue;
    }
    /* the symbols, 32 items at a time; item ni is the end-of-block code */
    int mb = 0;
    for (int t0 = 0; t0 <= ni; t0 += 32) {
      const int i = t0 + lane;
      const bool ism = i < ni && item[i] >= 256;
      const u32 mm = __ballot_sync(FULLMASK, ism);
      u64 v = 0;
      int nb = 0;
      if (i < ni) {
        const int it = item[i];
        if (it < 256) { v = S.code[it]; nb = S.len[it]; }
        else {
          const int l = it - 253, lc = dz_lcode(l), sym = 257 + lc;
          const int d = dend[-1 - (mb + __popc(mm & ((1u << lane) - 1u)))], dc = dz_dcode(d);
          v = S.code[sym]; nb = S.len[sym];
          v |= (u64)(l - k_inf_lens[lc]) << nb; nb += k_inf_lext[lc];
          v |= (u64)S.code[DZ_DOFF + dc] << nb; nb += S.len[DZ_DOFF + dc];
          v |= (u64)(d - k_inf_dists[dc]) << nb; nb += k_inf_dext[dc];
        }
      } else if (i == ni) { v = S.code[256]; nb = S.len[256]; }
      mb += __popc(mm);
      int off = nb;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(FULLMASK, off, d);
        if (lane >= d) off += t;
      }
      const int tot = __shfl_sync(FULLMASK, off, 31);
      off -= nb;
      if (wb + tot > DZ_WIN_BITS) dz_flush(S.win, out, wb, ob, lane, 32, false);
      if (nb) {
        const int p = wb + off, w = p >> 5, sh = p & 31;
        const u64 x = (v & 0xffffffffull) << sh, y = (v >> 32) << sh;
        if ((u32)x) atomicOr(&S.win[w], (u32)x);
        if ((u32)(x >> 32) | (u32)y) atomicOr(&S.win[w + 1], (u32)(x >> 32) | (u32)y);
        if ((u32)(y >> 32)) atomicOr(&S.win[w + 2], (u32)(y >> 32));
      }
      __syncwarp();
      wb += tot;
    }
  }
  dz_flush(S.win, out, wb, ob, lane, 32, true);
  const u32 ad = dz_adler32_warp(s, n);
  if (lane == 0) { out[ob] = (u8)(ad >> 24); out[ob + 1] = (u8)(ad >> 16); out[ob + 2] = (u8)(ad >> 8); out[ob + 3] = (u8)ad; }
  __syncwarp();
  return ob + 4;
}

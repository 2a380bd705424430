/*
 * dev_inflate.cuh -- zlib (RFC 1950) / DEFLATE (RFC 1951) decoder for one stream.
 *
 * SURVEY.md section 8 row (f4): chunks written with Blosc's "zlib" codec hold one zlib stream
 * per split (reference blosc/blosc.c:485-497 zlib_wrap_decompress -> uncompress()).  This is
 * a decode-only companion of the LZ4 / BloscLZ decoders so that such chunks (5 of the
 * compat .cdata goldens) decode on the GPU; the encoder side stays out of scope.
 *
 * DEFLATE's entropy coding is bit-serial, so one lane of the warp walks the stream (canonical
 * Huffman decoding by code length, the textbook method of RFC 1951 section 3.2.2) while the
 * other 2047 streams of a chunk run in other warps; the warp joins in for long LZ77 copies,
 * stored blocks and the Adler-32 check.  Accept / reject rules follow zlib's inflate():
 * bad header, reserved block type, stored-length mismatch, over-subscribed or incomplete code
 * sets (a single 1-bit code is allowed), missing end-of-block code, distances before the start
 * of the output, output overrun and a wrong Adler-32 all fail.  tests/test_zlib_decode_edges.py
 * reaches every reject site on hand-written streams and holds each verdict to Python's zlib.
 */
#pragma once
#include "dev_common.cuh"

#ifdef SIMT_EMU
static int g_inf_fail_line = 0;              /* emulator builds remember the first check that rejected the stream */
#define INF_FAIL (g_inf_fail_line = g_inf_fail_line ? g_inf_fail_line : __LINE__, -1)
#else
#define INF_FAIL (-1)
#endif

#define INF_MAXBITS 15
#define INF_MAXLCODES 286
#define INF_MAXDCODES 30
#define INF_FIXLCODES 288
/* shared-memory scratch of one stream (u16 units): two code tables + the code-length list */
#define INF_SMEM_U16 (16 + INF_FIXLCODES + 16 + INF_MAXDCODES + 2 + 320)
#define INF_SMEM_BYTES (INF_SMEM_U16 * 2)

static __device__ const u16 k_inf_lens[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
static __device__ const u8 k_inf_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static __device__ const u16 k_inf_dists[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static __device__ const u8 k_inf_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
static __device__ const u8 k_inf_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct InfState {
  const u8* in;
  int ip, iend;
  u64 bitbuf;
  int bitcnt;
  u8* out;
  int op, oend;
  bool bad;
};

/* make at least `need` bits available if the input still has them */
DEV void inf_fill(InfState& z, int need) {
  while (z.bitcnt < need && z.ip < z.iend) {
    z.bitbuf |= (u64)z.in[z.ip++] << z.bitcnt;
    z.bitcnt += 8;
  }
}
DEV u32 inf_bits(InfState& z, int n) {            /* n <= 16; sets bad when the input ends */
  if (n == 0) return 0;
  inf_fill(z, n);
  if (z.bitcnt < n) { z.bad = true; return 0; }
  const u32 v = (u32)(z.bitbuf & ((1ull << n) - 1ull));
  z.bitbuf >>= n; z.bitcnt -= n;
  return v;
}

/* Canonical Huffman table: count[len] codes of each length, symbols ordered by code.
 * Returns 0 for a complete code, > 0 for an incomplete one, < 0 when over-subscribed. */
DEV int inf_construct(u16* count, u16* symbol, const u16* length, int n) {
  u16 offs[INF_MAXBITS + 1];
  for (int len = 0; len <= INF_MAXBITS; len++) count[len] = 0;
  for (int s = 0; s < n; s++) count[length[s]]++;
  if (count[0] == n) return 0;                    /* no codes at all: complete, but decoding will fail */
  int left = 1;
  for (int len = 1; len <= INF_MAXBITS; len++) {
    left <<= 1;
    left -= count[len];
    if (left < 0) return left;
  }
  offs[1] = 0;
  for (int len = 1; len < INF_MAXBITS; len++) offs[len + 1] = (u16)(offs[len] + count[len]);
  for (int s = 0; s < n; s++)
    if (length[s] != 0) symbol[offs[length[s]]++] = (u16)s;
  return left;
}

/* one symbol; -1 on a code that does not exist or when the input ends */
DEV int inf_decode(InfState& z, const u16* count, const u16* symbol) {
  inf_fill(z, INF_MAXBITS);
  int code = 0, first = 0, index = 0;
  u64 buf = z.bitbuf;
  for (int len = 1; len <= INF_MAXBITS; len++) {
    if (len > z.bitcnt) return -1;
    code |= (int)(buf & 1u);
    buf >>= 1;
    const int cnt = count[len];
    if (code - cnt < first) {
      z.bitbuf = buf; z.bitcnt -= len;
      return symbol[index + (code - first)];
    }
    index += cnt; first += cnt;
    first <<= 1; code <<= 1;
  }
  return -1;
}

/* Runs on ONE lane.  Returns the number of bytes written, or -1. */
DEV int inf_deflate_serial(InfState& z, u16* sm) {
  u16* lcount = sm;
  u16* lsym = sm + 16;
  u16* dcount = sm + 16 + INF_FIXLCODES;
  u16* dsym = dcount + 16;
  u16* lengths = dsym + INF_MAXDCODES + 2;
  int last;
  do {
    last = (int)inf_bits(z, 1);
    const int type = (int)inf_bits(z, 2);
    if (z.bad) return INF_FAIL;                              /* no block header */
    if (type == 0) {                                         /* stored */
      z.ip -= z.bitcnt >> 3;                                 /* RFC 1951 3.2.4: skip to a byte boundary -- whole bytes that were */
      z.bitbuf = 0; z.bitcnt = 0;                            /* fetched ahead go back, the rest of the current byte is dropped */
      if (z.ip + 4 > z.iend) return INF_FAIL;
      const u32 len = (u32)z.in[z.ip] | ((u32)z.in[z.ip + 1] << 8);
      const u32 nlen = (u32)z.in[z.ip + 2] | ((u32)z.in[z.ip + 3] << 8);
      z.ip += 4;
      if (len != (~nlen & 0xffffu)) return INF_FAIL;
      if (z.ip + (int)len > z.iend || z.op + (int)len > z.oend) return INF_FAIL;
      for (u32 k = 0; k < len; k++) z.out[z.op + k] = z.in[z.ip + k];
      z.ip += (int)len; z.op += (int)len;
      continue;
    }
    if (type == 3) return INF_FAIL;
    if (type == 1) {                                         /* fixed codes, RFC 1951 3.2.6 */
      int s = 0;
      for (; s < 144; s++) lengths[s] = 8;
      for (; s < 256; s++) lengths[s] = 9;
      for (; s < 280; s++) lengths[s] = 7;
      for (; s < INF_FIXLCODES; s++) lengths[s] = 8;
      inf_construct(lcount, lsym, lengths, INF_FIXLCODES);
      for (s = 0; s < INF_MAXDCODES; s++) lengths[s] = 5;
      inf_construct(dcount, dsym, lengths, INF_MAXDCODES);
    } else {                                                 /* dynamic codes, RFC 1951 3.2.7 */
      const int nlen = (int)inf_bits(z, 5) + 257, ndist = (int)inf_bits(z, 5) + 1, ncode = (int)inf_bits(z, 4) + 4;
      if (z.bad || nlen > INF_MAXLCODES || ndist > INF_MAXDCODES) return INF_FAIL;
      int idx = 0;
      for (; idx < ncode; idx++) lengths[k_inf_order[idx]] = (u16)inf_bits(z, 3);
      for (; idx < 19; idx++) lengths[k_inf_order[idx]] = 0;
      if (z.bad) return INF_FAIL;                            /* code-length code cut */
      if (inf_construct(lcount, lsym, lengths, 19) != 0) return INF_FAIL;   /* the code-length code must be complete */
      idx = 0;
      while (idx < nlen + ndist) {
        int sym = inf_decode(z, lcount, lsym);
        if (sym < 0) return INF_FAIL;                        /* not a code-length code */
        if (sym < 16) lengths[idx++] = (u16)sym;
        else {
          int rep, val = 0;
          if (sym == 16) {
            if (idx == 0) return INF_FAIL;                         /* nothing to repeat */
            val = lengths[idx - 1];
            rep = 3 + (int)inf_bits(z, 2);
          } else if (sym == 17) rep = 3 + (int)inf_bits(z, 3);
          else rep = 11 + (int)inf_bits(z, 7);
          if (z.bad || idx + rep > nlen + ndist) return INF_FAIL;
          while (rep--) lengths[idx++] = (u16)val;
        }
      }
      if (lengths[256] == 0) return INF_FAIL;                      /* no end-of-block code */
      /* the distance lengths follow the literal/length ones; build dist first, it reads its slice */
      int err = inf_construct(dcount, dsym, lengths + nlen, ndist);
      if (err && (err < 0 || ndist != dcount[0] + dcount[1])) return INF_FAIL;
      err = inf_construct(lcount, lsym, lengths, nlen);
      if (err && (err < 0 || nlen != lcount[0] + lcount[1])) return INF_FAIL;
    }
    for (;;) {                                               /* the block's symbols */
      int sym = inf_decode(z, lcount, lsym);
      if (sym < 0) return INF_FAIL;                          /* not a literal/length code */
      if (sym < 256) {
        if (z.op >= z.oend) return INF_FAIL;
        z.out[z.op++] = (u8)sym;
        continue;
      }
      if (sym == 256) break;
      sym -= 257;
      if (sym >= 29) return INF_FAIL;
      const int len = k_inf_lens[sym] + (int)inf_bits(z, k_inf_lext[sym]);
      const int ds = inf_decode(z, dcount, dsym);
      if (ds < 0 || ds >= 30) return INF_FAIL;
      const int dist = k_inf_dists[ds] + (int)inf_bits(z, k_inf_dext[ds]);
      if (z.bad || dist > z.op || z.op + len > z.oend) return INF_FAIL;
      for (int k = 0; k < len; k++) z.out[z.op + k] = z.out[z.op + k - dist];
      z.op += len;
    }
  } while (!last);
  return z.op;
}

/* uncompress() of one zlib stream (zlib.h; reference blosc/blosc.c:485-497): returns the
 * number of bytes written or -1.  Uniform across the warp.  `smem` = INF_SMEM_BYTES of
 * warp-private shared memory. */
DEV int zlib_decode_warp(const u8* __restrict__ in, const int csize, u8* out, const int cap, void* smem) {
  const int lane = lane_id();
  int n = -1, endpos = 0;
  if (lane == 0) {
    do {
      if (csize < 2 + 4) { n = INF_FAIL; break; }            /* header + Adler-32 at least */
      const u32 cmf = in[0], flg = in[1];
      if ((cmf & 15u) != 8u || (cmf >> 4) > 7u) { n = INF_FAIL; break; }                    /* RFC 1950 2.2: deflate, window <= 32 KiB */
      if (((cmf << 8) | flg) % 31u != 0u) { n = INF_FAIL; break; }                         /* FCHECK */
      if (flg & 0x20u) { n = INF_FAIL; break; }                                            /* FDICT: no preset dictionary */
      InfState z;
      z.in = in; z.ip = 2; z.iend = csize; z.bitbuf = 0; z.bitcnt = 0; z.out = out; z.op = 0; z.oend = cap; z.bad = false;
      n = inf_deflate_serial(z, (u16*)smem);
      if (z.bad) n = INF_FAIL;                               /* the input ended inside the last symbol */
      endpos = z.ip - (z.bitcnt >> 3);                       /* whole unread bytes go back: the trailer is byte aligned */
    } while (0);
  }
  n = __shfl_sync(FULLMASK, n, 0);
  endpos = __shfl_sync(FULLMASK, endpos, 0);
  if (n < 0) return -1;                                      /* refused above, where the line was recorded */
  if (endpos + 4 > csize) return INF_FAIL;
  __syncwarp();
  /* Adler-32 of the output by the whole warp: lane l sums a contiguous slice (a = 1 + sum of bytes,
   * b = sum of the running a), slices are combined with b_total = sum(b_i + len_after_i * (a_i - ...)) */
  const int per = (n + 31) / 32;
  const int lo = lane * per < n ? lane * per : n, hi = lo + per < n ? lo + per : n;
  u32 a = 0, b = 0;                                          /* slice sums without the initial 1 */
  for (int k = lo; k < hi;) {
    int run = hi - k < 3800 ? hi - k : 3800;                 /* keeps b below 2^32 before the modulo */
    for (int e = k + run; k < e; k++) { a += out[k]; b += a; }
    a %= 65521u; b %= 65521u;
  }
  /* prefix of slice sums: the a of everything before this slice contributes (hi - lo) times to b */
  u32 pa = a;                                                /* inclusive scan of a */
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u32 t = __shfl_up_sync(FULLMASK, pa, d);
    if (lane >= d) pa = (pa + t) % 65521u;
  }
  const u32 before = (pa + 65521u - a) % 65521u;             /* sum of bytes before this slice */
  u32 tb = (b + (u32)(((u64)(before + 1u) * (u64)(hi - lo)) % 65521u)) % 65521u;   /* the initial a = 1 counts too */
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) tb = (tb + __shfl_xor_sync(FULLMASK, tb, d)) % 65521u;
  const u32 ta = (__shfl_sync(FULLMASK, pa, 31) + 1u) % 65521u;
  const u32 want = ((u32)in[endpos] << 24) | ((u32)in[endpos + 1] << 16) | ((u32)in[endpos + 2] << 8) | (u32)in[endpos + 3];
  if (((tb << 16) | ta) != want) return INF_FAIL;
  return n;
}

/*
 * dev_zstd.cuh -- Zstandard frame decoder (RFC 8878) for one stream.
 *
 * SURVEY.md section 8 row (f4): chunks written with Blosc's "zstd" codec hold one zstd frame
 * per block (never split, reference blosc/blosc.c:929-934; zstd_wrap_decompress ->
 * ZSTD_decompress(), :517-529).  Decode-only companion of dev_inflate.cuh so that such chunks
 * (3 of the compat .cdata goldens) decode on the GPU.  The encoder is dev_zstdenc.cuh, which shares the
 * code tables and predefined distributions below.
 *
 * The format is entropy coded with backward bitstreams (Huffman literals, FSE sequences), which
 * is serial work: one lane of the warp walks the frame while the chunk's other frames run in
 * other warps.  Literals are decoded on demand, straight into their place in the output, so no
 * per-block literal buffer is needed; the tables live in the warp's shared-memory scratch.
 * Everything zstd's own decoder checks on the way is checked here as well: magic, reserved
 * bits, sizes against the input, table descriptions, offsets beyond the decoded data, exact
 * consumption of every bitstream, declared content size and the optional XXH64 checksum.  Like
 * ZSTD_decompress, the input may hold several frames and skippable frames one after the other, and
 * a compressed block and its literals are limited by min(window size, 128 KiB).
 *
 * Verdict rule: never accept a frame that zstd 1.5.6's ZSTD_decompress rejects, never reject an
 * RFC 8878-valid frame that it accepts.  RFC-invalid frames that it accepts are refused here only for
 * the STRICT list of tests/test_zstd_decode_edges.py (each entry pinned by a test): Huffman codes of
 * 12 bits, raw / RLE blocks above 128 KiB, a compressed block that decodes to more than 128 KiB, and
 * a literal stream with bits left over (zstd's fast Huffman loops do not check it).
 */
#pragma once
#include "dev_common.cuh"

#ifdef SIMT_EMU
static int g_zs_fail_line = 0;               /* emulator builds remember the first check that rejected the frame */
#define ZS_FAIL (g_zs_fail_line = g_zs_fail_line ? g_zs_fail_line : __LINE__, -1)
#else
#define ZS_FAIL (-1)
#endif
#define ZS_HUFLOG 11
#define ZS_BLOCKMAX (128 * 1024)
struct ZsFse { u8 sym, nbits; u16 base; };

/* shared-memory layout of one stream's tables (bytes) */
#define ZS_OFF_HUF 0                                        /* u16[2048]: symbol | nbits << 8 */
#define ZS_OFF_LL (ZS_OFF_HUF + 2 * (1 << ZS_HUFLOG))       /* ZsFse[512] */
#define ZS_OFF_ML (ZS_OFF_LL + 4 * 512)
#define ZS_OFF_OF (ZS_OFF_ML + 4 * 512)                     /* ZsFse[256] */
#define ZS_OFF_WT (ZS_OFF_OF + 4 * 256)                     /* ZsFse[64]: Huffman-weight FSE table */
#define ZS_OFF_NORM (ZS_OFF_WT + 4 * 64)                    /* short[64] normalised counts */
#define ZS_OFF_NEXT (ZS_OFF_NORM + 2 * 64)                  /* u16[64] next-state counters */
#define ZS_OFF_WEIGHT (ZS_OFF_NEXT + 2 * 64)                /* u8[256] Huffman weights */
#define ZS_SMEM_BYTES (ZS_OFF_WEIGHT + 256)

static __device__ const u8 k_zs_ll_bits[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
static __device__ const u32 k_zs_ll_base[36] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
static __device__ const u8 k_zs_ml_bits[53] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
static __device__ const u32 k_zs_ml_base[53] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539};
static __device__ const short k_zs_ll_norm[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
static __device__ const short k_zs_ml_norm[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
static __device__ const short k_zs_of_norm[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};

DEV int zs_highbit(u32 v) { return 31 - __clz((int)v); }    /* v != 0 */

/* n <= 32 bits at bit position `pos` of a byte string (little-endian); positions below 0 read as 0 */
DEV u32 zs_bits_at(const u8* p, int pos, int n) {
  int up = 0;                                                /* bits below position 0: the result is shifted up by that many */
  if (pos < 0) { up = -pos; n += pos; pos = 0; }
  if (n <= 0) return 0;
  const int byte = pos >> 3, sh = pos & 7, nb = (sh + n + 7) >> 3;
  u64 v = 0;
  for (int k = 0; k < nb; k++) v |= (u64)p[byte + k] << (8 * k);
  return (u32)((v >> sh) & ((n == 32) ? 0xffffffffull : ((1ull << n) - 1ull))) << up;
}

/* backward bitstream over p[0, len): `pos` = number of still unread bits */
struct ZsBack { const u8* p; int pos; };
DEV bool zs_back_init(ZsBack& b, const u8* p, int len) {
  if (len <= 0 || p[len - 1] == 0) return false;
  b.p = p;
  b.pos = (len - 1) * 8 + zs_highbit(p[len - 1]);
  return true;
}
DEV u32 zs_back_read(ZsBack& b, int n) { b.pos -= n; return zs_bits_at(b.p, b.pos, n); }

/* FSE decoding table from normalised counts (RFC 8878 4.1.1) */
DEV void zs_fse_build(ZsFse* t, const short* norm, int nsym, int log, u16* next) {
  const int size = 1 << log;
  int high = size - 1;
  for (int s = 0; s < nsym; s++) {
    if (norm[s] == -1) { t[high--].sym = (u8)s; next[s] = 1; }
    else next[s] = (u16)norm[s];
  }
  const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
  int pos = 0;
  for (int s = 0; s < nsym; s++)
    for (int i = 0; i < norm[s]; i++) {
      t[pos].sym = (u8)s;
      do pos = (pos + step) & mask; while (pos > high);
    }
  for (int u = 0; u < size; u++) {
    const u32 ns = next[t[u].sym]++;
    const int nb = log - zs_highbit(ns);
    t[u].nbits = (u8)nb;
    t[u].base = (u16)((ns << nb) - size);
  }
}

/* FSE table description (RFC 8878 4.1.1): fills norm[0, *nsym) and *log; returns bytes used or -1 */
DEV int zs_fse_header(const u8* p, int len, short* norm, int maxsym, int maxlog, int* nsym, int* log) {
  if (len < 1) return ZS_FAIL;                                   /* no description */
  const int total = len * 8;
  int pos = 0;
  const int alog = 5 + (int)zs_bits_at(p, pos, 4);
  pos += 4;
  if (alog > maxlog) return ZS_FAIL;
  int remaining = 1 << alog, s = 0;
  while (remaining > 0 && s <= maxsym) {
    const int bits = zs_highbit((u32)(remaining + 1)) + 1;
    const int avail = total - pos;
    if (avail <= 0) return ZS_FAIL;
    u32 val = zs_bits_at(p, pos, bits < avail ? bits : avail);    /* bits past the end read as 0 */
    const u32 lower = (1u << (bits - 1)) - 1u, thresh = (1u << bits) - 1u - (u32)(remaining + 1);
    if ((val & lower) < thresh) { pos += bits - 1; val &= lower; }
    else { pos += bits; if (val > lower) val -= thresh; }
    if (pos > total) return ZS_FAIL;
    const int prob = (int)val - 1;
    remaining -= prob < 0 ? -prob : prob;
    norm[s++] = (short)prob;
    if (prob == 0) {
      for (;;) {
        if (pos + 2 > total) return ZS_FAIL;
        const int rep = (int)zs_bits_at(p, pos, 2);
        pos += 2;
        for (int i = 0; i < rep && s <= maxsym; i++) norm[s++] = 0;
        if (rep != 3) break;
      }
    }
  }
  if (remaining != 0 || s > maxsym + 1) return ZS_FAIL;
  *nsym = s; *log = alog;
  return (pos + 7) >> 3;
}

struct ZsLit {              /* literals of the current block, produced on demand */
  int type;                 /* 0 raw, 1 rle, 2 huffman */
  const u8* raw;            /* raw / rle source */
  int left;                 /* literals not yet delivered */
  ZsBack s[4];
  int quota[4], cur, nstreams, hlog;
};

DEV bool zs_lit_take(ZsLit& L, const u16* huf, u8* dst, int n) {
  if (n > L.left) return false;
  L.left -= n;
  if (L.type == 0) { for (int k = 0; k < n; k++) dst[k] = L.raw[k]; L.raw += n; return true; }
  if (L.type == 1) { const u8 v = L.raw[0]; for (int k = 0; k < n; k++) dst[k] = v; return true; }
  int k = 0;
  while (k < n) {
    while (L.quota[L.cur] == 0) { if (++L.cur >= L.nstreams) return false; }
    int m = n - k < L.quota[L.cur] ? n - k : L.quota[L.cur];
    ZsBack& b = L.s[L.cur];
    L.quota[L.cur] -= m;
    for (; m > 0; m--) {
      const u32 e = huf[zs_bits_at(b.p, b.pos - L.hlog, L.hlog)];
      b.pos -= (int)(e >> 8);
      dst[k++] = (u8)e;
    }
    if (b.pos < 0) return false;                             /* read past the start of the stream */
  }
  return true;
}

/* Huffman table from the tree description at p (RFC 8878 4.2.1); returns bytes used or -1 */
DEV int zs_huf_table(const u8* p, int len, u8* sm, int* hlog) {
  u16* huf = (u16*)(sm + ZS_OFF_HUF);
  u8* w = sm + ZS_OFF_WEIGHT;
  if (len < 1) return ZS_FAIL;                                   /* no tree description */
  const int hb = p[0];
  int n, used;
  if (hb >= 128) {                                           /* 4-bit weights */
    n = hb - 127;
    used = 1 + (n + 1) / 2;
    if (used > len) return ZS_FAIL;
    for (int i = 0; i < n; i++) w[i] = (i & 1) ? (p[1 + i / 2] & 15) : (p[1 + i / 2] >> 4);
  } else {                                                   /* FSE-compressed weights, two interleaved states */
    used = 1 + hb;
    if (hb == 0 || used > len) return ZS_FAIL;
    short* norm = (short*)(sm + ZS_OFF_NORM);
    int nsym, log;
    const int h = zs_fse_header(p + 1, hb, norm, 12, 6, &nsym, &log);
    if (h < 0 || h >= hb) return ZS_FAIL;
    ZsFse* t = (ZsFse*)(sm + ZS_OFF_WT);
    zs_fse_build(t, norm, nsym, log, (u16*)(sm + ZS_OFF_NEXT));
    ZsBack b;
    if (!zs_back_init(b, p + 1 + h, hb - h)) return ZS_FAIL;
    u32 s1 = zs_back_read(b, log), s2 = zs_back_read(b, log);
    if (b.pos < 0) return ZS_FAIL;
    n = 0;
    for (;;) {                                               /* at most 255 explicit weights */
      if (n >= 254) return ZS_FAIL;                          /* first state */
      w[n++] = t[s1].sym;
      s1 = t[s1].base + zs_back_read(b, t[s1].nbits);
      if (b.pos < 0) { w[n++] = t[s2].sym; break; }
      if (n >= 254) return ZS_FAIL;                          /* second state */
      w[n++] = t[s2].sym;
      s2 = t[s2].base + zs_back_read(b, t[s2].nbits);
      if (b.pos < 0) { w[n++] = t[s1].sym; break; }
    }
  }
  /* the last weight is implied: the weights' powers of two must add up to a power of two */
  u32 sum = 0;
  for (int i = 0; i < n; i++) { if (w[i] > ZS_HUFLOG) return ZS_FAIL; if (w[i]) sum += 1u << (w[i] - 1); }
  if (sum == 0) return ZS_FAIL;
  const int maxbits = zs_highbit(sum) + 1;
  if (maxbits > ZS_HUFLOG) return ZS_FAIL;
  const u32 rest = (1u << maxbits) - sum;
  if (rest & (rest - 1u)) return ZS_FAIL;                         /* not a power of two */
  w[n++] = (u8)(zs_highbit(rest) + 1);
  /* codes with more bits (smaller weight) come first; within a weight, symbols in natural order */
  int rank[ZS_HUFLOG + 2];
  for (int i = 0; i <= ZS_HUFLOG + 1; i++) rank[i] = 0;
  for (int i = 0; i < n; i++) rank[w[i]]++;
  if (rank[1] < 2 || (rank[1] & 1)) return ZS_FAIL;               /* at least two longest codes, in pairs */
  int start[ZS_HUFLOG + 2], at = 0;
  for (int wt = 1; wt <= maxbits; wt++) { start[wt] = at; at += rank[wt] << (wt - 1); }
  for (int i = 0; i < n; i++) {
    if (!w[i]) continue;
    const int span = 1 << (w[i] - 1);
    const u16 e = (u16)(i | ((maxbits + 1 - w[i]) << 8));
    for (int k = 0; k < span; k++) huf[start[w[i]] + k] = e;
    start[w[i]] += span;
  }
  *hlog = maxbits;
  return used;
}

/* One of the three sequence tables (RFC 8878 3.1.1.3.2.1); returns bytes used or -1 */
DEV int zs_seq_table(int mode, const u8* p, int len, ZsFse* t, int* log, bool* have, const short* dnorm, int dn, int dlog,
                     int maxsym, int maxlog, u8* sm) {
  u16* next = (u16*)(sm + ZS_OFF_NEXT);
  if (mode == 0) { zs_fse_build(t, dnorm, dn, dlog, next); *log = dlog; *have = true; return 0; }
  if (mode == 1) {
    if (len < 1 || p[0] > maxsym) return ZS_FAIL;
    t[0].sym = p[0]; t[0].nbits = 0; t[0].base = 0; *log = 0; *have = true;
    return 1;
  }
  if (mode == 2) {
    short* norm = (short*)(sm + ZS_OFF_NORM);
    int nsym, l;
    const int h = zs_fse_header(p, len, norm, maxsym, maxlog, &nsym, &l);
    if (h < 0) return ZS_FAIL;
    zs_fse_build(t, norm, nsym, l, next);
    *log = l; *have = true;
    return h;
  }
  return *have ? 0 : -1;                                      /* repeat: the previous table must exist */
}

DEV u64 zs_rotl64(u64 x, int r) { return (x << r) | (x >> (64 - r)); }
DEV u64 zs_rd64(const u8* p) { u64 v = 0; for (int i = 0; i < 8; i++) v |= (u64)p[i] << (8 * i); return v; }
DEV u64 zs_xxh64(const u8* p, int len) {                    /* XXH64, seed 0 */
  const u64 P1 = 11400714785074694791ull, P2 = 14029467366897019727ull, P3 = 1609587929392839161ull,
            P4 = 9650029242287828579ull, P5 = 2870177450012600261ull;
  const u8* end = p + len;
  u64 h;
  if (len >= 32) {
    u64 v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0ull - P1;
    do {
      v1 = zs_rotl64(v1 + zs_rd64(p) * P2, 31) * P1; p += 8;
      v2 = zs_rotl64(v2 + zs_rd64(p) * P2, 31) * P1; p += 8;
      v3 = zs_rotl64(v3 + zs_rd64(p) * P2, 31) * P1; p += 8;
      v4 = zs_rotl64(v4 + zs_rd64(p) * P2, 31) * P1; p += 8;
    } while (p + 32 <= end);
    h = zs_rotl64(v1, 1) + zs_rotl64(v2, 7) + zs_rotl64(v3, 12) + zs_rotl64(v4, 18);
    h = (h ^ (zs_rotl64(v1 * P2, 31) * P1)) * P1 + P4;
    h = (h ^ (zs_rotl64(v2 * P2, 31) * P1)) * P1 + P4;
    h = (h ^ (zs_rotl64(v3 * P2, 31) * P1)) * P1 + P4;
    h = (h ^ (zs_rotl64(v4 * P2, 31) * P1)) * P1 + P4;
  } else h = P5;
  h += (u64)len;
  while (p + 8 <= end) { h ^= zs_rotl64(zs_rd64(p) * P2, 31) * P1; h = zs_rotl64(h, 27) * P1 + P4; p += 8; }
  if (p + 4 <= end) { h ^= (u64)((u32)p[0] | ((u32)p[1] << 8) | ((u32)p[2] << 16) | ((u32)p[3] << 24)) * P1; h = zs_rotl64(h, 23) * P2 + P3; p += 4; }
  while (p < end) { h ^= (u64)(*p++) * P5; h = zs_rotl64(h, 11) * P1; }
  h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
  return h;
}

/* Runs on ONE lane: the frame at the start of in[0, csize).  Returns bytes written or -1, and the frame's size in *used. */
DEV int zs_frame_one(const u8* in, int csize, u8* out, int cap, u8* sm, int* used) {
  if (csize < 6) return ZS_FAIL;
  if (((u32)in[0] | ((u32)in[1] << 8) | ((u32)in[2] << 16) | ((u32)in[3] << 24)) != 0xFD2FB528u) return ZS_FAIL;
  const int fhd = in[4];
  const int fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, checksum = (fhd >> 2) & 1, did_flag = fhd & 3;
  if (fhd & 0x08) return ZS_FAIL;                                 /* reserved bit */
  int ip = 5;
  u32 window = ZS_BLOCKMAX;                                       /* min(window size, ZS_BLOCKMAX) */
  if (!single) {
    if (ip >= csize) return ZS_FAIL;
    if ((in[ip] >> 3) > 21) return ZS_FAIL;                       /* window above 2 GiB: more than ZSTD_decompress accepts (31 bits) */
    const int wexp = (in[ip] >> 3) + 10;
    if (wexp < 17) window = (1u << wexp) + ((1u << wexp) >> 3) * (in[ip] & 7u);   /* from 2^17 on, no block is limited by it */
    ip++;
  }
  const int did_bytes = did_flag == 3 ? 4 : did_flag;
  if (ip + did_bytes > csize) return ZS_FAIL;
  for (int i = 0; i < did_bytes; i++) if (in[ip + i]) return ZS_FAIL;   /* a dictionary is required: not available */
  ip += did_bytes;
  const int fcs_bytes = fcs_flag == 0 ? single : (1 << fcs_flag);
  if (ip + fcs_bytes > csize) return ZS_FAIL;
  u64 fcs = 0;
  for (int i = 0; i < fcs_bytes; i++) fcs |= (u64)in[ip + i] << (8 * i);
  if (fcs_bytes == 2) fcs += 256;
  ip += fcs_bytes;
  if (fcs_bytes && fcs > (u64)cap) return ZS_FAIL;
  if (single && fcs < (u64)window) window = (u32)fcs;             /* a single-segment frame's window is its content size */
  /* RFC 8878 Block_Maximum_Size: a compressed block and its literals stay within min(window, 128 KiB), as in
   * ZSTD_decompress.  Raw and RLE block sizes and a compressed block's output are held to 128 KiB only. */
  const int bmax = (int)window;

  u16* huf = (u16*)(sm + ZS_OFF_HUF);
  ZsFse* tll = (ZsFse*)(sm + ZS_OFF_LL);
  ZsFse* tml = (ZsFse*)(sm + ZS_OFF_ML);
  ZsFse* tof = (ZsFse*)(sm + ZS_OFF_OF);
  bool have_huf = false, have_ll = false, have_ml = false, have_of = false;
  int hlog = 0, ll_log = 0, ml_log = 0, of_log = 0;
  u32 rep1 = 1, rep2 = 4, rep3 = 8;
  int op = 0, last;
  do {
    if (ip + 3 > csize) return ZS_FAIL;
    const u32 bh = (u32)in[ip] | ((u32)in[ip + 1] << 8) | ((u32)in[ip + 2] << 16);
    ip += 3;
    last = (int)(bh & 1u);
    const int btype = (int)((bh >> 1) & 3u), bsize = (int)(bh >> 3);
    if (btype == 3) return ZS_FAIL;
    if (btype == 0) {                                        /* raw */
      if (bsize > ZS_BLOCKMAX || ip + bsize > csize || op + bsize > cap) return ZS_FAIL;
      for (int k = 0; k < bsize; k++) out[op + k] = in[ip + k];
      ip += bsize; op += bsize;
      continue;
    }
    if (btype == 1) {                                        /* RLE */
      if (bsize > ZS_BLOCKMAX || ip + 1 > csize || op + bsize > cap) return ZS_FAIL;
      const u8 v = in[ip++];
      for (int k = 0; k < bsize; k++) out[op + k] = v;
      op += bsize;
      continue;
    }
    if (bsize > bmax || bsize < 2 || ip + bsize > csize) return ZS_FAIL;   /* compressed block */
    const u8* b = in + ip;
    const int bend = bsize;
    ip += bsize;
    const int block_start = op;
    /* ---- literals section ---- */
    ZsLit L;
    int lp;                                                  /* position inside the block */
    {
      const int ltype = b[0] & 3, sf = (b[0] >> 2) & 3;
      int regen, comp = 0, hdr;
      if (ltype < 2) {
        if (sf == 0 || sf == 2) { hdr = 1; regen = b[0] >> 3; }
        else if (sf == 1) { hdr = 2; if (bend < 2) return ZS_FAIL; regen = (b[0] >> 4) | ((int)b[1] << 4); }
        else { hdr = 3; if (bend < 3) return ZS_FAIL; regen = (b[0] >> 4) | ((int)b[1] << 4) | ((int)b[2] << 12); }
      } else {
        if (bend < (sf < 2 ? 3 : sf + 2)) return ZS_FAIL;
        if (sf < 2) { hdr = 3; const u32 v = (u32)b[0] | ((u32)b[1] << 8) | ((u32)b[2] << 16); regen = (int)((v >> 4) & 0x3ffu); comp = (int)(v >> 14); }
        else if (sf == 2) { hdr = 4; const u32 v = (u32)b[0] | ((u32)b[1] << 8) | ((u32)b[2] << 16) | ((u32)b[3] << 24); regen = (int)((v >> 4) & 0x3fffu); comp = (int)(v >> 18); }
        else { hdr = 5; const u64 v = (u64)b[0] | ((u64)b[1] << 8) | ((u64)b[2] << 16) | ((u64)b[3] << 24) | ((u64)b[4] << 32); regen = (int)((v >> 4) & 0x3ffffu); comp = (int)(v >> 22); }
      }
      if (regen > bmax) return ZS_FAIL;
      L.left = regen; L.cur = 0;
      if (ltype == 0) { if (hdr + regen > bend) return ZS_FAIL; L.type = 0; L.raw = b + hdr; lp = hdr + regen; }
      else if (ltype == 1) { if (hdr + 1 > bend) return ZS_FAIL; L.type = 1; L.raw = b + hdr; lp = hdr + 1; }
      else {
        if (hdr + comp > bend) return ZS_FAIL;
        L.type = 2;
        const u8* q = b + hdr;
        int qlen = comp;
        if (ltype == 2) {
          const int used = zs_huf_table(q, qlen, sm, &hlog);
          if (used < 0) return ZS_FAIL;
          have_huf = true;
          q += used; qlen -= used;
        } else if (!have_huf) return ZS_FAIL;                     /* treeless block without a previous table */
        L.hlog = hlog;
        L.nstreams = (ltype >= 2 && sf == 0) ? 1 : 4;
        if (L.nstreams == 4 && regen < 6) return ZS_FAIL;         /* zstd refuses 4 streams for fewer than 6 literals */
        if (L.nstreams == 1) {
          if (!zs_back_init(L.s[0], q, qlen)) return ZS_FAIL;
          L.quota[0] = regen;
        } else {
          if (qlen < 6) return ZS_FAIL;
          const int l1 = q[0] | (q[1] << 8), l2 = q[2] | (q[3] << 8), l3 = q[4] | (q[5] << 8), l4 = qlen - 6 - l1 - l2 - l3;
          if (l4 < 1 || l1 < 1 || l2 < 1 || l3 < 1) return ZS_FAIL;
          const int seg = (regen + 3) / 4;
          if (regen < 3 * seg) return ZS_FAIL;                    /* the last stream's share would be negative */
          if (!zs_back_init(L.s[0], q + 6, l1) || !zs_back_init(L.s[1], q + 6 + l1, l2) ||
              !zs_back_init(L.s[2], q + 6 + l1 + l2, l3) || !zs_back_init(L.s[3], q + 6 + l1 + l2 + l3, l4)) return ZS_FAIL;
          L.quota[0] = L.quota[1] = L.quota[2] = seg; L.quota[3] = regen - 3 * seg;
        }
        lp = hdr + comp;
      }
    }
    /* ---- sequences section ---- */
    if (lp >= bend) return ZS_FAIL;                          /* no sequence count */
    int nseq = b[lp++];
    if (nseq >= 128) {
      if (nseq == 255) { if (lp + 2 > bend) return ZS_FAIL; nseq = (b[lp] | (b[lp + 1] << 8)) + 0x7F00; lp += 2; }
      else { if (lp + 1 > bend) return ZS_FAIL; nseq = ((nseq - 128) << 8) + b[lp++]; }
    }
    if (nseq > 0) {
      if (lp >= bend) return ZS_FAIL;                        /* no modes byte */
      const int modes = b[lp++];
      if (modes & 3) return ZS_FAIL;
      int u = zs_seq_table(modes >> 6, b + lp, bend - lp, tll, &ll_log, &have_ll, k_zs_ll_norm, 36, 6, 35, 9, sm);
      if (u < 0) return ZS_FAIL;                             /* LL table */
      lp += u;
      u = zs_seq_table((modes >> 4) & 3, b + lp, bend - lp, tof, &of_log, &have_of, k_zs_of_norm, 29, 5, 31, 8, sm);
      if (u < 0) return ZS_FAIL;                             /* OF table */
      lp += u;
      u = zs_seq_table((modes >> 2) & 3, b + lp, bend - lp, tml, &ml_log, &have_ml, k_zs_ml_norm, 53, 6, 52, 9, sm);
      if (u < 0) return ZS_FAIL;                             /* ML table */
      lp += u;
      ZsBack sb;
      if (!zs_back_init(sb, b + lp, bend - lp)) return ZS_FAIL;
      u32 sl = zs_back_read(sb, ll_log), so = zs_back_read(sb, of_log), sml = zs_back_read(sb, ml_log);
      if (sb.pos < 0) return ZS_FAIL;
      for (int i = 0; i < nseq; i++) {
        const int oc = tof[so].sym, mc = tml[sml].sym, lc = tll[sl].sym;
        if (oc > 31 || mc > 52 || lc > 35) return ZS_FAIL;
        const u32 ov = (1u << oc) + zs_back_read(sb, oc);
        const u32 ml = k_zs_ml_base[mc] + zs_back_read(sb, k_zs_ml_bits[mc]);
        const u32 ll = k_zs_ll_base[lc] + zs_back_read(sb, k_zs_ll_bits[lc]);
        if (i + 1 < nseq) {                                  /* state updates: literal length, match length, offset */
          sl = tll[sl].base + zs_back_read(sb, tll[sl].nbits);
          sml = tml[sml].base + zs_back_read(sb, tml[sml].nbits);
          so = tof[so].base + zs_back_read(sb, tof[so].nbits);
        }
        if (sb.pos < 0) return ZS_FAIL;
        u32 offset;
        if (ov > 3) { offset = ov - 3; rep3 = rep2; rep2 = rep1; rep1 = offset; }
        else {
          const u32 idx = ov + (ll == 0 ? 1u : 0u);
          if (idx == 1) offset = rep1;
          else {
            offset = idx == 2 ? rep2 : (idx == 3 ? rep3 : rep1 - 1u);
            if (offset == 0) return ZS_FAIL;
            if (idx != 2) rep3 = rep2;
            rep2 = rep1; rep1 = offset;
          }
        }
        if ((u64)op + ll + ml > (u64)cap || op + (int)ll + (int)ml - block_start > ZS_BLOCKMAX) return ZS_FAIL;
        if (!zs_lit_take(L, huf, out + op, (int)ll)) return ZS_FAIL;
        op += (int)ll;
        if (offset > (u32)op) return ZS_FAIL;                     /* before the start of the frame */
        for (u32 k = 0; k < ml; k++) out[op + k] = out[op + k - offset];
        op += (int)ml;
      }
      if (sb.pos != 0) return ZS_FAIL;                            /* the sequence bitstream must be used up exactly */
    } else if (lp != bend) return ZS_FAIL;
    /* ---- the literals after the last sequence ---- */
    {
      const int rest = L.left;
      if (op + rest > cap || op + rest - block_start > ZS_BLOCKMAX) return ZS_FAIL;
      if (!zs_lit_take(L, huf, out + op, rest)) return ZS_FAIL;
      op += rest;
      if (L.type == 2) for (int k = 0; k < L.nstreams; k++) if (L.s[k].pos != 0 || L.quota[k] != 0) return ZS_FAIL;
    }
  } while (!last);
  if (fcs_bytes && (u64)op != fcs) return ZS_FAIL;
  if (checksum) {
    if (ip + 4 > csize) return ZS_FAIL;
    const u32 want = (u32)in[ip] | ((u32)in[ip + 1] << 8) | ((u32)in[ip + 2] << 16) | ((u32)in[ip + 3] << 24);
    if ((u32)zs_xxh64(out, op) != want) return ZS_FAIL;
    ip += 4;
  }
  *used = ip;
  return op;
}

/* Runs on ONE lane: frames and skippable frames until the input is used up, as ZSTD_decompress does
 * (ZSTD_decompressMultiFrame).  Each frame starts with fresh tables and repeat offsets, its content size is held
 * to the room left and its checksum covers its own output.  Returns bytes written or -1; an input of skippable
 * frames only gives 0. */
DEV int zs_frame_serial(const u8* in, int csize, u8* out, int cap, u8* sm) {
  int ip = 0, op = 0;
  while (ip < csize) {
    if (csize - ip < 5) return ZS_FAIL;                          /* 1 to 4 bytes after the last frame */
    const u32 magic = (u32)in[ip] | ((u32)in[ip + 1] << 8) | ((u32)in[ip + 2] << 16) | ((u32)in[ip + 3] << 24);
    if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {                  /* skippable frame: 4-byte size, then that many bytes */
      if (csize - ip < 8) return ZS_FAIL;
      const u32 fsz = (u32)in[ip + 4] | ((u32)in[ip + 5] << 8) | ((u32)in[ip + 6] << 16) | ((u32)in[ip + 7] << 24);
      if (fsz > (u32)(csize - ip - 8)) return ZS_FAIL;
      ip += 8 + (int)fsz;
      continue;
    }
    int used = 0;
    const int n = zs_frame_one(in + ip, csize - ip, out + op, cap - op, sm, &used);
    if (n < 0) return -1;
    ip += used; op += n;
  }
  return op;
}

/* ZSTD_decompress() of one frame (reference blosc/blosc.c:517-529): bytes written or -1.
 * Uniform across the warp.  `smem` = ZS_SMEM_BYTES of warp-private shared memory. */
DEV int zstd_decode_warp(const u8* __restrict__ in, const int csize, u8* out, const int cap, void* smem) {
  int n = -1;
  if (lane_id() == 0) n = zs_frame_serial(in, csize, out, cap, (u8*)smem);
  n = __shfl_sync(FULLMASK, n, 0);
  __syncwarp();
  return n;
}

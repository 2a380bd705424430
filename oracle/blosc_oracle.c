/*
 * blosc_oracle.c -- TEST INFRASTRUCTURE ONLY (see blosc_oracle.h).
 *
 * A from-scratch, index-based, single-threaded restatement of the c-blosc hot path.
 * Written for clarity, not speed: every loop is the textbook form of what the
 * reference's SIMD / pointer code computes.  Parity is pinned against the reference
 * itself (oracle/_ref) and the compat golden chunks by the tests.
 */
#include "blosc_oracle.h"

#include <limits.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------- */
/* small helpers                                                             */
/* ------------------------------------------------------------------------- */
static uint32_t ld32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint64_t ld64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
static int32_t  ldi32(const uint8_t* p) { /* blosc.c:243-265 sw32_, little-endian wire order */
  return (int32_t)((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24));
}
static void sti32(uint8_t* p, int32_t v) { /* blosc.c:269-289 _sw32 */
  uint32_t u = (uint32_t)v;
  p[0] = (uint8_t)u; p[1] = (uint8_t)(u >> 8); p[2] = (uint8_t)(u >> 16); p[3] = (uint8_t)(u >> 24);
}

/* ------------------------------------------------------------------------- */
/* filters                                                                   */
/* ------------------------------------------------------------------------- */

/* shuffle-generic.h:32-52: dst[j*N+i] = src[i*ts+j]; the blocksize%ts tail is copied. */
void orc_shuffle(size_t ts, size_t n, const uint8_t* src, uint8_t* dst) {
  size_t ne = n / ts, i, j;
  for (j = 0; j < ts; j++)
    for (i = 0; i < ne; i++) dst[j * ne + i] = src[i * ts + j];
  memcpy(dst + ne * ts, src + ne * ts, n - ne * ts);
}

/* shuffle-generic.h:61-81 */
void orc_unshuffle(size_t ts, size_t n, const uint8_t* src, uint8_t* dst) {
  size_t ne = n / ts, i, j;
  for (i = 0; i < ne; i++)
    for (j = 0; j < ts; j++) dst[i * ts + j] = src[j * ne + i];
  memcpy(dst + ne * ts, src + ne * ts, n - ne * ts);
}

/* shuffle.c:393-416 + bitshuffle-generic.c:125-139.  For N = n/ts elements with N%8==0:
 * output row r = 8*b + k (b = byte index inside the element, k = bit, LSB first) has N/8
 * bytes; bit m of byte i of that row is bit k of byte b of element 8*i+m.  The tail
 * n - N*ts is copied.  If N%8 != 0 the whole block is copied (shuffle.c:412-415). */
int orc_bitshuffle(size_t ts, size_t n, const uint8_t* src, uint8_t* dst) {
  size_t N = n / ts, rowlen, b, k, i, m;
  if (N % 8) { memcpy(dst, src, n); return (int)N; }
  rowlen = N / 8;
  for (b = 0; b < ts; b++)
    for (k = 0; k < 8; k++)
      for (i = 0; i < rowlen; i++) {
        unsigned v = 0;
        for (m = 0; m < 8; m++) v |= ((src[(8 * i + m) * ts + b] >> k) & 1u) << m;
        dst[(8 * b + k) * rowlen + i] = (uint8_t)v;
      }
  memcpy(dst + N * ts, src + N * ts, n - N * ts);
  return (int)(N * ts);
}

/* shuffle.c:420-443 + bitshuffle-generic.c:208-220 (exact inverse of the above) */
int orc_bitunshuffle(size_t ts, size_t n, const uint8_t* src, uint8_t* dst) {
  size_t N = n / ts, rowlen, b, k, e;
  if (N % 8) { memcpy(dst, src, n); return (int)N; }
  rowlen = N / 8;
  for (e = 0; e < N; e++)
    for (b = 0; b < ts; b++) {
      unsigned v = 0;
      for (k = 0; k < 8; k++) v |= ((src[(8 * b + k) * rowlen + e / 8] >> (e % 8)) & 1u) << k;
      dst[e * ts + b] = (uint8_t)v;
    }
  memcpy(dst + N * ts, src + N * ts, n - N * ts);
  return (int)(N * ts);
}

/* ------------------------------------------------------------------------- */
/* BloscLZ                                                                   */
/* ------------------------------------------------------------------------- */
#define BLZ_MAX_COPY 32
#define BLZ_MAX_DISTANCE 8191                       /* blosclz.c:43 */
#define BLZ_MAX_FARDISTANCE (65535 + 8191 - 1)      /* blosclz.c:44 */

static uint32_t blz_hash(uint32_t seq, unsigned hashlog) { /* blosclz.c:58-60 */
  return (seq * 2654435761u) >> (32u - hashlog);
}

/* What get_run_or_match returns (blosclz.c:117-163,166-188,216-243), as an index:
 * with p the first position >= ip where b[p] != b[p-dist], the result is min(p+1, bound).
 * (get_match stops one PAST the mismatch; get_run stops AT the mismatch of the
 * ref pointer, which trails ip by one -- the same number.) */
static int32_t blz_match_end(const uint8_t* b, int32_t ip, int32_t dist, int32_t bound) {
  while (ip < bound && b[ip] == b[ip - dist]) ip++;
  return ip < bound ? ip + 1 : bound;
}

/* blosclz.c:318-418 get_cratio: dry run of the encoder over <= 4096 bytes with a
 * 2^12 x u16 table, counting output bytes only. */
static double blz_probe(const uint8_t* b, int maxlen, int minlen, int ipshift) {
  uint16_t htab[1 << 12];
  int32_t limit = maxlen > 4096 ? 4096 : maxlen;
  int32_t ip = 0, ip_bound = limit - 1, ip_limit = limit - 12, oc = 0;
  unsigned copy = 4;
  memset(htab, 0, sizeof htab);
  oc += 5;
  while (ip < ip_limit) {
    int32_t anchor = ip, ref, len;
    uint32_t seq = ld32(b + ip), h = blz_hash(seq, 12);
    unsigned distance;
    int is_lit = 0;
    ref = htab[h];
    distance = (unsigned)(anchor - ref);
    htab[h] = (uint16_t)anchor;
    if (distance == 0 || distance >= BLZ_MAX_FARDISTANCE) is_lit = 1;
    else if (ld32(b + ref) != seq) is_lit = 1;
    else {
      distance--;
      ip = blz_match_end(b, anchor + 4, (int32_t)distance + 1, ip_bound);
      ip -= ipshift;
      len = ip - anchor;
      if (len < minlen) is_lit = 1;
      else {
        if (!copy) oc--;
        copy = 0;
        if (len >= 7) oc += (len - 7) / 255 + 1;
        oc += (distance < BLZ_MAX_DISTANCE) ? 2 : 4;
        h = blz_hash(ld32(b + ip), 12);
        htab[h] = (uint16_t)ip;
        ip += 2;
        oc++;
      }
    }
    if (is_lit) { /* LITERAL2, blosclz.c:258-266 */
      oc++; anchor++; ip = anchor; copy++;
      if (copy == BLZ_MAX_COPY) { copy = 0; oc++; }
    }
  }
  return (double)ip / (double)oc;
}

int orc_blosclz_compress(int clevel, const void* input, int length, void* output,
                         int maxout, int split_block) {
  static const double min_cratio[10] = {0, 2, 1.5, 1.2, 1.2, 1.2, 1.2, 1.15, 1.1, 1.0};
  static const uint8_t hashlog_[10] = {0, 12, 13, 14, 14, 14, 14, 14, 14, 14};
  const uint8_t* b = (const uint8_t*)input;
  uint8_t* out = (uint8_t*)output;
  int maxlen = length / 4, shift = length - maxlen;
  double cratio = blz_probe(b + shift, maxlen, 3, 3);          /* blosclz.c:425-430 */
  int32_t ipshift = 4, minlen = 4;
  unsigned hashlog;
  uint32_t* htab;
  int32_t ip = 0, ip_bound = length - 1, ip_limit = length - 12, op = 0, op_limit = maxout;
  unsigned copy;

  if (cratio < min_cratio[clevel]) return 0;                    /* :432-435 */
  if (!split_block || cratio < 4) { ipshift = 3; minlen = 3; }  /* :445-457 */
  hashlog = hashlog_[clevel];
  if (length < 16 || maxout < 66) return 0;                     /* :473-475 */

  htab = (uint32_t*)calloc((size_t)1 << 14, sizeof(uint32_t));
  if (!htab) return 0;

  copy = 4;                                                     /* :481-487 */
  out[op++] = BLZ_MAX_COPY - 1;
  out[op++] = b[ip++]; out[op++] = b[ip++]; out[op++] = b[ip++]; out[op++] = b[ip++];

#define ORC_FAIL do { free(htab); return 0; } while (0)
  while (ip < ip_limit) {                                       /* :490 */
    int32_t anchor = ip, ref;
    uint32_t seq = ld32(b + ip), h = blz_hash(seq, hashlog), len;
    unsigned distance;
    int is_lit = 0;
    ref = (int32_t)htab[h];
    distance = (unsigned)(anchor - ref);
    htab[h] = (uint32_t)anchor;
    if (distance == 0 || distance >= BLZ_MAX_FARDISTANCE) is_lit = 1;      /* :506 */
    else if (ld32(b + ref) != seq) is_lit = 1;                              /* :512 */
    else {
      distance--;                                                           /* :524 */
      ip = blz_match_end(b, anchor + 4, (int32_t)distance + 1, ip_bound);   /* :527 */
      ip -= ipshift;                                                        /* :530 */
      len = (uint32_t)(ip - anchor);
      if (len < (uint32_t)minlen || (len <= 5 && distance >= BLZ_MAX_DISTANCE)) is_lit = 1;  /* :535 */
    }
    if (is_lit) {                                                           /* LITERAL :246-256 */
      if (op + 2 > op_limit) ORC_FAIL;
      out[op++] = b[anchor++];
      ip = anchor;
      copy++;
      if (copy == BLZ_MAX_COPY) { copy = 0; out[op++] = BLZ_MAX_COPY - 1; }
      continue;
    }
    if (copy) out[op - copy - 1] = (uint8_t)(copy - 1); else op--;         /* :541-546 */
    copy = 0;
    if (distance < BLZ_MAX_DISTANCE) {
      if (len < 7) {                                                        /* MATCH_SHORT :268-273 */
        if (op + 2 > op_limit) ORC_FAIL;
        out[op++] = (uint8_t)((len << 5) + (distance >> 8));
        out[op++] = (uint8_t)(distance & 255);
      } else {                                                              /* MATCH_LONG :275-288 */
        if (op + 1 > op_limit) ORC_FAIL;
        out[op++] = (uint8_t)((7u << 5) + (distance >> 8));
        for (len -= 7; len >= 255; len -= 255) { if (op + 1 > op_limit) ORC_FAIL; out[op++] = 255; }
        if (op + 2 > op_limit) ORC_FAIL;
        out[op++] = (uint8_t)len;
        out[op++] = (uint8_t)(distance & 255);
      }
    } else {
      distance -= BLZ_MAX_DISTANCE;                                         /* :559 */
      if (len < 7) {                                                        /* MATCH_SHORT_FAR :290-297 */
        if (op + 4 > op_limit) ORC_FAIL;
        out[op++] = (uint8_t)((len << 5) + 31);
        out[op++] = 255;
        out[op++] = (uint8_t)(distance >> 8);
        out[op++] = (uint8_t)(distance & 255);
      } else {                                                              /* MATCH_LONG_FAR :299-314 */
        if (op + 1 > op_limit) ORC_FAIL;
        out[op++] = (uint8_t)((7u << 5) + 31);
        for (len -= 7; len >= 255; len -= 255) { if (op + 1 > op_limit) ORC_FAIL; out[op++] = 255; }
        if (op + 4 > op_limit) ORC_FAIL;
        out[op++] = (uint8_t)len;
        out[op++] = 255;
        out[op++] = (uint8_t)(distance >> 8);
        out[op++] = (uint8_t)(distance & 255);
      }
    }
    seq = ld32(b + ip);                                                     /* :568-580 */
    htab[blz_hash(seq, hashlog)] = (uint32_t)ip++;
    if (clevel == 9) { seq >>= 8; htab[blz_hash(seq, hashlog)] = (uint32_t)ip++; }
    else ip++;
    if (op + 1 > op_limit) ORC_FAIL;                                        /* :582-586 */
    out[op++] = BLZ_MAX_COPY - 1;
  }
  while (ip <= ip_bound) {                                                  /* :589-598 */
    if (op + 2 > op_limit) ORC_FAIL;
    out[op++] = b[ip++];
    copy++;
    if (copy == BLZ_MAX_COPY) { copy = 0; out[op++] = BLZ_MAX_COPY - 1; }
  }
  if (copy) out[op - copy - 1] = (uint8_t)(copy - 1); else op--;           /* :600-604 */
  out[0] |= (1u << 5);                                                      /* :607 */
  free(htab);
  return op;
#undef ORC_FAIL
}

int orc_blosclz_decompress(const void* input, int length, void* output, int maxout) {
  const uint8_t* in = (const uint8_t*)input;
  uint8_t* out = (uint8_t*)output;
  int64_t ip = 0, op = 0;
  uint32_t ctrl;
  if (length == 0) return 0;                                    /* blosclz.c:685-687 */
  ctrl = in[ip++] & 31u;
  for (;;) {
    if (ctrl >= 32) {                                           /* match, :691-765 */
      int64_t len = (int64_t)(ctrl >> 5) - 1, ofs = (int64_t)(ctrl & 31u) << 8, ref = op - ofs, i;
      uint8_t code;
      if (len == 6) {
        do {
          if (ip + 1 >= length) return 0;
          code = in[ip++];
          len += code;
        } while (code == 255);
      } else if (ip + 1 >= length) return 0;
      code = in[ip++];
      len += 3;
      ref -= code;
      if (code == 255 && ofs == (31 << 8)) {                    /* 16-bit far distance, :717-726 */
        if (ip + 1 >= length) return 0;
        ofs = (int64_t)in[ip++] << 8;
        ofs += in[ip++];
        ref = op - ofs - BLZ_MAX_DISTANCE;
      }
      if (op + len > maxout) return 0;                          /* :728-730 */
      if (ref - 1 < 0) return 0;                                /* :732-734 */
      if (ip >= length) break;                                  /* :736 -- ends WITHOUT copying */
      ctrl = in[ip++];
      ref--;
      for (i = 0; i < len; i++) out[op + i] = out[ref + i];     /* forward byte copy, overlap ok */
      op += len;
    } else {                                                    /* literal run, :766-785 */
      ctrl++;
      if (op + ctrl > (uint32_t)maxout) return 0;
      if (ip + ctrl > (uint32_t)length) return 0;
      memcpy(out + op, in + ip, ctrl);
      op += ctrl; ip += ctrl;
      if (ip >= length) break;
      ctrl = in[ip++];
    }
  }
  return (int)op;
}

/* ------------------------------------------------------------------------- */
/* LZ4 block codec                                                           */
/* ------------------------------------------------------------------------- */
#define LZ4_MFLIMIT 12
#define LZ4_LASTLITERALS 5
#define LZ4_MAXDIST 65535u

static uint32_t lz4_hash(const uint8_t* p, int byU16) {        /* lz4.c:777-806 */
  if (byU16) return (ld32(p) * 2654435761u) >> (32 - 13);
  return (uint32_t)(((ld64(p) << 24) * 889523592379ull) >> (64 - 12));
}

int orc_lz4_compress_fast(const char* source, char* dest, int n, int cap, int accel) {
  const uint8_t* s = (const uint8_t*)source;
  uint8_t* d = (uint8_t*)dest;
  uint32_t tab[4096];          /* byU32 mode: 4096 x u32 (hash5, 12 bits) */
  uint16_t tab16[8192];        /* byU16 mode: 8192 x u16 (hash4, 13 bits) -- same 16 KiB budget */
  int byU16, limited;
  int64_t bound, ip, anchor = 0, op = 0, olimit, mflimitPlusOne, matchlimit, match, token;
  uint32_t forwardH;

  if (accel < 1) accel = 1;                                     /* lz4.c:1386-1387 */
  if (accel > 65537) accel = 65537;
  if ((unsigned)n > 0x7E000000u) return 0;                      /* :1360 */
  bound = (int64_t)n + n / 255 + 16;                            /* lz4.h:215 */
  limited = cap < bound;                                        /* :1388,1395 */
  if (n == 0) {                                                 /* :1361-1371 */
    if (limited && cap <= 0) return 0;
    d[0] = 0;
    return 1;
  }
  byU16 = n < 65536 + LZ4_MFLIMIT - 1;                          /* :710, :1389 */
  olimit = cap;
  mflimitPlusOne = (int64_t)n - LZ4_MFLIMIT + 1;
  matchlimit = (int64_t)n - LZ4_LASTLITERALS;
  memset(tab, 0, sizeof tab);
  memset(tab16, 0, sizeof tab16);

#define TGET(h) (byU16 ? (int64_t)tab16[h] : (int64_t)tab[h])
#define TPUT(h, v) do { if (byU16) tab16[h] = (uint16_t)(v); else tab[h] = (uint32_t)(v); } while (0)

  if (n < LZ4_MFLIMIT + 1) goto last_literals;                  /* :1002 */
  TPUT(lz4_hash(s, byU16), 0);                                  /* :1005-1010 */
  ip = 1;
  forwardH = lz4_hash(s + ip, byU16);

  for (;;) {
    {                                                           /* find a match, :1043-1101 */
      int64_t forwardIp = ip;
      int step = 1, searchMatchNb = accel << 6;
      for (;;) {
        uint32_t h = forwardH;
        int64_t current = forwardIp, matchIndex = TGET(h);
        ip = forwardIp;
        forwardIp += step;
        step = searchMatchNb++ >> 6;
        if (forwardIp > mflimitPlusOne) goto last_literals;
        forwardH = lz4_hash(s + forwardIp, byU16);
        TPUT(h, current);
        if (!byU16 && matchIndex + LZ4_MAXDIST < current) continue;   /* too far */
        if (ld32(s + matchIndex) == ld32(s + ip)) { match = matchIndex; break; }
      }
    }
    while (ip > anchor && match > 0 && s[ip - 1] == s[match - 1]) { ip--; match--; }  /* catch up :1107-1109 */
    {                                                           /* literals, :1112-1136 */
      int64_t lit = ip - anchor;
      token = op++;
      if (limited && op + lit + (2 + 1 + LZ4_LASTLITERALS) + lit / 255 > olimit) return 0;
      if (lit >= 15) {
        int64_t len = lit - 15;
        d[token] = 15 << 4;
        for (; len >= 255; len -= 255) d[op++] = 255;
        d[op++] = (uint8_t)len;
      } else d[token] = (uint8_t)(lit << 4);
      memcpy(d + op, s + anchor, (size_t)lit);
      op += lit;
    }
  next_match:
    {
      int64_t off = ip - match, mc = 0, p = ip + 4, q = match + 4;
      d[op++] = (uint8_t)off; d[op++] = (uint8_t)(off >> 8);    /* :1162 */
      while (p < matchlimit && s[p] == s[q]) { p++; q++; mc++; } /* LZ4_count :671-702 */
      ip += mc + 4;
      if (limited && op + (1 + LZ4_LASTLITERALS) + (mc + 240) / 255 > olimit) return 0;  /* :1187-1211 */
      if (mc >= 15) {                                           /* :1212-1224 */
        d[token] += 15;
        mc -= 15;
        for (; mc >= 255; mc -= 255) d[op++] = 255;
        d[op++] = (uint8_t)mc;
      } else d[token] += (uint8_t)mc;
    }
    anchor = ip;
    if (ip >= mflimitPlusOne) break;                            /* :1230-1233 */
    TPUT(lz4_hash(s + ip - 2, byU16), ip - 2);                  /* :1236-1242 */
    {                                                           /* test next position, :1255-1294 */
      uint32_t h = lz4_hash(s + ip, byU16);
      int64_t current = ip, matchIndex = TGET(h);
      TPUT(h, current);
      if ((byU16 || matchIndex + LZ4_MAXDIST >= current) && ld32(s + matchIndex) == ld32(s + ip)) {
        token = op++;
        d[token] = 0;
        match = matchIndex;
        goto next_match;
      }
    }
    forwardH = lz4_hash(s + (++ip), byU16);                     /* :1298 */
  }

last_literals:                                                  /* :1302-1329 */
  {
    int64_t lastRun = (int64_t)n - anchor;
    if (limited && op + lastRun + 1 + (lastRun + 255 - 15) / 255 > olimit) return 0;
    if (lastRun >= 15) {
      int64_t acc = lastRun - 15;
      d[op++] = 15 << 4;
      for (; acc >= 255; acc -= 255) d[op++] = 255;
      d[op++] = (uint8_t)acc;
    } else d[op++] = (uint8_t)(lastRun << 4);
    memcpy(d + op, s + anchor, (size_t)lastRun);
    op += lastRun;
  }
  return (int)op;
#undef TGET
#undef TPUT
}

/* ------------------------------------------------------------------------- */
/* LZ4, segment-parallel parse (NOT the reference's parse: the specification of the library's  */
/* opt-in BLOSC_B200_PARSE=segmented mode, restated here so the GPU output can be checked byte  */
/* for byte and so that tests can hand it to the reference's decoder)                           */
/* ------------------------------------------------------------------------- */
/* A stream of n bytes is cut into segments of seg_bytes.  Every segment is parsed on its own by the
 * greedy loop of LZ4_compress_fast above with these differences:
 *   - the hash table starts empty and is warmed with every position of the `warm` bytes in front
 *     of the segment (ascending, so the most recent position of a hash wins); matches may reach
 *     back into earlier segments (the usual 64 KiB window), never forward;
 *   - the end-of-block rules (last match starts >= 12 bytes before the end, ends >= 5 bytes before
 *     it, lz4.c:954-955) are applied to the segment end as well as to the stream end;
 *   - the literals in front of the first match and after the last one are not encoded by the
 *     segment: it reports their counts (lit0, tail) and the bytes in between (`body`: offset and
 *     length bytes of the first match, then whole sequences).  A segment whose body does not fit a
 *     slot of its own size under the reference's limitedOutput checks counts as "no match".
 * The stream is the LZ4 encoding of the concatenated sequences: the tail of a segment (and whole
 * match-less segments) become part of the literal run of the next first match, and one final
 * literal run ends the block.  Any LZ4 decoder reads it; it is not the reference's byte stream. */
typedef struct { int lit0, tokml, body, tail; } orc_segmeta;

static int lz4_parse_segment(const uint8_t* s, int64_t n, int64_t b, int64_t e, int accel, int byU16, int64_t warm,
                             uint8_t* d, int64_t olimit, orc_segmeta* m) {
  uint32_t tab[4096];
  uint16_t tab16[8192];
  int64_t ip, anchor = b, op = 0, mflimitPlusOne, matchlimit, match, token = -1, q;
  uint32_t forwardH;
  int first = 1;
  m->lit0 = -1; m->tokml = 0; m->body = 0; m->tail = (int)(e - b);
  memset(tab, 0, sizeof tab);
  memset(tab16, 0, sizeof tab16);
#define TGET(h) (byU16 ? (int64_t)tab16[h] : (int64_t)tab[h])
#define TPUT(h, v) do { if (byU16) tab16[h] = (uint16_t)(v); else tab[h] = (uint32_t)(v); } while (0)
  for (q = b - warm > 0 ? b - warm : 0; q < b; q++)
    if (q + 8 <= n) TPUT(lz4_hash(s + q, byU16), q);
  mflimitPlusOne = e - LZ4_MFLIMIT + 1;
  matchlimit = e < n - LZ4_LASTLITERALS ? e : n - LZ4_LASTLITERALS;
  if (e - b < LZ4_MFLIMIT + 1) return 0;
  TPUT(lz4_hash(s + b, byU16), b);
  ip = b + 1;
  forwardH = lz4_hash(s + ip, byU16);
  for (;;) {
    {
      int64_t forwardIp = ip;
      int step = 1, searchMatchNb = accel << 6;
      for (;;) {
        uint32_t h = forwardH;
        int64_t current = forwardIp, matchIndex = TGET(h);
        ip = forwardIp;
        forwardIp += step;
        step = searchMatchNb++ >> 6;
        if (forwardIp > mflimitPlusOne) goto done;
        forwardH = lz4_hash(s + forwardIp, byU16);
        TPUT(h, current);
        if (!byU16 && matchIndex + LZ4_MAXDIST < current) continue;
        if (ld32(s + matchIndex) == ld32(s + ip)) { match = matchIndex; break; }
      }
    }
    while (ip > anchor && match > 0 && s[ip - 1] == s[match - 1]) { ip--; match--; }
    {
      int64_t lit = ip - anchor;
      if (first) {                                              /* counted, not stored */
        if (op + (2 + 1 + LZ4_LASTLITERALS) > olimit) return -1;
        m->lit0 = (int)lit;
      } else {
        token = op++;
        if (op + lit + (2 + 1 + LZ4_LASTLITERALS) + lit / 255 > olimit) return -1;
        if (lit >= 15) {
          int64_t len = lit - 15;
          d[token] = 15 << 4;
          for (; len >= 255; len -= 255) d[op++] = 255;
          d[op++] = (uint8_t)len;
        } else d[token] = (uint8_t)(lit << 4);
        memcpy(d + op, s + anchor, (size_t)lit);
        op += lit;
      }
    }
  next_match:
    {
      int64_t off = ip - match, mc = 0, p = ip + 4, r = match + 4;
      d[op++] = (uint8_t)off; d[op++] = (uint8_t)(off >> 8);
      while (p < matchlimit && s[p] == s[r]) { p++; r++; mc++; }
      ip += mc + 4;
      if (op + (1 + LZ4_LASTLITERALS) + (mc + 240) / 255 > olimit) return -1;
      if (mc >= 15) {
        if (first) m->tokml = 15; else d[token] += 15;
        mc -= 15;
        for (; mc >= 255; mc -= 255) d[op++] = 255;
        d[op++] = (uint8_t)mc;
      } else if (first) m->tokml = (int)mc;
      else d[token] += (uint8_t)mc;
      first = 0;
    }
    anchor = ip;
    if (ip >= mflimitPlusOne) break;
    TPUT(lz4_hash(s + ip - 2, byU16), ip - 2);
    {
      uint32_t h = lz4_hash(s + ip, byU16);
      int64_t current = ip, matchIndex = TGET(h);
      TPUT(h, current);
      if ((byU16 || matchIndex + LZ4_MAXDIST >= current) && ld32(s + matchIndex) == ld32(s + ip)) {
        token = op++;
        d[token] = 0;
        match = matchIndex;
        goto next_match;
      }
    }
    forwardH = lz4_hash(s + (++ip), byU16);
  }
done:
  if (first) return 0;                                          /* no match in this segment */
  m->body = (int)op;
  m->tail = (int)(e - anchor);
  return 1;
#undef TGET
#undef TPUT
}

static int64_t lz4_put_litlen(uint8_t* d, int64_t op, int64_t lit, int tokml) {
  d[op++] = (uint8_t)(((lit >= 15 ? 15 : lit) << 4) | tokml);
  if (lit >= 15) {
    int64_t len = lit - 15;
    for (; len >= 255; len -= 255) d[op++] = 255;
    d[op++] = (uint8_t)len;
  }
  return op;
}

/* returns the compressed size, or 0 when it would not fit in cap */
int orc_lz4_compress_segmented(const char* source, char* dest, int n, int cap, int accel, int seg_bytes, int warm) {
  const uint8_t* s = (const uint8_t*)source;
  uint8_t* d = (uint8_t*)dest;
  uint8_t* body;
  const int byU16 = n < 65536 + LZ4_MFLIMIT - 1;
  int64_t b, op = 0, carry = 0, need;
  if (accel < 1) accel = 1;
  if (accel > 65537) accel = 65537;
  if (n <= 0 || seg_bytes < 64) return 0;
  body = (uint8_t*)malloc((size_t)seg_bytes + 64);
  if (!body) return 0;
  for (b = 0; b < n; b += seg_bytes) {
    const int64_t e = b + seg_bytes < n ? b + seg_bytes : n;
    orc_segmeta m;
    const int r = lz4_parse_segment(s, n, b, e, accel, byU16, warm, body, e - b, &m);
    if (r <= 0) { carry += e - b; continue; }
    {
      const int64_t lit = carry + m.lit0;
      need = op + 1 + (lit >= 15 ? (lit - 15) / 255 + 1 : 0) + lit + m.body;
      if (need > cap) { free(body); return 0; }
      op = lz4_put_litlen(d, op, lit, m.tokml);
      memcpy(d + op, s + b - carry, (size_t)lit); op += lit;
      memcpy(d + op, body, (size_t)m.body); op += m.body;
      carry = m.tail;
    }
  }
  need = op + 1 + (carry >= 15 ? (carry - 15) / 255 + 1 : 0) + carry;
  free(body);
  if (need > cap) return 0;
  op = lz4_put_litlen(d, op, carry, 0);
  memcpy(d + op, s + n - carry, (size_t)carry); op += carry;
  return (int)op;
}

static int g_lz4_seg_bytes = 0, g_lz4_seg_warm = 0;   /* 0: the reference's parse */
void orc_set_lz4_segmented(int seg_bytes, int warm) { g_lz4_seg_bytes = seg_bytes; g_lz4_seg_warm = warm; }

/* LZ4_decompress_safe (lz4.c:2451-2456): full-block decode, no dictionary.  The accept /
 * reject rules below are those of the "safe" decode loop (lz4.c:2234-2436); the fast
 * loop (:2077-2230) only ever handles sequences far from both buffer ends and applies
 * the same offset check, so it accepts exactly the same streams.  offset == 0 (invalid, but
 * accepted) decodes to zeros in every copy routine of lz4.c 1.10 (they clear the first
 * destination word before replicating it), and so it does here. */
int orc_lz4_decompress_safe(const char* src, char* dst, int csize, int cap) {
  const uint8_t* in = (const uint8_t*)src;
  uint8_t* out = (uint8_t*)dst;
  int64_t ip = 0, op = 0, iend = csize, oend = cap;
  if (src == NULL || cap < 0) return -1;
  if (cap == 0) return (csize == 1 && in[0] == 0) ? 0 : -1;     /* :2062-2066 */
  if (csize == 0) return -1;
  for (;;) {
    unsigned token = in[ip++];
    int64_t len = token >> 4, cpy, off, match, i;
    if (len == 15) {                                            /* read_variable_length(.., iend-15, 1) :1975-2011 */
      unsigned sb;
      if (ip >= iend - 15) return -1;
      do {
        sb = in[ip++];
        len += sb;
        if (ip > iend - 15) return -1;
      } while (sb == 255);
    }
    cpy = op + len;
    if (cpy > oend - LZ4_MFLIMIT || ip + len > iend - (2 + 1 + LZ4_LASTLITERALS)) {  /* :2289-2331 */
      if (ip + len != iend || cpy > oend) return -1;
      memmove(out + op, in + ip, (size_t)len);
      op += len;
      break;
    }
    memcpy(out + op, in + ip, (size_t)len);
    ip += len; op = cpy;
    off = in[ip] | (in[ip + 1] << 8); ip += 2;                  /* :2337-2338 */
    match = op - off;
    len = token & 15;
    if (len == 15) {                                            /* read_variable_length(.., iend-4, 0) */
      unsigned sb;
      do {
        sb = in[ip++];
        len += sb;
        if (ip > iend - LZ4_LASTLITERALS + 1) return -1;
      } while (sb == 255);
    }
    len += 4;
    if (match < 0) return -1;                                   /* :2356 */
    cpy = op + len;
    if (cpy > oend - LZ4_LASTLITERALS) return -1;               /* :2423 */
    if (off == 0) memset(out + op, 0, (size_t)len);             /* :2386-2390: the copy routines clear the first word and replicate it */
    else for (i = 0; i < len; i++) out[op + i] = out[match + i];
    op = cpy;
  }
  return (int)op;
}

/* ------------------------------------------------------------------------- */
/* chunk framing                                                             */
/* ------------------------------------------------------------------------- */
#define ORC_MAX_OVERHEAD 16
#define ORC_MIN_BUFFERSIZE 128
#define ORC_MAX_SPLITS 16
#define ORC_MAX_TYPESIZE 255
#define ORC_MAX_BLOCKSIZE ((INT_MAX - ORC_MAX_TYPESIZE * (int)sizeof(int32_t)) / 3)
enum { ORC_BLOSCLZ = 0, ORC_LZ4 = 1, ORC_LZ4HC = 2, ORC_SNAPPY = 3, ORC_ZLIB = 4, ORC_ZSTD = 5 };

static int orc_compcode(const char* name) {                     /* blosc.c:377-409, build with LZ4 only */
  if (!strcmp(name, "blosclz")) return ORC_BLOSCLZ;
  if (!strcmp(name, "lz4")) return ORC_LZ4;
  if (!strcmp(name, "lz4hc")) return ORC_LZ4HC;
  return -1;
}

static int orc_split_block(int compcode, int typesize, int blocksize) {  /* blosc.c:948-953 */
  return compcode != ORC_ZSTD && typesize <= ORC_MAX_SPLITS && blocksize / typesize >= ORC_MIN_BUFFERSIZE;
}

int32_t orc_compute_blocksize(int compcode, int clevel, int32_t typesize, int32_t nbytes,
                              int32_t forced) {
  int hcr = compcode == ORC_LZ4HC || compcode == ORC_ZLIB || compcode == ORC_ZSTD;
  int32_t bs;
  if (nbytes < typesize) return 1;                              /* blosc.c:969-971 */
  bs = nbytes;
  if (forced) {                                                 /* :975-985 */
    bs = forced;
    if (bs < ORC_MIN_BUFFERSIZE) bs = ORC_MIN_BUFFERSIZE;
    if (bs > ORC_MAX_BLOCKSIZE) bs = ORC_MAX_BLOCKSIZE;
  } else if (nbytes >= 32 * 1024) {                             /* :986-1029 */
    static const int mul8[10] = {2, 4, 8, 16, 32, 32, 64, 64, 64, 64};  /* (x/8): /4,/2,*1,*2,*4,*4,*8,*8,*8,*8 */
    bs = 32 * 1024;
    if (hcr) bs *= 2;
    bs = bs / 8 * mul8[clevel];
    if (clevel == 9 && hcr) bs *= 2;
  }
  if (clevel > 0 && orc_split_block(compcode, typesize, bs)) {  /* :1032-1047 */
    if (bs > (1 << 18)) bs = 1 << 18;
    bs *= typesize;
    if (bs < (1 << 16)) bs = 1 << 16;
    if (bs > 1024 * 1024) bs = 1024 * 1024;
  }
  if (bs > nbytes) bs = nbytes;                                 /* :1050-1052 */
  if (bs > typesize) bs = bs / typesize * typesize;             /* :1055-1057 */
  return bs;
}

typedef struct {
  int compcode, clevel, typesize, flags;
  int32_t nbytes, blocksize, nblocks, leftover, destsize;
} orc_ctx;

/* blosc.c:591-722 blosc_c.  tmp must hold bsize bytes. */
static int orc_block_c(const orc_ctx* c, int32_t bsize, int leftoverblock, int32_t ntbytes,
                       int32_t maxbytes, const uint8_t* src, uint8_t* dest, uint8_t* tmp) {
  int dont_split = (c->flags & 0x10) >> 4;
  int32_t ts = c->typesize, nsplits, neblock, j, ctbytes = 0, cbytes, maxout;
  const uint8_t* in = src;
  if ((c->flags & 1) && ts > 1) { orc_shuffle((size_t)ts, (size_t)bsize, src, tmp); in = tmp; }
  else if ((c->flags & 4) && bsize >= ts) { orc_bitshuffle((size_t)ts, (size_t)bsize, src, tmp); in = tmp; }
  nsplits = (!dont_split && !leftoverblock) ? ts : 1;
  neblock = bsize / nsplits;
  for (j = 0; j < nsplits; j++) {
    dest += 4; ntbytes += 4; ctbytes += 4;
    maxout = neblock;
    if (ntbytes + maxout > maxbytes) {                          /* :646-651 */
      maxout = maxbytes - ntbytes;
      if (maxout <= 0) return 0;
    }
    if (c->compcode == ORC_BLOSCLZ)
      cbytes = orc_blosclz_compress(c->clevel, in + j * neblock, neblock, dest, maxout, !dont_split);
    else if (c->compcode == ORC_LZ4)
      cbytes = g_lz4_seg_bytes ? orc_lz4_compress_segmented((const char*)in + j * neblock, (char*)dest, neblock, maxout,
                                                            10 - c->clevel, g_lz4_seg_bytes, g_lz4_seg_warm)
                               : orc_lz4_compress_fast((const char*)in + j * neblock, (char*)dest, neblock, maxout,
                                                       10 - c->clevel);
    else return -5;
    if (cbytes > maxout) return -1;
    if (cbytes < 0) return -2;
    if (cbytes == 0 || cbytes == neblock) {                     /* stored raw, :705-714 */
      if (ntbytes + neblock > maxbytes) return 0;
      memcpy(dest, in + j * neblock, (size_t)neblock);
      cbytes = neblock;
    }
    sti32(dest - 4, cbytes);
    dest += cbytes; ntbytes += cbytes; ctbytes += cbytes;
  }
  return ctbytes;
}

int orc_compress_ctx(int clevel, int doshuffle, size_t typesize, size_t nbytes, const void* src,
                     void* dest, size_t destsize, const char* compressor, size_t blocksize,
                     int numinternalthreads) {
  orc_ctx c;
  uint8_t* d = (uint8_t*)dest;
  const uint8_t* s = (const uint8_t*)src;
  uint8_t *tmp, *blk;
  int32_t ntbytes, j, pass, ebsize;
  int compformat, pool;
  /* initialize_context_compression, blosc.c:1062-1145 */
  if (nbytes > (size_t)(INT_MAX - ORC_MAX_OVERHEAD)) return 0;
  if (destsize < ORC_MAX_OVERHEAD) return 0;
  if (destsize - ORC_MAX_OVERHEAD > nbytes) destsize = nbytes + ORC_MAX_OVERHEAD;
  if (clevel < 0 || clevel > 9) return -10;
  if (doshuffle != 0 && doshuffle != 1 && doshuffle != 2) return -10;
  if (typesize == 0) return -10;
  if (typesize > ORC_MAX_TYPESIZE) typesize = 1;
  c.compcode = orc_compcode(compressor);
  c.clevel = clevel; c.typesize = (int)typesize; c.nbytes = (int32_t)nbytes; c.destsize = (int32_t)destsize;
  c.blocksize = orc_compute_blocksize(c.compcode, clevel, c.typesize, c.nbytes, (int32_t)blocksize);
  c.nblocks = c.nbytes / c.blocksize;
  c.leftover = c.nbytes % c.blocksize;
  if (c.leftover > 0) c.nblocks++;
  /* write_compression_header, blosc.c:1148-1247 */
  if (c.compcode == ORC_BLOSCLZ) compformat = 0;
  else if (c.compcode == ORC_LZ4) compformat = 1;
  else return -5;   /* lz4hc/zlib/zstd/snappy encoders are outside the hot path (SURVEY.md section 8) */
  d[0] = 2; d[1] = 1; d[2] = 0; d[3] = (uint8_t)c.typesize;
  sti32(d + 4, c.nbytes);
  sti32(d + 8, c.blocksize);
  ntbytes = 16 + 4 * c.nblocks;
  c.flags = 0;
  if (clevel == 0) { c.flags |= 2; ntbytes = 16; }
  if (c.nbytes < ORC_MIN_BUFFERSIZE) { c.flags |= 2; ntbytes = 16; }
  if (doshuffle == 1) c.flags |= 1;
  if (doshuffle == 2) c.flags |= 4;
  c.flags |= (!orc_split_block(c.compcode, c.typesize, c.blocksize)) << 4;
  c.flags |= compformat << 5;
  d[2] = (uint8_t)c.flags;
  /* blosc_compress_context, blosc.c:1250-1279 */
  if ((c.flags & 2) && c.nbytes + ORC_MAX_OVERHEAD > c.destsize) return 0;
  /* do_job (blosc.c:908-913): serial_blosc when nthreads is 1 or there is at most one block, else the pool
   * (t_blosc), which first validates nthreads (:1975-1986) */
  pool = numinternalthreads != 1 && c.nbytes / c.blocksize > 1;
  if (pool && (numinternalthreads < 1 || numinternalthreads > 256)) return -1;
  /* the pool compresses each block on its own into a scratch of ebsize bytes (:1745,1810) */
  ebsize = c.blocksize + c.typesize * 4;
  tmp = (uint8_t*)malloc((size_t)c.blocksize + 16 + (size_t)ebsize);
  if (!tmp) return -1;
  blk = tmp + c.blocksize + 16;
  for (pass = 0; pass < 2; pass++) {                            /* second pass = memcpy fallback :1264-1272 */
    for (j = 0; j < c.nblocks; j++) {                           /* serial_blosc :814-861, t_blosc :1792-1856 */
      int32_t bsize = c.blocksize, cb;
      int leftoverblock = 0;
      if (!(c.flags & 2)) sti32(d + 16 + 4 * j, ntbytes);
      if (j == c.nblocks - 1 && c.leftover > 0) { bsize = c.leftover; leftoverblock = 1; }
      if (c.flags & 2) {
        memcpy(d + 16 + (size_t)j * c.blocksize, s + (size_t)j * c.blocksize, (size_t)bsize);
        cb = bsize;
      } else if (pool) {
        /* no per-split clamp: the pool gives up only when the running total passes destsize (:1845-1850).
         * It copies the blocks out in whatever order they finish; this takes them in order, as the
         * serial path does. */
        cb = orc_block_c(&c, bsize, leftoverblock, 0, ebsize, s + (size_t)j * c.blocksize, blk, tmp);
        if (cb == 0 || (cb > 0 && ntbytes + cb > c.destsize)) { ntbytes = 0; break; }
        if (cb > 0) memcpy(d + ntbytes, blk, (size_t)cb);
      } else {
        cb = orc_block_c(&c, bsize, leftoverblock, ntbytes, c.destsize, s + (size_t)j * c.blocksize,
                         d + ntbytes, tmp);
        if (cb == 0) { ntbytes = 0; break; }
      }
      if (cb < 0) { ntbytes = cb; break; }
      ntbytes += cb;
    }
    if (ntbytes < 0) { free(tmp); return -1; }
    if (ntbytes == 0 && !(c.flags & 2) && c.nbytes + ORC_MAX_OVERHEAD <= c.destsize) {
      c.flags |= 2; d[2] = (uint8_t)c.flags; ntbytes = 16;
      continue;
    }
    break;
  }
  free(tmp);
  sti32(d + 12, ntbytes);
  return ntbytes;
}

typedef int (*orc_dfunc)(const void*, int, void*, int);
static int orc_lz4_d(const void* in, int cl, void* out, int maxout) {
  return orc_lz4_decompress_safe((const char*)in, (char*)out, cl, maxout);
}

/* blosc.c:725-800 blosc_d.  tmp must hold bsize bytes. */
static int orc_block_d(int flags, int ts, int32_t compressedsize, orc_dfunc dfunc, int32_t bsize,
                       int leftoverblock, const uint8_t* base, int32_t src_offset, uint8_t* dest,
                       uint8_t* tmp) {
  int dont_split = (flags & 0x10) >> 4;
  int doshuffle = (flags & 1) && ts > 1;
  int dobitshuffle = (flags & 4) && bsize >= ts;
  uint8_t* o = (doshuffle || dobitshuffle) ? tmp : dest;
  int32_t nsplits, neblock, j, ntbytes = 0, cbytes, nb;
  nsplits = (!dont_split && ts <= ORC_MAX_SPLITS && bsize / ts >= ORC_MIN_BUFFERSIZE && !leftoverblock) ? ts : 1;
  neblock = bsize / nsplits;
  for (j = 0; j < nsplits; j++) {
    if (src_offset < 0 || (int64_t)src_offset > (int64_t)compressedsize - 4) return -1;
    cbytes = ldi32(base + src_offset);
    src_offset += 4;
    if (cbytes < 0 || cbytes > compressedsize - src_offset) return -1;
    if (cbytes == neblock) { memcpy(o, base + src_offset, (size_t)neblock); nb = neblock; }
    else {
      nb = dfunc(base + src_offset, cbytes, o, neblock);
      if (nb != neblock) return -2;
    }
    src_offset += cbytes; o += nb; ntbytes += nb;
  }
  if (doshuffle) orc_unshuffle((size_t)ts, (size_t)bsize, tmp, dest);
  else if (dobitshuffle) orc_bitunshuffle((size_t)ts, (size_t)bsize, tmp, dest);
  return ntbytes;
}

static int orc_pick_dfunc(int flags, int versionlz, orc_dfunc* f) {  /* blosc.c:525-574 (LZ4-only build) */
  int fmt = (flags & 0xe0) >> 5;
  if (fmt == 0) { if (versionlz != 1) return -9; *f = orc_blosclz_decompress; return 0; }
  if (fmt == 1) { if (versionlz != 1) return -9; *f = orc_lz4_d; return 0; }
  return -5;
}

int orc_decompress_ctx(const void* src, void* dest, size_t destsize, int numinternalthreads) {
  const uint8_t* s = (const uint8_t*)src;
  uint8_t* d = (uint8_t*)dest;
  int version = s[0], versionlz = s[1], flags = s[2], ts = s[3];
  int32_t nbytes = ldi32(s + 4), blocksize = ldi32(s + 8), cbytes = ldi32(s + 12);
  int32_t nblocks, leftover, j, ntbytes = 0;
  orc_dfunc dfunc = NULL;
  uint8_t* tmp;
  (void)numinternalthreads;
  if (nbytes == 0) return 0;                                    /* blosc.c:1463-1466 */
  if (blocksize <= 0 || (size_t)blocksize > destsize || blocksize > ORC_MAX_BLOCKSIZE || ts <= 0) return -1;
  if (version != 2) return -1;
  if (flags & 0x08) return -1;
  nblocks = nbytes / blocksize; leftover = nbytes % blocksize;
  if (leftover > 0) nblocks++;
  if (nbytes > (int32_t)destsize) return -1;
  if (flags & 2) { if (nbytes + 16 != cbytes) return -1; }
  else {
    int rc = orc_pick_dfunc(flags, versionlz, &dfunc);
    if (rc) return rc;
    if (nblocks > (cbytes - 16) / 4) return -1;
  }
  tmp = (uint8_t*)malloc((size_t)blocksize + 16);
  if (!tmp) return -1;
  for (j = 0; j < nblocks; j++) {
    int32_t bsize = blocksize, cb;
    int leftoverblock = 0;
    if (j == nblocks - 1 && leftover > 0) { bsize = leftover; leftoverblock = 1; }
    if (flags & 2) { memcpy(d + (size_t)j * blocksize, s + 16 + (size_t)j * blocksize, (size_t)bsize); cb = bsize; }
    else cb = orc_block_d(flags, ts, cbytes, dfunc, bsize, leftoverblock, s, ldi32(s + 16 + 4 * j),
                          d + (size_t)j * blocksize, tmp);
    if (cb < 0) { free(tmp); return -1; }
    ntbytes += cb;
  }
  free(tmp);
  return ntbytes;
}

int orc_getitem(const void* src, int start, int nitems, void* dest) {
  const uint8_t* s = (const uint8_t*)src;
  uint8_t* d = (uint8_t*)dest;
  int version = s[0], versionlz = s[1], flags = s[2], ts = s[3];
  int32_t nbytes = ldi32(s + 4), blocksize = ldi32(s + 8), cbytes = ldi32(s + 12);
  int32_t nblocks, leftover, j, ntbytes = 0;
  int stop = start + nitems;
  orc_dfunc dfunc = NULL;
  uint8_t *tmp, *tmp2;
  if (version != 2) return -9;                                  /* blosc.c:1603-1604 */
  if (blocksize <= 0 || blocksize > nbytes || blocksize > ORC_MAX_BLOCKSIZE || ts <= 0) return -1;
  nblocks = nbytes / blocksize; leftover = nbytes % blocksize;
  if (leftover > 0) nblocks++;
  if (flags & 2) { if (nbytes + 16 != cbytes) return -1; }
  else {
    int rc = orc_pick_dfunc(flags, versionlz, &dfunc);
    if (rc) return rc;
    if (nblocks >= (cbytes - 16) / 4) return -1;                /* :1630 (>=, unlike decompress) */
  }
  if (start < 0 || start * ts > nbytes) return -1;              /* :1645-1653 */
  if (stop < 0 || stop * ts > nbytes) return -1;
  tmp = (uint8_t*)malloc(2 * (size_t)blocksize + 32);
  if (!tmp) return -1;
  tmp2 = tmp + blocksize + 16;
  for (j = 0; j < nblocks; j++) {
    int32_t bsize = blocksize, startb, stopb, cb;
    int leftoverblock = 0;
    if (j == nblocks - 1 && leftover > 0) { bsize = leftover; leftoverblock = 1; }
    startb = start * ts - j * blocksize;
    stopb = stop * ts - j * blocksize;
    if (startb >= blocksize || stopb <= 0) continue;
    if (startb < 0) startb = 0;
    if (stopb > blocksize) stopb = blocksize;
    if (flags & 2) memcpy(d + ntbytes, s + 16 + (size_t)j * blocksize + startb, (size_t)(stopb - startb));
    else {
      cb = orc_block_d(flags, ts, cbytes, dfunc, bsize, leftoverblock, s, ldi32(s + 16 + 4 * j), tmp2, tmp);
      if (cb < 0) { ntbytes = cb; break; }
      memcpy(d + ntbytes, tmp2 + startb, (size_t)(stopb - startb));
    }
    ntbytes += stopb - startb;
  }
  free(tmp);
  return ntbytes;
}

/*
 * dev_blosclz.cuh -- BloscLZ codec, one warp per stream, sm_100a.
 *
 * Encoder: bit-exact replay of blosclz_compress (reference blosc/blosclz.c:421-613)
 * including its entropy probe get_cratio (:318-418).  BloscLZ visits EVERY position
 * (a miss costs one literal and advances by one), so a round examines the 32
 * consecutive positions ip..ip+31: each lane hashes its position, resolves the table
 * state it would observe (the table from earlier rounds, overridden by the nearest
 * lower lane with the same hash), and -- because the reference accepts a candidate
 * only if the match is long enough (len >= minlen, and > 5 for far matches,
 * blosclz.c:535) -- compares up to 12 bytes to take exactly that decision.  The first
 * accepting lane f yields f literals + one match; positions up to f are committed to
 * the table.  The result is byte-identical to the serial encoder.
 *
 * Decoder: blosclz_decompress (blosclz.c:679-789) with warp-wide copies.
 */
#pragma once
#include "dev_common.cuh"

#define BLZ_MAX_COPY 32
#define BLZ_MAX_DISTANCE 8191                      /* blosclz.c:43 */
#define BLZ_MAX_FARDISTANCE (65535 + 8191 - 1)     /* blosclz.c:44 */
#define BLZ_PROBE_TABLE_BYTES 8192                 /* 2^12 x u16, blosclz.c:321-322 */

/* Hash-table layouts.  blosclz_compress uses 2^hashlog x u32 (64 KiB at clevel >= 3), which would
 * limit an SM (228 KiB of shared memory) to three resident streams.  For streams of at most 128 KiB (every split Blosc
 * produces with its default block sizes) positions fit in 17 bits: 16 low bits in a u16 array plus
 * one bit in a bitmap = 34 KiB, i.e. six streams per SM.  Same contents, same replacement policy. */
struct BlzTab32 {
  enum { PACKED = 0 };
  u32* t;
  DEV int get(u32 h) const { return (int)t[h]; }
  DEV void put(u32 h, int pos) const { t[h] = (u32)pos; }
};
struct BlzTab16 {                              /* the entropy probe's 2^12 x u16 table (blosclz.c:321-322) */
  enum { PACKED = 0 };
  u16* t;
  DEV int get(u32 h) const { return (int)t[h]; }
  DEV void put(u32 h, int pos) const { t[h] = (u16)pos; }
};
struct BlzTab17 {
  enum { PACKED = 1 };
  u16* lo;
  u32* hi;
  DEV int get(u32 h) const { return (int)lo[h] | (int)(((hi[h >> 5] >> (h & 31u)) & 1u) << 16); }
  DEV void put(u32 h, int pos) const {
    lo[h] = (u16)pos;
    const u32 m = 1u << (h & 31u);
    if (pos & 0x10000) atomicOr(&hi[h >> 5], m); else atomicAnd(&hi[h >> 5], ~m);
  }
};
#define BLZ_TAB17_BYTES (32768 + 2048)
#define BLZ_TAB17_MAXLEN 131072

/* branch ids of the encoder (blz_encode_warp, blz_search_round, blz_probe_one, blz_probe_warp); emulator builds count
 * them so that tests can tell which path a stream reached */
enum {
  /* entropy probe */
  BLZE_H_PROBE_BELOW, BLZE_H_PROBE_EQUAL, BLZE_H_PROBE_ABOVE,   /* cratio below / equal to / above the clevel's threshold */
  BLZE_H_PROBE_EXT,                          /* the probe's own match extension (m >= 12) */
  BLZE_H_SHIFT3_NOSPLIT, BLZE_H_SHIFT3_LOWRATIO, BLZE_H_SHIFT4,   /* ipshift / minlen 3: split_block 0 / cratio < 4; else 4 */
  /* refusals */
  BLZE_H_REF_SHORT, BLZE_H_REF_MAXOUT,       /* length < 16 / maxout < 66 */
  /* tables */
  BLZE_H_TAB_HL12, BLZE_H_TAB_HL13, BLZE_H_TAB_HL14, BLZE_H_TAB_17, BLZE_H_TAB_32,
  BLZE_H_TAB17_HI,                           /* a match whose candidate is at position >= 65536 (bit 16 of BlzTab17) */
  /* search round */
  BLZE_H_R_LANE0, BLZE_H_R_LANE31, BLZE_H_R_NONE,   /* the accepting lane is 0 / 31 / none (32 literals) */
  BLZE_H_R_FWD,                              /* the accepting lane's candidate comes from a lower lane with its hash */
  BLZE_H_R_PARTIAL,                          /* fewer than 32 valid lanes (ip_limit) */
  BLZE_H_R_MINLEN3, BLZE_H_R_BELOW3, BLZE_H_R_MINLEN4, BLZE_H_R_BELOW4,   /* len == minlen (taken) / minlen - 1, per ipshift */
  BLZE_H_EXT_MISMATCH, BLZE_H_EXT_BOUND,     /* m == 12, extended to a mismatch / to ip_bound */
  /* distance rules (search round and blz_probe_one) */
  BLZE_H_FAR5, BLZE_H_FAR6,                  /* equal bytes at a far distance, len 5 (refused) / 6 (taken) */
  BLZE_H_MAXFAR_M1, BLZE_H_MAXFAR,           /* equal bytes at distance MAX_FARDISTANCE - 1 (taken) / MAX_FARDISTANCE (refused) */
  /* blz_probe_one after a match */
  BLZE_H_P1_HIT, BLZE_H_P1_DIST, BLZE_H_P1_BYTES, BLZE_H_P1_LEN,   /* a hit; misses: distance, bytes, length / far rule */
  /* emission */
  BLZE_H_NEAR8190, BLZE_H_FAR8191,           /* biased distance 8190 (the farthest near) / 8191 (the nearest far) */
  BLZE_H_SHORT_NEAR, BLZE_H_SHORT_FAR,
  BLZE_H_LONG_NEAR0, BLZE_H_LONG_NEAR1, BLZE_H_LONG_NEAR2,   /* MATCH_LONG with zero / one / two 255 bytes */
  BLZE_H_LONG_FAR0, BLZE_H_LONG_FAR1, BLZE_H_LONG_FAR2,
  BLZE_H_COPY0,                              /* a match right after a match: op-- */
  BLZE_H_LIT_CROSS,                          /* a literal run that crosses a 32-byte control boundary */
  BLZE_H_L9_STORE,                           /* clevel 9: the second table store */
  /* BLZ_LIMIT: the check that refused the stream */
  BLZE_H_LIM_LIT, BLZE_H_LIM_SHORT, BLZE_H_LIM_LONG, BLZE_H_LIM_CTRL, BLZE_H_LIM_LEFT,
  BLZE_NHIT
};
#ifdef SIMT_EMU
static long long g_blze_hit[BLZE_NHIT + 1];      /* [BLZE_NHIT]: "none of these", not counted */
#define BLZE_HIT(id) do { if (lane_id() == 0) g_blze_hit[id]++; } while (0)         /* warp-uniform branch */
#define BLZE_HITL(id, c) do { if (c) g_blze_hit[id]++; } while (0)                /* per lane */
#else
#define BLZE_HIT(id) do {} while (0)
#define BLZE_HITL(id, c) do {} while (0)
#endif

DEV u32 blz_hash(u32 seq, u32 hashlog) { return (seq * 2654435761u) >> (32u - hashlog); }   /* blosclz.c:58-60 */

/* min(p+1, bound) with p the first position >= start where b[p] != b[p-dist]
 * (what get_run_or_match returns, blosclz.c:117-243). */
DEV int blz_match_end_warp(const u8* __restrict__ b, int start, int dist, int bound) {
  const int p = start + warp_count_match(b, start, start - dist, bound);
  return p < bound ? p + 1 : bound;
}

/* One search round shared by the probe and the encoder.  Examines positions
 * ip .. ip+31 (those < ip_limit).  Returns the first accepting lane (32 if none),
 * the number of valid lanes in *nvalid, and for the accepting lane its candidate and
 * its capped match length (4..12) in *cand_f / *m_f.  Commits table entries. */
template <typename Tab, bool FARRULE>
DEV int blz_search_round(const u8* __restrict__ b, int ip, int ip_limit, const Tab tab, u32 hashlog,
                         int ipshift, int minlen, int* nvalid, int* cand_f, int* m_f) {
  const int lane = lane_id();
  const int pos = ip + lane;
  const bool valid = pos < ip_limit;
  u32 seq = 0, h = 0x80000000u | (u32)lane;
  if (valid) { seq = ld_u32(b + pos); h = blz_hash(seq, hashlog); }
  const unsigned vmask = __ballot_sync(FULLMASK, valid);
  const unsigned peers = __match_any_sync(FULLMASK, h);
  const unsigned lower = peers & ((1u << lane) - 1u);
  int cand = 0, m = 0;
  bool acc = false;
  if (valid) {
    cand = lower ? ip + (31 - __clz((int)lower)) : tab.get(h);
    const u32 dist = (u32)(pos - cand);                                    /* blosclz.c:501 */
    if (dist != 0 && dist < BLZ_MAX_FARDISTANCE && ld_u32(b + cand) == seq) {   /* :506,:512 */
      const u32 x1 = ld_u32(b + pos + 4) ^ ld_u32(b + cand + 4);
      if (x1) m = 4 + eq_bytes32(x1);
      else m = 8 + eq_bytes32(ld_u32(b + pos + 8) ^ ld_u32(b + cand + 8));
      /* m equal bytes (capped at 12) => match end = pos+m+1 => len = m+1-ipshift (:527-532) */
      const int len = m + 1 - ipshift;
      const bool far = FARRULE && (dist - 1u >= BLZ_MAX_DISTANCE);
      acc = m >= 12 || (len >= minlen && !(len <= 5 && far));               /* :535 */
      if (FARRULE) {
        BLZE_HITL(ipshift == 3 ? BLZE_H_R_MINLEN3 : BLZE_H_R_MINLEN4, m < 12 && len == minlen && !far);
        BLZE_HITL(ipshift == 3 ? BLZE_H_R_BELOW3 : BLZE_H_R_BELOW4, m < 12 && len == minlen - 1 && !far);
        BLZE_HITL(len == 5 ? BLZE_H_FAR5 : BLZE_H_FAR6, far && m < 12 && (len == 5 || len == 6) && len >= minlen);
        BLZE_HITL(BLZE_H_MAXFAR_M1, dist == BLZ_MAX_FARDISTANCE - 1);
      }
    }
    if (FARRULE) BLZE_HITL(BLZE_H_MAXFAR, dist == BLZ_MAX_FARDISTANCE && ld_u32(b + cand) == seq);
  }
  const unsigned found = __ballot_sync(FULLMASK, acc);
  const int nv = __popc(vmask);
  const int f = found ? __ffs((int)found) - 1 : 32;
  const int last = f < nv - 1 ? f : nv - 1;
  __syncwarp();                              /* all lookups done before any commit */
  if (valid && lane <= last) {
    const unsigned le = last >= 31 ? FULLMASK : ((1u << (last + 1)) - 1u);
    if ((((peers & le) >> lane) >> 1) == 0) tab.put(h, pos);              /* :504, last writer per hash */
  }
  __syncwarp();
  *nvalid = nv;
  if (FARRULE) {
    BLZE_HIT(f == 0 ? BLZE_H_R_LANE0 : f == 31 ? BLZE_H_R_LANE31 : f == 32 && nv == 32 ? BLZE_H_R_NONE : BLZE_NHIT);
    if (nv < 32) BLZE_HIT(BLZE_H_R_PARTIAL);
    BLZE_HITL(BLZE_H_R_FWD, lane == f && lower != 0);
  }
  if (found) {
    *cand_f = __shfl_sync(FULLMASK, cand, f);
    *m_f = __shfl_sync(FULLMASK, m, f);
  }
  return f;
}

/* The same step for ONE position, warp-uniform (all lanes compute the same values and do the
 * same table store): used right after a match, where the next position very often matches
 * again (chains of short matches dominate shuffled data) and a 32-wide round would be wasted. */
template <typename Tab, bool FARRULE>
DEV int blz_probe_one(const u8* __restrict__ b, int pos, const Tab tab, u32 hashlog, int ipshift, int minlen,
                      int* cand_f, int* m_f) {
  const u32 seq = ld_u32(b + pos);
  const u32 h = blz_hash(seq, hashlog);
  const int cand = tab.get(h);
  __syncwarp();                              /* all lanes have read the old entry */
  if (lane_id() == 0) tab.put(h, pos);
  __syncwarp();                              /* ordered before lane 0's later inserts and everybody's next lookups */
  const u32 dist = (u32)(pos - cand);
  if (FARRULE) BLZE_HIT(dist == BLZ_MAX_FARDISTANCE && ld_u32(b + cand) == seq ? BLZE_H_MAXFAR : BLZE_NHIT);
  if (dist == 0 || dist >= BLZ_MAX_FARDISTANCE) { BLZE_HIT(BLZE_H_P1_DIST); return 32; }
  if (ld_u32(b + cand) != seq) { BLZE_HIT(BLZE_H_P1_BYTES); return 32; }
  int m;
  const u32 x1 = ld_u32(b + pos + 4) ^ ld_u32(b + cand + 4);
  if (x1) m = 4 + eq_bytes32(x1);
  else m = 8 + eq_bytes32(ld_u32(b + pos + 8) ^ ld_u32(b + cand + 8));
  const int len = m + 1 - ipshift;
  const bool far = FARRULE && (dist - 1u >= BLZ_MAX_DISTANCE);
  if (FARRULE) {
    BLZE_HIT(far && m < 12 && len >= minlen && (len == 5 || len == 6) ? (len == 5 ? BLZE_H_FAR5 : BLZE_H_FAR6) : BLZE_NHIT);
    BLZE_HIT(dist == BLZ_MAX_FARDISTANCE - 1 ? BLZE_H_MAXFAR_M1 : BLZE_NHIT);
  }
  if (!(m >= 12 || (len >= minlen && !(len <= 5 && far)))) { BLZE_HIT(BLZE_H_P1_LEN); return 32; }
  BLZE_HIT(BLZE_H_P1_HIT);
  *cand_f = cand; *m_f = m;
  return 0;
}

/* get_cratio (blosclz.c:318-418) on the probe window b[0..maxlen).  `tabmem` is
 * BLZ_PROBE_TABLE_BYTES of warp-private shared memory. */
DEV double blz_probe_warp(const u8* __restrict__ b, int maxlen, void* tabmem) {
  const int lane = lane_id();
  BlzTab16 tab;
  tab.t = (u16*)tabmem;
  for (int i = lane; i < BLZ_PROBE_TABLE_BYTES / 4; i += 32) ((u32*)tabmem)[i] = 0;
  __syncwarp();
  const int limit = maxlen > 4096 ? 4096 : maxlen;
  const int ip_bound = limit - 1, ip_limit = limit - 12;
  int ip = 0, oc = 5, copy = 4;
  while (ip < ip_limit) {
    int nvalid, cand, m;
    const int f = blz_search_round<BlzTab16, false>(b, ip, ip_limit, tab, 12, 3, 3, &nvalid, &cand, &m);
    const int nlit = f < 32 ? f : nvalid;
    oc += nlit + ((copy + nlit) >> 5);                       /* LITERAL2, :258-266 */
    copy = (copy + nlit) & 31;
    ip += nlit;
    if (f == 32) continue;
    const int anchor = ip, dist = anchor - cand;
    if (m >= 12) BLZE_HIT(BLZE_H_PROBE_EXT);
    const int e = m < 12 ? anchor + m + 1 : blz_match_end_warp(b, anchor + 12, dist, ip_bound);
    ip = e - 3;
    const int len = ip - anchor;
    if (!copy) oc--;                                         /* :386-390 */
    copy = 0;
    if (len >= 7) oc += (len - 7) / 255 + 1;
    oc += (dist - 1 < BLZ_MAX_DISTANCE) ? 2 : 4;
    if (lane == 0) tab.put(blz_hash(ld_u32(b + ip), 12), ip);     /* :407-411 */
    __syncwarp();
    ip += 2;
    oc++;
  }
  return (double)ip / (double)oc;
}

/* blosclz_compress for one stream.  Returns the compressed size or 0 (not
 * compressible / does not fit in maxout).  `tabmem`: (4 << hashlog) bytes, at least
 * BLZ_PROBE_TABLE_BYTES, warp-private shared memory. */
template <typename Tab>
DEV int blz_encode_main(const int clevel, const u8* __restrict__ b, const int length, u8* __restrict__ out,
                        const int maxout, const int ipshift, const int minlen, const u32 hashlog, const Tab tab,
                        int* need_out);

DEV int blz_encode_warp(const int clevel, const u8* __restrict__ b, const int length, u8* __restrict__ out,
                        const int maxout, const int split_block, void* tabmem, int table_bytes, int* need_out) {
  const int lane = lane_id();
  const int maxlen = length / 4, shift = length - maxlen;
  const double cratio = blz_probe_warp(b + shift, maxlen, tabmem);          /* :425-430 */
  double thr;
  switch (clevel) {                                                          /* :432 */
    case 0: thr = 0; break;
    case 1: thr = 2; break;
    case 2: thr = 1.5; break;
    case 7: thr = 1.15; break;
    case 8: thr = 1.1; break;
    case 9: thr = 1.0; break;
    default: thr = 1.2; break;
  }
  BLZE_HIT(cratio < thr ? BLZE_H_PROBE_BELOW : cratio == thr ? BLZE_H_PROBE_EQUAL : BLZE_H_PROBE_ABOVE);
  if (cratio < thr) return 0;
  int ipshift = 4, minlen = 4;
  if (!split_block || cratio < 4) { ipshift = 3; minlen = 3; }               /* :445-457 */
  BLZE_HIT(!split_block ? BLZE_H_SHIFT3_NOSPLIT : cratio < 4 ? BLZE_H_SHIFT3_LOWRATIO : BLZE_H_SHIFT4);
  const u32 hashlog = clevel == 1 ? 12u : (clevel == 2 ? 13u : 14u);         /* :459-461 */
  if (length < 16 || maxout < 66) { BLZE_HIT(length < 16 ? BLZE_H_REF_SHORT : BLZE_H_REF_MAXOUT); return 0; }   /* :473-475 */
  BLZE_HIT(BLZE_H_TAB_HL12 + (hashlog - 12));

  __syncwarp();
  if (hashlog == 14 && table_bytes < 65536) {                               /* packed 17-bit table (host guarantees length <= 128 KiB) */
    for (int i = lane; i < BLZ_TAB17_BYTES / 4; i += 32) ((u32*)tabmem)[i] = 0;
    __syncwarp();
    BLZE_HIT(BLZE_H_TAB_17);
    BlzTab17 t;
    t.lo = (u16*)tabmem;
    t.hi = (u32*)((u8*)tabmem + 32768);
    return blz_encode_main<BlzTab17>(clevel, b, length, out, maxout, ipshift, minlen, hashlog, t, need_out);
  }
  for (int i = lane; i < (1 << hashlog); i += 32) ((u32*)tabmem)[i] = 0;
  __syncwarp();
  if (hashlog == 14) BLZE_HIT(BLZE_H_TAB_32);
  BlzTab32 t;
  t.t = (u32*)tabmem;
  return blz_encode_main<BlzTab32>(clevel, b, length, out, maxout, ipshift, minlen, hashlog, t, need_out);
}

template <typename Tab>
DEV int blz_encode_main(const int clevel, const u8* __restrict__ b, const int length, u8* __restrict__ out,
                        const int maxout, const int ipshift, const int minlen, const u32 hashlog, const Tab tab,
                        int* need_out) {
  const int lane = lane_id();
  const int ip_bound = length - 1, ip_limit = length - 12, op_limit = maxout;
  int ip = 4, op = 5, copy = 4;
  int need = 66;                                                            /* :473-475: maxout < 66 is refused */
#define BLZ_LIMIT(v, site) do { const int v_ = (v); if (v_ > need) need = v_; if (v_ > op_limit) { BLZE_HIT(site); return 0; } } while (0)
  if (lane == 0) { out[0] = BLZ_MAX_COPY - 1; out[1] = b[0]; out[2] = b[1]; out[3] = b[2]; out[4] = b[3]; }   /* :481-487 */

  bool post = false;                                                         /* a match was just emitted */
  while (ip < ip_limit) {
    int nvalid = 1, cand = 0, m = 0, f;
    if (post) f = blz_probe_one<Tab, true>(b, ip, tab, hashlog, ipshift, minlen, &cand, &m);
    else f = blz_search_round<Tab, true>(b, ip, ip_limit, tab, hashlog, ipshift, minlen, &nvalid, &cand, &m);
    post = f < 32;
    const int nlit = f < 32 ? f : nvalid;
    if (nlit > 0) {                                                          /* LITERAL x nlit, :246-256 */
      BLZ_LIMIT(op + (nlit - 1) + ((copy + nlit - 1) >> 5) + 2, BLZE_H_LIM_LIT);
      if ((copy + nlit) >> 5) BLZE_HIT(BLZE_H_LIT_CROSS);
      if (lane < nlit) {
        const int o = op + lane + ((copy + lane) >> 5);
        out[o] = b[ip + lane];
        if (((copy + lane + 1) & 31) == 0) out[o + 1] = BLZ_MAX_COPY - 1;
      }
      op += nlit + ((copy + nlit) >> 5);
      copy = (copy + nlit) & 31;
      ip += nlit;
      __syncwarp();            /* a lane may have written the control byte that lane 0 patches below */
    }
    if (f == 32) continue;

    const int anchor = ip;
    u32 distance = (u32)(anchor - cand) - 1u;                                /* biased, :524 */
    const int e = m < 12 ? anchor + m + 1 : blz_match_end_warp(b, anchor + 12, (int)distance + 1, ip_bound);
    if (m >= 12) BLZE_HIT(e < ip_bound ? BLZE_H_EXT_MISMATCH : BLZE_H_EXT_BOUND);
    if (Tab::PACKED && cand >= 65536) BLZE_HIT(BLZE_H_TAB17_HI);
    BLZE_HIT(distance == 8190 ? BLZE_H_NEAR8190 : distance == 8191 ? BLZE_H_FAR8191 : BLZE_NHIT);
    ip = e - ipshift;                                                        /* :530 */
    u32 len = (u32)(ip - anchor);

    if (copy) { if (lane == 0) out[op - copy - 1] = (u8)(copy - 1); }        /* :541-546 */
    else { BLZE_HIT(BLZE_H_COPY0); op--; }
    copy = 0;
    const bool far = distance >= BLZ_MAX_DISTANCE;
    if (far) distance -= BLZ_MAX_DISTANCE;                                   /* :559 */
    if (len < 7) {                                                           /* MATCH_SHORT[_FAR] */
      BLZE_HIT(far ? BLZE_H_SHORT_FAR : BLZE_H_SHORT_NEAR);
      BLZ_LIMIT(op + (far ? 4 : 2), BLZE_H_LIM_SHORT);
      if (lane == 0) {
        if (!far) { out[op] = (u8)((len << 5) + (distance >> 8)); out[op + 1] = (u8)(distance & 255); }
        else { out[op] = (u8)((len << 5) + 31); out[op + 1] = 255; out[op + 2] = (u8)(distance >> 8); out[op + 3] = (u8)(distance & 255); }
      }
      op += far ? 4 : 2;
    } else {                                                                 /* MATCH_LONG[_FAR] */
      len -= 7;
      const int nff = (int)(len / 255);
      BLZE_HIT((far ? BLZE_H_LONG_FAR0 : BLZE_H_LONG_NEAR0) + (nff < 2 ? nff : 2));
      BLZ_LIMIT(op + 1 + nff + (far ? 4 : 2), BLZE_H_LIM_LONG);
      if (lane == 0) out[op] = (u8)((7u << 5) + (far ? 31u : (distance >> 8)));
      op++;
      warp_fill_bytes(out + op, nff, 255);
      op += nff;
      if (lane == 0) {
        out[op] = (u8)(len - (u32)nff * 255u);
        if (!far) out[op + 1] = (u8)(distance & 255);
        else { out[op + 1] = 255; out[op + 2] = (u8)(distance >> 8); out[op + 3] = (u8)(distance & 255); }
      }
      op += far ? 4 : 2;
    }
    /* update the hash at match boundary (:567-580) */
    u32 seq = ld_u32(b + ip);
    if (lane == 0) {
      tab.put(blz_hash(seq, hashlog), ip);
      if (clevel == 9) { BLZE_HIT(BLZE_H_L9_STORE); seq >>= 8; tab.put(blz_hash(seq, hashlog), ip + 1); }
    }
    __syncwarp();
    ip += 2;
    BLZ_LIMIT(op + 1, BLZE_H_LIM_CTRL);                                      /* :582-586 */
    if (lane == 0) out[op] = BLZ_MAX_COPY - 1;
    op++;
  }

  /* left-over as literal copy (:589-598) */
  while (ip <= ip_bound) {
    int nlit = ip_bound - ip + 1;
    if (nlit > 32) nlit = 32;
    BLZ_LIMIT(op + (nlit - 1) + ((copy + nlit - 1) >> 5) + 2, BLZE_H_LIM_LEFT);
    if (lane < nlit) {
      const int o = op + lane + ((copy + lane) >> 5);
      out[o] = b[ip + lane];
      if (((copy + lane + 1) & 31) == 0) out[o + 1] = BLZ_MAX_COPY - 1;
    }
    op += nlit + ((copy + nlit) >> 5);
    copy = (copy + nlit) & 31;
    ip += nlit;
  }
  __syncwarp();
  if (copy) { if (lane == 0) out[op - copy - 1] = (u8)(copy - 1); }          /* :600-604 */
  else op--;
  __syncwarp();
  if (lane == 0) out[0] |= (1u << 5);                                        /* :607 */
  *need_out = need;
  return op;
#undef BLZ_LIMIT
}

/* branch ids of blz_decode_warp; emulator builds count them, and remember the first check that refused a stream */
enum { BLZ_H_DENSE, BLZ_H_DENSE_FEW, BLZ_H_DENSE_BAD, BLZ_H_FAR, BLZ_H_LENEXT, BLZ_H_LITERAL, BLZ_H_DROPPED, BLZ_NHIT };
#ifdef SIMT_EMU
static int g_blz_fail_line = 0;
#define BLZ_FAIL (g_blz_fail_line = g_blz_fail_line ? g_blz_fail_line : __LINE__, 0)
static long long g_blz_hit[BLZ_NHIT];
#define BLZ_HIT(id) do { if (lane_id() == 0) g_blz_hit[id]++; } while (0)
#else
#define BLZ_FAIL 0
#define BLZ_HIT(id) do {} while (0)
#endif

/* blosclz_decompress for one stream (blosclz.c:679-789).  Returns bytes written, 0 on error. */
DEV int blz_decode_warp(const u8* __restrict__ in, const int length, u8* out, const int maxout) {
  int ip = 0, op = 0;
  if (length == 0) return BLZ_FAIL;
  u32 ctrl = in[ip++] & 31u;
  const int lane = lane_id();
  int dense_skip = 0, dense_back = 0;
  for (;;) {
    /* ---- dense path: a chain of short near matches, one per lane ----
     * The byte-planes of shuffled data decode to long chains of 2-byte tokens (ctrl with 3 <= len <= 8, 13-bit
     * distance, no length extension, no far distance: blosclz.c:699-727).  If the token at hand is of that form the
     * next one starts two bytes later, so lane l looks at the bytes ip-1+2l, ip+2l and the leading run of lanes that
     * all see this form are real tokens.  A prefix sum of the lengths places every match; matches whose source lies
     * entirely before the step's first output byte are independent and every lane copies its own. */
    if (dense_skip > 0) dense_skip--;
    else if (ctrl >= 32 && ip + 66 <= length && (long long)op + 256 <= maxout) {
      const u32 c = lane == 0 ? ctrl : (u32)in[ip - 1 + 2 * lane];
      const u32 code = in[ip + 2 * lane];
      const bool simple = c >= 32u && (c >> 5) != 7u && !((c & 31u) == 31u && code == 255u);
      const int len = (int)(c >> 5) + 2;                                   /* (ctrl >> 5) - 1 + 3 */
      const int dist = (int)((c & 31u) << 8) + (int)code + 1;
      const unsigned okm = __ballot_sync(FULLMASK, simple);
      int cnt = okm == FULLMASK ? 32 : __ffs((int)~okm) - 1;
      if (cnt < 4) {                                                       /* not worth a step: straight to the token machine */
        BLZ_HIT(BLZ_H_DENSE_FEW);
        dense_back = dense_back < 32 ? dense_back + dense_back / 2 + 1 : 32;
        dense_skip = dense_back;
        goto serial;
      }
      int incl = lane < cnt ? len : 0;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(FULLMASK, incl, d);
        if (lane >= d) incl += t;
      }
      const int dst = op + incl - len, ref = dst - dist;
      /* a source that touches this step's own output (or is in front of the buffer: the serial code below gives the
       * verdict) ends the run; 8 bytes of slack for the word-wise read */
      const unsigned bad = __ballot_sync(FULLMASK, lane < cnt && (dist < incl + 8 || ref < 0));
      if (bad) cnt = __ffs((int)bad) - 1;
      if (cnt >= 4) {
        const int total = __shfl_sync(FULLMASK, incl, cnt - 1);
        BLZ_HIT(BLZ_H_DENSE);
        if (lane < cnt) {
          const u32 v0 = ld_u32(out + ref), v1 = ld_u32(out + ref + 4);
          u8* o = out + dst;
          o[0] = (u8)v0; o[1] = (u8)(v0 >> 8); o[2] = (u8)(v0 >> 16);
          if (len > 3) o[3] = (u8)(v0 >> 24);
          if (len > 4) o[4] = (u8)v1;
          if (len > 5) o[5] = (u8)(v1 >> 8);
          if (len > 6) o[6] = (u8)(v1 >> 16);
          if (len > 7) o[7] = (u8)(v1 >> 24);
        }
        __syncwarp();
        op += total; ip += 2 * cnt;
        ctrl = in[ip - 1];
        dense_back = 0;
        continue;
      }
      BLZ_HIT(BLZ_H_DENSE_BAD);
      dense_back = dense_back < 32 ? dense_back + dense_back / 2 + 1 : 32;   /* not that kind of data right here: back off */
      dense_skip = dense_back;
    }
  serial:
    if (ctrl >= 32) {
      long long len = (long long)(ctrl >> 5) - 1;
      int ofs = (int)(ctrl & 31u) << 8;
      long long ref = (long long)op - ofs;
      u32 code;
      if (len == 6) {
        BLZ_HIT(BLZ_H_LENEXT);
        do {
          if (ip + 1 >= length) return BLZ_FAIL;               /* length bytes run into the end */
          code = in[ip++];
          len += code;
        } while (code == 255);
      } else if (ip + 1 >= length) return BLZ_FAIL;
      code = in[ip++];
      len += 3;
      ref -= code;
      if (code == 255 && ofs == (31 << 8)) {                  /* 16-bit far distance (:717-726) */
        BLZ_HIT(BLZ_H_FAR);
        if (ip + 1 >= length) return BLZ_FAIL;                 /* no room for the 16-bit distance */
        ofs = (int)in[ip++] << 8;
        ofs += in[ip++];
        ref = (long long)op - ofs - BLZ_MAX_DISTANCE;
      }
      if (op + len > maxout) return BLZ_FAIL;                        /* :728-730 */
      if (ref - 1 < 0) return BLZ_FAIL;                              /* :732-734 */
      if (ip >= length) { BLZ_HIT(BLZ_H_DROPPED); break; }    /* :736 ends without copying */
      ctrl = in[ip++];
      ref--;
      __syncwarp();
      warp_copy_match(out, op, (int)ref, (int)len);
      __syncwarp();
      op += (int)len;
    } else {
      ctrl++;
      BLZ_HIT(BLZ_H_LITERAL);
      if ((long long)op + ctrl > maxout) return BLZ_FAIL;            /* :769-774 */
      if ((long long)ip + ctrl > length) return BLZ_FAIL;
      warp_copy_bytes(out + op, in + ip, (int)ctrl);
      op += (int)ctrl; ip += (int)ctrl;
      if (ip >= length) break;
      ctrl = in[ip++];
    }
  }
  __syncwarp();
  return op;
}

/*
 * dev_lz4.cuh -- LZ4 block codec, one warp per stream, sm_90a.
 *
 * Encoder: bit-exact replay of LZ4_compress_fast's greedy parse
 * (reference: internal-complibs/lz4-1.10.0/lz4.c:930-1338, called from
 * blosc/blosc.c:413-420 with acceleration = 10 - clevel and maxout = neblock, i.e.
 * limitedOutput).  The sequential "probe, skip, probe" search loop (lz4.c:1043-1101)
 * is evaluated 32 probes at a time: lane l computes the position the l-th probe
 * WOULD visit (closed form of the skip schedule), hashes it, and resolves the hash
 * table state it would observe -- the table as left by earlier rounds, overridden by
 * the nearest lower lane with the same hash (__match_any_sync).  The first hitting
 * lane wins, and only probes up to and including it are committed to the table, so
 * the table evolves exactly as in the serial code and the output is byte-identical.
 *
 * Decoder: LZ4_decompress_safe semantics (lz4.c:2022-2445).  Five tiers: a dense path for
 * chains of literal-free sequences (one 3-byte sequence per lane, long matches with one
 * extra length byte taken inline: up to 32 sequences per step, every lane copying its own
 * match), a lone long match that overlaps its own output, a batch path (every lane speculatively parses the sequence that would start at
 * its input byte; the chain of real starts is resolved with one ballot or a short shuffle
 * walk and up to 11 sequences are copied 32 output bytes per instruction), a
 * single-sequence fast path, and the general path with warp-wide literal and
 * period-replicating match copies.  A per-warp shared-memory ring mirrors the last 16 KiB
 * of output so match sources do not wait behind the global stores that produced them.
 * The tier walk (lz4d_walk) is written once and hands the copies of every step to a copy
 * routine: run by the same warp (lz4_decode_warp), or by a second warp that takes them from a
 * queue (lz4_pair_parse, dev_lz4dpair.cuh).
 */
#pragma once
#include "dev_common.cuh"

#define LZ4_MFLIMIT 12
#define LZ4_LASTLITERALS 5
#define LZ4_TABLE_BYTES 16384          /* lz4.h:163,696  LZ4_MEMORY_USAGE 14 */
#define LZ4_TAB17_BYTES (8192 + 512)    /* packed variant of the 4096-entry table: u16 + 1 bit per entry */
#define LZ4_TAB17_MINLEN 65547         /* shorter streams use the 8192-entry byU16 table (lz4.c:710,1389), which cannot shrink */
#define LZ4_TAB17_MAXLEN 131072

template <bool U16>
DEV u32 lz4_hash_at(const u8* __restrict__ s, int pos) {       /* lz4.c:777-806 */
  if (U16) return (ld_u32(s + pos) * 2654435761u) >> (32 - 13);
  const u64 seq = (u64)ld_u32(s + pos) | ((u64)s[pos + 4] << 32);   /* low 5 bytes are all hash5 uses */
  return (u32)(((seq << 24) * 889523592379ull) >> (64 - 12));
}

#define LZ4_SCALAR_PROBES 4     /* probes done one at a time before the 32-wide rounds (must be <= 64) */

/* Offset from the search start of the it-th probe of the skip schedule
 * (lz4.c:1043-1053): steps are 1, then accel + (k >> 6) for k = 0,1,2,... */
DEV long long lz4_probe_offset(int it, int accel) {
  if (it == 0) return 0;
  const long long m = it - 1;
  const long long c = m >> 6;
  return 1 + m * accel + 32 * c * (c - 1) + c * (m - 64 * c);
}

/* Position-based window loads: the stream base is split once into an aligned word pointer
 * (s32) and a byte phase (sal); a window at byte position p then costs one 64-bit address
 * computation (IMAD.WIDE) instead of one per word. */
struct StreamBase {
  const u8* s;
  const u32* s32;
  int sal;
  const uint4* s128;     /* the same stream seen as aligned 16-byte granules */
  int sal16;
};
DEV StreamBase make_stream_base(const u8* s) {
  StreamBase b;
  b.s = s;
  b.s32 = (const u32*)((uintptr_t)s & ~(uintptr_t)3);
  b.sal = (int)((uintptr_t)s & 3u);
  b.s128 = (const uint4*)((uintptr_t)s & ~(uintptr_t)15);
  b.sal16 = (int)((uintptr_t)s & 15u);
  return b;
}
/* 12 bytes at position p as three little-endian words.  GPU: four aligned read-only word loads
 * + funnel shifts; touches the aligned words around [p, p+12), i.e. at most byte p+15 --
 * callers guarantee p+16 <= end of the stream (the emulator build reads exactly 12 bytes). */
DEV void ldp_win12(const StreamBase& sb, int p, u32& b0, u32& b1, u32& b2) {
#ifdef SIMT_EMU
  memcpy(&b0, sb.s + p, 4); memcpy(&b1, sb.s + p + 4, 4); memcpy(&b2, sb.s + p + 8, 4);
#else
  const int q = p + sb.sal;
  const u32* w = sb.s32 + (q >> 2);
  const u32 sh = (u32)(q & 3) * 8u;
  const u32 w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2), w3 = __ldg(w + 3);
  b0 = __funnelshift_r(w0, w1, sh); b1 = __funnelshift_r(w1, w2, sh); b2 = __funnelshift_r(w2, w3, sh);
#endif
}
/* The same in two steps, for loads that are requested long before their bytes are needed:
 * ldp_raw12 only issues the aligned word loads, ldp_take12 aligns them (first use of the data). */
DEV void ldp_raw12(const StreamBase& sb, int p, u32& r0, u32& r1, u32& r2, u32& r3) {
#ifdef SIMT_EMU
  memcpy(&r0, sb.s + p, 4); memcpy(&r1, sb.s + p + 4, 4); memcpy(&r2, sb.s + p + 8, 4); r3 = 0;
#else
  const u32* w = sb.s32 + ((p + sb.sal) >> 2);
  r0 = __ldg(w); r1 = __ldg(w + 1); r2 = __ldg(w + 2); r3 = __ldg(w + 3);
#endif
}
DEV void ldp_take12(const StreamBase& sb, int p, u32 r0, u32 r1, u32 r2, u32 r3, u32& b0, u32& b1, u32& b2) {
#ifdef SIMT_EMU
  (void)sb; (void)p; (void)r3; b0 = r0; b1 = r1; b2 = r2;
#else
  const u32 sh = (u32)((p + sb.sal) & 3) * 8u;
  b0 = __funnelshift_r(r0, r1, sh); b1 = __funnelshift_r(r1, r2, sh); b2 = __funnelshift_r(r2, r3, sh);
#endif
}
/* 8 bytes at position p; touches at most byte p+11 */
DEV void ldp_win8(const StreamBase& sb, int p, u32& b0, u32& b1) {
#ifdef SIMT_EMU
  memcpy(&b0, sb.s + p, 4); memcpy(&b1, sb.s + p + 4, 4);
#else
  const int q = p + sb.sal;
  const u32* w = sb.s32 + (q >> 2);
  const u32 sh = (u32)(q & 3) * 8u;
  const u32 w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2);
  b0 = __funnelshift_r(w0, w1, sh); b1 = __funnelshift_r(w1, w2, sh);
#endif
}

/* 17 bytes at position p (four words + the byte p+16) in two steps, as ldp_raw12 / ldp_take12:
 * ldp_raw20 issues five aligned word loads (touches at most byte p+19), ldp_take17 aligns them. */
DEV void ldp_raw20(const StreamBase& sb, int p, u32 (&r)[5]) {
#ifdef SIMT_EMU
  memcpy(&r[0], sb.s + p, 16); r[4] = sb.s[p + 16];
#else
  const u32* w = sb.s32 + ((p + sb.sal) >> 2);
  r[0] = __ldg(w); r[1] = __ldg(w + 1); r[2] = __ldg(w + 2); r[3] = __ldg(w + 3); r[4] = __ldg(w + 4);
#endif
}
DEV void ldp_take17(const StreamBase& sb, int p, const u32 (&r)[5], u32& a0, u32& a1, u32& a2, u32& a3, u32& a4b) {
#ifdef SIMT_EMU
  (void)sb; (void)p; a0 = r[0]; a1 = r[1]; a2 = r[2]; a3 = r[3]; a4b = r[4] & 0xffu;
#else
  const u32 sh = (u32)((p + sb.sal) & 3) * 8u;
  a0 = __funnelshift_r(r[0], r[1], sh); a1 = __funnelshift_r(r[1], r[2], sh);
  a2 = __funnelshift_r(r[2], r[3], sh); a3 = __funnelshift_r(r[3], r[4], sh);
  a4b = (r[4] >> sh) & 0xffu;
#endif
}
/* The same 17 bytes for a GATHER (every lane its own, unrelated position): two aligned 128-bit
 * loads instead of five 32-bit ones -- a warp-wide gather costs one L1 tag cycle per distinct line
 * and instruction, so the instruction count is what matters -- and a two-level select network that
 * brings the five words that hold the bytes into place.  Touches [p & ~15, +32). */
DEV void ldp_gather17(const StreamBase& sb, int p, u32& c0, u32& c1, u32& c2, u32& c3, u32& c4b) {
#ifdef SIMT_EMU
  memcpy(&c0, sb.s + p, 4); memcpy(&c1, sb.s + p + 4, 4); memcpy(&c2, sb.s + p + 8, 4); memcpy(&c3, sb.s + p + 12, 4);
  c4b = sb.s[p + 16];
#else
  const int q = p + sb.sal16;
  const uint4* w = sb.s128 + (q >> 4);
  const uint4 v0 = __ldg(w), v1 = __ldg(w + 1);
  const bool k1 = (q & 4) != 0, k2 = (q & 8) != 0;
  const u32 sh = (u32)(q & 3) * 8u;
  const u32 t0 = k1 ? v0.y : v0.x, t1 = k1 ? v0.z : v0.y, t2 = k1 ? v0.w : v0.z, t3 = k1 ? v1.x : v0.w;
  const u32 t4 = k1 ? v1.y : v1.x, t5 = k1 ? v1.z : v1.y, t6 = k1 ? v1.w : v1.z;
  const u32 u0 = k2 ? t2 : t0, u1 = k2 ? t3 : t1, u2 = k2 ? t4 : t2, u3 = k2 ? t5 : t3, u4 = k2 ? t6 : t4;
  c0 = __funnelshift_r(u0, u1, sh); c1 = __funnelshift_r(u1, u2, sh);
  c2 = __funnelshift_r(u2, u3, sh); c3 = __funnelshift_r(u3, u4, sh);
  c4b = (u4 >> sh) & 0xffu;
#endif
}

/* L1 prefetch of the line holding byte p of a stream of `end` bytes (no-op past the end) */
DEV void lz4d_prefetch(const u8* base, int p, int end) {
#ifndef SIMT_EMU
  if (p < end) asm volatile("prefetch.global.L1 [%0];" :: "l"(base + p));
#else
  (void)base; (void)p; (void)end;
#endif
}

/* 4 bytes at position p; touches at most byte p+7 */
DEV u32 ldp_win4(const StreamBase& sb, int p) {
#ifdef SIMT_EMU
  u32 b0; memcpy(&b0, sb.s + p, 4); return b0;
#else
  const int q = p + sb.sal;
  const u32* w = sb.s32 + (q >> 2);
  return __funnelshift_r(__ldg(w), __ldg(w + 1), (u32)(q & 3) * 8u);
#endif
}

template <bool U16>
DEV u32 lz4_hash_seq(u32 lo, u32 b4) {                        /* lz4.c:777-806 on bytes already in registers */
  if (U16) return (lo * 2654435761u) >> (32 - 13);
  const u64 seq = (u64)lo | ((u64)(b4 & 0xffu) << 32);
  return (u32)(((seq << 24) * 889523592379ull) >> (64 - 12));
}

/* LZ4_count continuation for matches that outgrow the scalar compares: first round 4 bytes per
 * lane (128 bytes, two loads per lane), only then the 512-bytes-per-round loop.  p > q, `n` =
 * stream length, limit = matchlimit. */
DEV int lz4_count_tail(const StreamBase& sb, const u8* __restrict__ s, int p, int q, int limit, int n) {
  if (p + 136 <= n) {                                           /* p + 128 <= limit and the loads stay inside the stream */
    const int lane = lane_id();
    const u32 x = ldp_win4(sb, p + 4 * lane) ^ ldp_win4(sb, q + 4 * lane);
    const unsigned full = __ballot_sync(FULLMASK, x == 0u);
    if (full != FULLMASK) {
      const int fl = __ffs((int)~full) - 1;
      return fl * 4 + eq_bytes32(__shfl_sync(FULLMASK, x, fl));
    }
    return 128 + warp_count_match(s, p + 128, q + 128, limit);
  }
  return warp_count_match(s, p, q, limit);
}

/* catch-up (lz4.c:1107-1109) of the match at ip with candidate `match`, from `back` bytes on: the length of the
 * run of equal bytes before them, 32 per round, bounded by the anchor and by the start of the stream */
DEV int lz4_catch_up(const u8* __restrict__ s, int ip, int match, int anchor, int back) {
  const int lane = lane_id();
  for (;;) {
    const int a = ip - 1 - back - lane, b = match - 1 - back - lane;
    const bool ok = a >= anchor && b >= 0 && s[a] == s[b];
    const unsigned m = __ballot_sync(FULLMASK, ok);
    const int step = m == FULLMASK ? 32 : __ffs((int)~m) - 1;
    back += step;
    if (step < 32) return back;
  }
}

/* ---- team mode: one CTA of four warps per stream ------------------------------------------------
 * A lone warp spends ~6 cycles per instruction on its dependent chain (ALU latency 4, one issue
 * per 2 cycles and pipe), so on a hard byte-plane the serial LZ4 loop is bound by the NUMBER of
 * instructions one warp has to issue per sequence, not by memory.  In team mode the stream's warp
 * ("walker") keeps only what is inherently serial -- which position the parse lands on next, the
 * table stores, the output -- and three helper warps ("preparers") do the rest ahead of it:
 * for every position of a 32-position tile a preparer computes hash, table lookup, candidate
 * gather, 17-byte compare and packs the verdict {hit, match length, offset} into a shared-memory
 * ring; the walker reads the verdict of the position it lands on with one 8-byte shared load.
 * A verdict carries the candidate it was computed from (`snap`, the table entry the preparer read).
 * It is a pure function of (position, snap): the 4-byte equality, the 65535-distance rule and the
 * 17-byte length depend on nothing else.  The walker makes every table store in serial order, so
 * after its store at ip-2 the live table[h(ip)] is what LZ4_compress_fast would read; when it equals
 * snap the verdict is exact, however old it is, and otherwise (rare) the scalar code probes itself.
 * The parse, the table and the output stay byte-identical to LZ4_compress_fast.
 * Preparation follows stream positions, not chains: tile T (positions 32T .. 32T+31) lives in ring
 * slot T mod LZ4T_TILES and is prepared by preparer T mod 3, which owns the slot (LZ4T_TILES is a
 * multiple of 3), so a slot's entries and ready word are written by one warp in order.  The walker
 * publishes the lowest tile it still reads (`wt`, the tile of ip-2); a preparer skips tiles below it
 * and prepares up to LZ4T_AHEAD tiles past it, then naps.  After each tile it posts the tile number
 * in the slot's ready word.  A chain that starts again after a search or a long match reads tiles
 * that are prepared or in flight, or moves `wt` past them, which re-bases the preparers: nothing is
 * restarted or drained.  Per stream, the walker starts preparer i through barrier GO(i) and, at the end,
 * waits at barrier IDLE(i) until it has stopped (bar.sync / bar.arrive, 64 threads: the walker and
 * preparer i); after the last stream, LZ4T_QUIT and GO(i) end it. */
#ifdef SIMT_EMU
/* x[]: 0 LZ4T_LONG, 1 match of 270+ bytes, 2 re-base, 3 chain start on prepared tiles, 4 chained miss, 5 walker waited for a tile */
static long long g_dbg_lz4t_sessions = 0, g_dbg_lz4t_seqs = 0, g_dbg_lz4t_stale = 0, g_dbg_lz4t_x[6];
/* the search after a chained miss, taken from the verdicts (LZ4T_S_*) */
enum {
  LZ4T_S_HIT0,                             /* + k: a hit at probe k (0..3) */
  LZ4T_S_STALE = 4,                        /* a probe's verdict was computed from another candidate: the scalar probes take over */
  LZ4T_S_MISS4,                            /* all four probes missed: on to the 32-wide rounds */
  LZ4T_S_LIT,                              /* a hit with literals: general emission */
  LZ4T_S_CAPPED,                           /* a hit whose catch-up length is 7+ and more than 7 bytes from the anchor: warp catch-up */
  LZ4T_S_LONG,                             /* a hit whose length field is LZ4T_LONG */
  LZ4T_S_HUGE,                             /* a hit of 270+ bytes with its catch-up: general emission */
  LZ4T_S_N
};
static long long g_dbg_lz4t_s[LZ4T_S_N];
/* the chained windows (LZ4T_W_*): how many, how many elements they committed, and what ended them */
enum {
  LZ4T_W_WINDOWS,
  LZ4T_W_ELEMS,                            /* elements committed (valid, stores made), summed over the windows */
  LZ4T_W_STALE0, LZ4T_W_STALEJ,            /* the first invalid element was element 0 / a later one */
  LZ4T_W_FWD,                              /* an element's lookup was answered by an earlier store of the same window */
  LZ4T_W_CROSS,                            /* h(q_j - 2) == h(q_k) for two different elements j, k of a window */
  LZ4T_W_MISS0, LZ4T_W_MISSJ,              /* a valid miss ended the window at element 0 / a later one */
  LZ4T_W_LONG0, LZ4T_W_LONGJ,              /* a valid LZ4T_LONG ended the window at element 0 / a later one */
  LZ4T_W_HUGE,                             /* ... and its match was 270+ bytes: general emission */
  LZ4T_W_END, LZ4T_W_CAP, LZ4T_W_TILE,     /* the next position is too close to the end / the window is full / past vt */
  LZ4T_W_FULL,                             /* the flush before a window found the output too small */
  LZ4T_W_N
};
static long long g_dbg_lz4t_w[LZ4T_W_N];
#define LZ4T_DBG(x) do { if (lane_id() == 0) (x)++; } while (0)
#define LZ4T_DBGN(x, v) do { if (lane_id() == 0) (x) += (v); } while (0)
#else
#define LZ4T_DBG(x) do {} while (0)
#define LZ4T_DBGN(x, v) do {} while (0)
#endif
#ifndef LZ4T_TILES
#define LZ4T_TILES 12                      /* ring slots of 32 positions; a multiple of 3 (one owner per slot) */
#endif
#ifndef LZ4T_AHEAD
#define LZ4T_AHEAD 8                       /* tiles a preparer may work past `wt`; at most LZ4T_TILES - 1 */
#endif
#ifndef LZ4T_NAP
#define LZ4T_NAP 128                       /* ns a preparer naps when it is LZ4T_AHEAD tiles ahead */
#endif
#define LZ4T_RING (32 * LZ4T_TILES)
#define LZ4T_BAR_IDLE(i) (1 + (i))
#define LZ4T_BAR_GO(i) (4 + (i))
#define LZ4T_QUIT 1
#define LZ4T_STOP 0x7fffffff               /* `wt` at the end of a stream: preparers go to IDLE(i) */
#define LZ4T_END 0xffffffffu               /* snap of a position that was not compared (too close to the end of the
                                            * stream, or the table held no earlier position): no table entry equals it */
#define LZ4T_LONG 13                       /* match-length field: 13 = "13 or more bytes after the first four" */
#define LZ4T_HSHIFT 19                     /* the hash (at most 13 bits) is the top of a verdict's .x */
#define LZ4T_BACKCAP 7                     /* catch-up length field: 7 = "7 or more" */
#define LZ4T_W 16                          /* chained sequences the walker takes per window: two table stores each, one per lane */
static_assert(LZ4T_TILES % 3 == 0 && LZ4T_AHEAD >= 1 && LZ4T_AHEAD < LZ4T_TILES && LZ4T_RING > 15 + 255 + 4, "team ring layout");
static_assert(2 * LZ4T_W <= 32, "window layout");
/* a preparer pulls the bytes this far past its tile into L1 (measured on an H100, power limit 400 and 700 W, on the bench.c planes, typesize 4:
 * encode 4.17 -> 4.08 ms; 4 and 16 KiB ahead into L2 instead: 4.10 and 4.15 ms) */
#define LZ4T_PREFETCH 512

/* Cycle accounting (builds with -DB2_LZ4_CYCLES only, scripts/lz4_cycles.py): the walker and the preparers
 * add the clock64() time of each phase into counters in Lz4Team, and the kernel copies them per stream into
 * g_lz4_cycles.  Without the flag the macros are empty and the kernels compile to the same SASS. */
enum {
  LZ4C_TOTAL,        /* the whole lz4_encode_warp call */
  LZ4C_START,        /* chain start: publishing `wt` until the first tiles of the chain are ready */
  LZ4C_SESSION,      /* rest of a chain, waits included */
  LZ4C_FULLWAIT,     /* of that: walker waiting for the ready word of a tile */
  LZ4C_REPROBE,      /* stale verdict / post-match probe done by the scalar code */
  LZ4C_SEARCH,       /* search after a chain break (scalar probes, 32-wide rounds, catch-up) */
  LZ4C_SESSIONS, LZ4C_SEQS, LZ4C_CHAIN_SEQS,
  LZ4C_PREP_BUSY,    /* preparers, summed over the three: tile allowed .. ready word posted */
  LZ4C_PREP_OWN,     /* of that: load of the tile's own bytes, hash, table read */
  LZ4C_PREP_GATHER,  /* of that: candidate gather and compare */
  LZ4C_PREP_TILES,
  LZ4C_SMID, LZ4C_SUBP,
  LZ4C_STALE,        /* chained positions whose verdict's snap differed from the live table */
  LZ4C_N = 16
};
/* the chained windows and what ended each: a stale element, a valid miss or LZ4T_LONG, the end of the stream,
 * LZ4T_W elements, the next position past the checked tiles */
enum {
  LZ4C_WINDOWS = LZ4C_N, LZ4C_W_STALE, LZ4C_W_MISS, LZ4C_W_LONG, LZ4C_W_END, LZ4C_W_CAP, LZ4C_W_TILE,
  LZ4C_NREC                                /* columns of a stream's record */
};
#ifdef B2_LZ4_CYCLES
#define LZ4C_MAXSTREAMS 16384
__device__ unsigned long long g_lz4_cycles[LZ4C_MAXSTREAMS][LZ4C_NREC];
#define LZ4C_T(t) const long long t = clock64()
#define LZ4C_TW(t) const long long t = TEAM ? clock64() : 0ll     /* in code that encode_kernel shares */
#define LZ4C_ADD(k, v) do { if (lane_id() == 0) atomicAdd(&tm->cyc[k], (unsigned long long)(v)); } while (0)
#define LZ4C_SPAN(k, t) LZ4C_ADD(k, clock64() - (t))
#else
#define LZ4C_T(t) do {} while (0)
#define LZ4C_TW(t) do {} while (0)
#define LZ4C_ADD(k, v) do {} while (0)
#define LZ4C_SPAN(k, t) do {} while (0)
#endif

struct Lz4Team {
  uint2 vd[LZ4T_RING];                     /* .x: bit 0 hit, bits 2..5 length field, bits 8..10 catch-up length (hits
                                            * only), bits 19..31 hash (one shift takes it out); .y snap */
  int rdy[LZ4T_TILES];                     /* ready word of each slot: number + 1 of the tile whose verdicts it holds */
  const u8* s;                             /* current stream */
  int n;
  int u16;                                 /* table flavour of the current stream */
  int wt;                                  /* lowest tile the walker still reads, or LZ4T_STOP */
  int gen;                                 /* streams started by this team (zeroed at launch, with cmd) */
  int cmd;                                 /* LZ4T_QUIT ends the preparers */
  int sub[4];                              /* SM sub-partition of each warp of the CTA */
  int slot;                                /* sub-partition this CTA's walker should run on */
  u32 seen[8192 / 32];                     /* walker: hashes of the stores of the window being checked, one bit each (zero between windows) */
#ifdef B2_LZ4_CYCLES
  unsigned long long cyc[LZ4C_NREC];
#endif
};
#define LZ4T_SMEM_BYTES ((int)sizeof(Lz4Team))

DEV int lz4t_ld_i32(const int* p) { return *(const volatile int*)p; }
DEV void lz4t_st_i32(int* p, int v) { *(volatile int*)p = v; }

template <bool U16>
DEV void lz4_team_prepare_tile(Lz4Team* tm, const void* tabmem, const u8* s, int n, int tile) {
  const int lane = lane_id();
  const int w0 = 32 * tile, p = w0 + lane;
  const int e = (tile % LZ4T_TILES) * 32 + lane;
  if (w0 + 31 + 24 > n) { tm->vd[e] = make_uint2(0u, LZ4T_END); return; }     /* loads below reach byte p+19 (+3) */
  const StreamBase sb = make_stream_base(s);
  u32 r[5], a0, a1, a2, a3, a4, c0, c1, c2, c3, c4;
  LZ4C_T(c_t0);
  ldp_raw20(sb, p, r);
  ldp_take17(sb, p, r, a0, a1, a2, a3, a4);
  const u32 h = lz4_hash_seq<U16>(a0, a1);
  /* racing with the walker's stores (and, at a stream's start, with its clearing of the table) is fine:
   * the walker takes the verdict only if the live entry still equals snap */
  const int snap = U16 ? (int)((const volatile u16*)tabmem)[h] : (int)((const volatile u32*)tabmem)[h];
  u32 vx = h << LZ4T_HSHIFT, sn = LZ4T_END;
  if ((unsigned)snap < (unsigned)p) {                  /* always true for entries the serial code could see here */
    LZ4C_T(c_t1);
    LZ4C_ADD(LZ4C_PREP_OWN, c_t1 - c_t0);
    ldp_gather17(sb, snap, c0, c1, c2, c3, c4);
    const u32 x1 = a1 ^ c1, x2 = a2 ^ c2, x3 = a3 ^ c3;
    u32 m;
    if (x1) m = (u32)(__ffs((int)x1) - 1) >> 3;
    else if (x2) m = 4u + ((u32)(__ffs((int)x2) - 1) >> 3);
    else if (x3) m = 8u + ((u32)(__ffs((int)x3) - 1) >> 3);
    else m = a4 != c4 ? 12u : (u32)LZ4T_LONG;
    const bool hit = (U16 || snap + 65535 >= p) && c0 == a0;
    /* catch-up length (lz4.c:1107-1109 without the anchor bound, which only the walker knows): equal bytes
     * before p and before snap, at most 7 ("7 or more"), never reaching before the start of the stream */
    u32 bk = 0;
    if (hit) {
      if (snap >= 8) {                                 /* p > snap: both windows lie inside the stream */
        u32 p0, p1, q0, q1;
        ldp_win8(sb, p - 8, p0, p1);
        ldp_win8(sb, snap - 8, q0, q1);
        const u32 y1 = p1 ^ q1, z0 = (u32)__clz((int)(p0 ^ q0)) >> 3;   /* equal bytes at the top of each word */
        bk = y1 ? (u32)__clz((int)y1) >> 3 : 4u + (z0 < 3u ? z0 : 3u);
      } else {
        while (bk < (u32)snap && s[p - 1 - (int)bk] == s[snap - 1 - (int)bk]) bk++;
      }
    }
    vx |= (hit ? 1u : 0u) | (m << 2) | (bk << 8);
    sn = (u32)snap;
    LZ4C_SPAN(LZ4C_PREP_GATHER, c_t1);
  }
  tm->vd[e] = make_uint2(vx, sn);
}

/* body of preparer warp i (0..2): per stream, tiles i, i+3, i+6, ... from GO(i) until the walker posts
 * LZ4T_STOP; returns when the walker posts LZ4T_QUIT */
DEV void lz4_team_preparer(Lz4Team* tm, const void* tabmem, int i) {
  for (;;) {
    bar_sync(LZ4T_BAR_GO(i), 64);
    if (lz4t_ld_i32(&tm->cmd) == LZ4T_QUIT) return;
    const u8* s = *(const u8* const volatile*)&tm->s;
    const int n = lz4t_ld_i32(&tm->n), u16 = lz4t_ld_i32(&tm->u16);
    for (int tile = i;; tile += 3) {
      int w;
      for (;;) {                                       /* until the tile may be prepared */
        w = __shfl_sync(FULLMASK, lz4t_ld_i32(&tm->wt), 0);
        if (w == LZ4T_STOP) break;
        if (tile < w) tile = w + (i + 3 - w % 3) % 3;  /* the walker is past it: first own tile from w on */
        if (tile <= w + LZ4T_AHEAD) break;             /* slot of tile - LZ4T_TILES (< w) is no longer read */
        __nanosleep(LZ4T_NAP);
      }
      if (w == LZ4T_STOP) break;
      LZ4C_T(c_go);
      lz4d_prefetch(s, 32 * tile + LZ4T_PREFETCH + lane_id(), n);
      if (u16) lz4_team_prepare_tile<true>(tm, tabmem, s, n, tile);
      else lz4_team_prepare_tile<false>(tm, tabmem, s, n, tile);
      __syncwarp();
      if (lane_id() == 0) { __threadfence_block(); lz4t_st_i32(&tm->rdy[tile % LZ4T_TILES], tile + 1); }
      LZ4C_SPAN(LZ4C_PREP_BUSY, c_go);
      LZ4C_ADD(LZ4C_PREP_TILES, 1);
    }
    __syncwarp();
    bar_arrive(LZ4T_BAR_IDLE(i), 64);
  }
}

/* walker: the chain needs the tiles of ip-2 and ip.  Publishes the tile of ip-2 as `wt` (moving it past
 * the tiles the preparers may have started re-bases them there) and waits for the ready words of the
 * tiles up to that of ip not yet checked (vt = highest tile checked). */
DEV void lz4t_reach(Lz4Team* tm, int ip, int& wt, int& vt) {
  const int lo = (ip - 2) >> 5, hi = ip >> 5;
  if (lo > wt + LZ4T_AHEAD) LZ4T_DBG(g_dbg_lz4t_x[2]);
  if (lo != wt) { wt = lo; lz4t_st_i32(&tm->wt, lo); }
  for (int t = vt + 1 > lo ? vt + 1 : lo; t <= hi; t++) {
    const int* r = &tm->rdy[t % LZ4T_TILES];
    if (lz4t_ld_i32(r) != t + 1) {
      LZ4T_DBG(g_dbg_lz4t_x[5]);
      do { __syncwarp(); } while (__any_sync(FULLMASK, lz4t_ld_i32(r) != t + 1));
    }
  }
  if (hi > vt) vt = hi;
}

/* walker: moves vt over the tiles after it whose ready words are posted already, without waiting, up to
 * wt + LZ4T_AHEAD (a preparer only reuses the slot of a tile below wt) */
DEV void lz4t_extend(Lz4Team* tm, int wt, int& vt) {
  const int t = vt + 1 + lane_id();
  const bool ready = t <= wt + LZ4T_AHEAD && lz4t_ld_i32(&tm->rdy[t % LZ4T_TILES]) == t + 1;
  vt += __ffs((int)~__ballot_sync(FULLMASK, ready)) - 1;
}

/* walker, after a chained miss at `anchor`: the first LZ4_SCALAR_PROBES probes of the search (lz4.c:1043-1101), which
 * starts at anchor + 1, taken from the verdicts.  A probe gets table[h(pos)], puts pos and tests the candidate exactly as
 * the chained step does (without its store at ip-2), so a verdict whose snap equals the live entry is exact here too.
 * Most breaks of a shuffled byte-plane end in one more literal-free 3- or 4-byte sequence a probe or two later; such a
 * sequence is the chained hit at the anchor with candidate snap - back (same offset, length back + m), so it is handed
 * back to the chain as that verdict.  Returns true then (pk, snap, ip = anchor).  Otherwise returns false with either
 *   hit false: ip = anchor + 1 and lit = the first probe the scalar code still has to make (a stale verdict, the end
 *              of the stream, or all four probes missed: LZ4_SCALAR_PROBES, on to the 32-wide rounds), or
 *   hit true:  literals, a catch-up of more than 7 bytes or a match of 270+ bytes; ip, match, back, lit and the length
 *              after the first four (have_mc, mc_carry) as the general emission takes them.
 * Team mode has no PACK table. */
template <bool U16>
DEV bool lz4t_search(Lz4Team* tm, smem_addr_t vda, void* tabmem, const StreamBase& sb, int n, int anchor, int accel,
                     int& twt, int& tvt, u32& pk, u32& snap, int& ip, bool& hit, int& match, int& back, int& lit,
                     bool& have_mc, int& mc_carry) {
  u16* tab16 = (u16*)tabmem;
  u32* tab32 = (u32*)tabmem;
  const int mfl1 = n - LZ4_MFLIMIT + 1;
  ip = anchor + 1;
  int it = 0, pos = ip;
  for (;; it++) {
    if (it == LZ4_SCALAR_PROBES) { LZ4T_DBG(g_dbg_lz4t_s[LZ4T_S_MISS4]); lit = it; return false; }
    pos = ip + (it ? 1 + (it - 1) * accel : 0);                    /* lz4.c:1043-1053 */
    if (ip + 1 + it * accel > mfl1) { lit = it; return false; }    /* the scalar loop ends the stream (lz4.c:1055) */
    if ((pos >> 5) > tvt) lz4t_reach(tm, pos, twt, tvt);          /* publishes the tile of pos-2: nothing later reads below it */
    u32 qk, qs;
    smem_ld_u32x2(vda, ((u32)pos % (u32)LZ4T_RING) << 3, qk, qs);
    const u32 h = qk >> LZ4T_HSHIFT;
    const int cand = U16 ? (int)tab16[h] : (int)tab32[h];
    __syncwarp();                                                  /* every lane has read the entry before any overwrites it */
    if (cand != (int)qs) { LZ4T_DBG(g_dbg_lz4t_s[LZ4T_S_STALE]); lit = it; return false; }
    if (U16) tab16[h] = (u16)pos; else tab32[h] = (u32)pos;
    if (qk & 1u) { pk = qk; snap = qs; break; }
  }
  LZ4T_DBG(g_dbg_lz4t_s[LZ4T_S_HIT0 + it]);
  const int vb = (int)((pk >> 8) & 7u), dist = pos - anchor;       /* catch-up length, cut at the anchor below */
  const int bq = vb < dist ? vb : dist;
  int m = (int)((pk >> 2) & 15u);
  if (m == LZ4T_LONG) {
    LZ4T_DBG(g_dbg_lz4t_s[LZ4T_S_LONG]);
    m = LZ4T_LONG + lz4_count_tail(sb, sb.s, pos + 4 + LZ4T_LONG, (int)snap + 4 + LZ4T_LONG, n - LZ4_LASTLITERALS, n);
  }
  if (bq == dist && bq + m < 15 + 255) {                           /* no literals (a capped catch-up has bq = 7 < dist) */
    const int mc = bq + m;
    snap -= (u32)bq;
    pk = 1u | ((u32)(mc < LZ4T_LONG ? mc : LZ4T_LONG) << 2);         /* from LZ4T_LONG on the chain counts again from the anchor */
    ip = anchor;
    LZ4C_ADD(LZ4C_SEQS, 1);
    LZ4C_ADD(LZ4C_CHAIN_SEQS, ~0ull);                              /* the chain counts it as its own: moved to SEQS */
    return true;
  }
  hit = true; ip = pos; match = (int)snap;                         /* imm stays false: the general path checks the limits */
  have_mc = true; mc_carry = m;
  back = bq;
  if (vb == LZ4T_BACKCAP && dist > LZ4T_BACKCAP) {                 /* 7 or more: the rest of the catch-up (lz4.c:1107-1109) */
    LZ4T_DBG(g_dbg_lz4t_s[LZ4T_S_CAPPED]);
    back = lz4_catch_up(sb.s, pos, (int)snap, anchor, LZ4T_BACKCAP);
  } else if (bq != dist) LZ4T_DBG(g_dbg_lz4t_s[LZ4T_S_LIT]);
  else LZ4T_DBG(g_dbg_lz4t_s[LZ4T_S_HUGE]);
  lit = pos - back - anchor;
  return false;
}

/* branch ids of lz4_encode_stream's one-warp paths and of the search, emission and last-literals code it shares with
 * team mode; emulator builds count them so that tests can tell which parse path a stream reached */
enum {
  /* chained "test next position" on the lane-cached window */
  LZ4E_H_WIN_PREFETCHED, LZ4E_H_WIN_BLOCKING,  /* the window refilled from the prefetched words / with a blocking load */
  LZ4E_H_WIN_PB_OFF,                         /* no prefetch: the next window would reach past the stream */
  LZ4E_H_WIN_FLUSH,                          /* parked records flushed at a refill (nrec >= 24) */
  LZ4E_H_CH_MISS,
  LZ4E_H_CH_D65535, LZ4E_H_CH_D65536,        /* 32-bit table: equal bytes at distance 65535 (taken) / 65536 (refused) */
  LZ4E_H_CH_LEN_REG, LZ4E_H_CH_LEN_X3, LZ4E_H_CH_LEN_X4,   /* the match length from x1|x2 / x3 / x4 */
  LZ4E_H_CH_TAIL_BALLOT, LZ4E_H_CH_TAIL_LOOP,  /* ... from lz4_count_tail: inside its 128-byte ballot / past it */
  LZ4E_H_CH_HUGE,                            /* a 270+ match leaves the chain */
  LZ4E_H_CH_EXT,                             /* a record with a length byte (mc 15..269) */
  LZ4E_H_CH_END_LAST, LZ4E_H_CH_END_PROBE,   /* ip + 64 > n: then ip >= mfl1 / the scalar probe */
  /* scalar post-match probe */
  LZ4E_H_POST_WIDE, LZ4E_H_POST_NARROW, LZ4E_H_POST_HIT, LZ4E_H_POST_MISS,
  LZ4E_H_POST_D65535, LZ4E_H_POST_D65536,
  /* search */
  LZ4E_H_SP_HIT0,                            /* + k: a hit at scalar probe k (0..3) */
  LZ4E_H_SP_ENDED = LZ4E_H_SP_HIT0 + 4,      /* the scalar probes ran into mflimit */
  LZ4E_H_SP_D65535, LZ4E_H_SP_D65536,
  LZ4E_H_R_HIT,                              /* a hit in a 32-wide round */
  LZ4E_H_R_FWD_HIT, LZ4E_H_R_FWD_MISS,       /* a lane's candidate forwarded from a lower lane with its hash hits / misses */
  LZ4E_H_R_PARTIAL,                          /* a round with fewer than 32 valid lanes */
  LZ4E_H_R_STEP64, LZ4E_H_R_STEP128, LZ4E_H_R_STEP192,   /* a probe past 64 / 128 / 192: the step grew */
  /* catch-up */
  LZ4E_H_CU_NONE, LZ4E_H_CU_SHORT, LZ4E_H_CU_LONG,   /* none / < 32 bytes / 32 or more (a second ballot round) */
  LZ4E_H_CU_ANCHOR, LZ4E_H_CU_ZERO,          /* stopped by the anchor / by position 0 */
  /* match length */
  LZ4E_H_ML_NEXT,                            /* have_next with x != 0 */
  LZ4E_H_ML_X0, LZ4E_H_ML_X1, LZ4E_H_ML_X2, LZ4E_H_ML_TAIL,   /* room > 20 */
  LZ4E_H_ML_ROOM20, LZ4E_H_ML_ROOM4,         /* room <= 20 / room <= 4 */
  LZ4E_H_ML_CLAMP,                           /* mc > room */
  LZ4E_H_ML_NARROW,                          /* !have_next */
  /* emission */
  LZ4E_H_EM_COMPACT,                         /* lit < 15 and mc < 15: one predicated store */
  LZ4E_H_EM_LIT_FF0, LZ4E_H_EM_LIT_FF1, LZ4E_H_EM_LIT_FF2,   /* lit >= 15 with zero / one / two 255 bytes */
  LZ4E_H_EM_ML_FF0, LZ4E_H_EM_ML_FF1, LZ4E_H_EM_ML_FF2,      /* mc >= 15 ... */
  LZ4E_H_EM_IMM, LZ4E_H_EM_LITS,             /* a sequence without literals (post-match) / from the search */
  /* limitedOutput: the check that refused the stream */
  LZ4E_H_LIM_FLUSH, LZ4E_H_LIM_FIRST, LZ4E_H_LIM_COMPACT, LZ4E_H_LIM_LONG, LZ4E_H_LIM_LAST,
  /* last literals */
  LZ4E_H_LAST_SHORT, LZ4E_H_LAST_FF0, LZ4E_H_LAST_FF1,   /* lastRun < 15 / 15..269 / 270 and more */
  LZ4E_H_LAST_NOPARSE,                       /* n < 13: no parse at all */
  /* tables */
  LZ4E_H_TAB_U16, LZ4E_H_TAB_U32, LZ4E_H_TAB_PACK,
  LZ4E_H_PACK_HI,                            /* PACK: a match whose candidate is at position >= 65536 (bit 16) */
  LZ4E_NHIT
};
#ifdef SIMT_EMU
static long long g_lz4e_hit[LZ4E_NHIT + 1];       /* [LZ4E_NHIT]: "none of these", not counted */
#define LZ4E_HIT(id) do { if (lane_id() == 0) g_lz4e_hit[id]++; } while (0)          /* warp-uniform branch */
#define LZ4E_HITL(id, c) do { if (c) g_lz4e_hit[id]++; } while (0)                 /* per lane */
#else
#define LZ4E_HIT(id) do {} while (0)
#define LZ4E_HITL(id, c) do {} while (0)
#endif

/* Returns the compressed size, or 0 when the stream does not fit in `cap`
 * (LZ4_compress_fast's limitedOutput failure).  Uniform across the warp.
 * `tabmem` is LZ4_TABLE_BYTES of shared memory private to this warp.
 *
 * Hot-path shape (driven by the ncu source view: ~250 dependent warp instructions per sequence
 * on the hard byte-plane in v1, 72 now): everything uniform across the warp is computed
 * redundantly by all lanes; table stores in the scalar sections are done by lane 0 between
 * __syncwarp()s.  The first four probes of every search are scalar and work on 12-byte register
 * windows (one round of aligned loads each); the "test next position" probe that follows every
 * match is an inner loop on a lane-cached window (see below); a sequence with < 15 literals and a
 * short match is written by ONE predicated store (lane 0 = token, lanes 1..lit = literals, the
 * next two = offset).  The 32-wide probe rounds only run when the scalar probes miss. */
/* PACK (only with the 12-bit byU32 table, streams of at most 128 KiB): positions are 17 bits wide, so
 * the table is kept as 4096 x u16 plus one bit per entry -- 8.5 KiB instead of 16 KiB, i.e. twice as
 * many streams per SM.  It costs a few instructions per probe; measured with 4 chunks in flight it wins
 * at typesize 2 and 8 and loses at typesize 4, so the host only uses it on request (BLOSC_B200_LZ4_PACK=1). */
template <bool U16, bool PACK, bool TEAM>
DEV int lz4_encode_stream(const u8* __restrict__ s, const int n, u8* __restrict__ d, const int cap,
                          const int accel, void* tabmem, int* need_out, Lz4Team* tm) {
  const int lane = lane_id();
  const StreamBase sb = make_stream_base(s);
  u16* tab16 = (u16*)tabmem;
  u32* tab32 = (u32*)tabmem;
  u32* tabhi = (u32*)((u8*)tabmem + 8192);                   /* PACK: bit 16 of the 4096 entries */
#define LZ4_TGET(h) (U16 ? (int)tab16[h] : PACK ? ((int)tab16[h] | (int)(((tabhi[(h) >> 5] >> ((h) & 31u)) & 1u) << 16)) : (int)tab32[h])
#define LZ4_TPUT(h, v) do { if (U16) tab16[h] = (u16)(v); else if (PACK) { tab16[h] = (u16)(v); const u32 m_ = 1u << ((h) & 31u); \
                            if ((v) & 0x10000) atomicOr(&tabhi[(h) >> 5], m_); else atomicAnd(&tabhi[(h) >> 5], ~m_); } \
                            else tab32[h] = (u32)(v); } while (0)

  for (int i = lane; i < (PACK ? LZ4_TAB17_BYTES : LZ4_TABLE_BYTES) / 4; i += 32) tab32[i] = 0;   /* LZ4_initStream, lz4.c:1384 */
  __syncwarp();
  LZ4E_HIT(U16 ? LZ4E_H_TAB_U16 : PACK ? LZ4E_H_TAB_PACK : LZ4E_H_TAB_U32);

  const bool limited = (long long)cap < (long long)n + n / 255 + 16;   /* lz4.c:1388,1395 */
  const int olimit = cap;
  const int mfl1 = n - LZ4_MFLIMIT + 1;       /* mflimitPlusOne */
  const int matchlimit = n - LZ4_LASTLITERALS;
  int ip = 1, anchor = 0, op = 0;
  int need = 0;                               /* max left-hand side of the limitedOutput checks = smallest capacity that passes */
#define LZ4_LIMIT(v, site) do { const int v_ = (v); if (v_ > need) need = v_; if (limited && v_ > olimit) { LZ4E_HIT(site); return 0; } } while (0)
  /* first byte (lz4.c:1005-1010): table[hash(0)] = 0, which the zeroed table already says */

  /* Lane-cached window for the literal-free chains that dominate shuffled data: lane l keeps the
   * 12 bytes at position w0+l and their hash, so the "fill table at ip-2 / test ip" step
   * (lz4.c:1236-1294) fetches both hashes and the bytes to compare with shuffles instead of
   * reloading and re-hashing; a refill costs one round of loads per 2-3 sequences.  The 3-byte
   * sequences such a chain produces (token, offset) are parked one per lane and written together. */
  int w0 = -(1 << 30);
  u32 wq0 = 0, wq1 = 0, wq2 = 0, wh = 0;
  int pb = -(1 << 30);                       /* base of the window requested ahead of time */
  u32 pq0 = 0, pq1 = 0, pq2 = 0, pq3 = 0;    /* its raw aligned words */
  int nrec = 0, recop = 0;
  u32 rec = 0;
  int twt = 0, tvt = -1;                     /* TEAM: `wt` as last published, highest tile whose ready word was checked */
#define LZ4_FLUSH_CHECKED() do { if (nrec) { LZ4_LIMIT(op + (1 + LZ4_LASTLITERALS), LZ4E_H_LIM_FLUSH); } LZ4_FLUSH(); } while (0)
#define LZ4_FLUSH() do { if (lane < nrec) { d[recop] = (u8)rec; d[recop + 1] = (u8)(rec >> 8); d[recop + 2] = (u8)(rec >> 16); \
                                             if ((rec & 15u) == 15u) d[recop + 3] = (u8)(rec >> 24); } nrec = 0; } while (0)

  if (n >= LZ4_MFLIMIT + 1) {                 /* lz4.c:1002 */
    bool post = false;                        /* true: a match just ended at ip (== anchor) */
    for (;;) {
      int match = 0, lit = 0, back = 0;
      u32 ipn = 0, cn = 0;                    /* bytes [ip+4, ip+8) and [match+4, match+8) of the hit */
      bool have_next = false, hit = false, imm = false, have_mc = false;
      int mc_carry = 0;

      bool scalar_post = post;
      if constexpr (TEAM) if (post && ip + 64 <= n) {   /* (not instantiated for encode_kernel) */
        /* ---- chained "test next position" (lz4.c:1236-1294) with the verdicts prepared by the helper
         * warps (see "team mode" above), a window of up to LZ4T_W sequences per step:
         * 1. path: hop from q_0 = ip along the verdicts, q_{j+1} = q_j + 4 + length field; a miss or an LZ4T_LONG is
         *    the window's last element, and the hop stops before a position whose tile is past tvt, that is too close
         *    to the end of the stream, or when the window is full.
         * 2. check: the serial code would store S_2j = (h(q_j - 2), q_j - 2) and S_2j+1 = (h(q_j), q_j), and element
         *    j reads table[h(q_j)] after S_2j.  Lane m takes S_m; that read is the position of the highest lower lane
         *    with the same hash, or else the live entry (read before any store of the window).  Element j is exact
         *    when it equals the verdict's snap, so the elements before the first one that is not are exactly what as
         *    many serial iterations would have done.
         * 3. commit: their stores (per hash the last one in serial order) and their 3-byte records.
         * The element that ends the window goes to the code that handled it one sequence at a time. ---- */
        scalar_post = false;
        bool finished = false;
        LZ4T_DBG(g_dbg_lz4t_sessions);
        LZ4C_T(c_s0);
        LZ4C_ADD(LZ4C_SESSIONS, 1);
        if ((ip - 2) >> 5 <= twt + LZ4T_AHEAD) LZ4T_DBG(g_dbg_lz4t_x[3]);     /* its tiles are prepared or in flight */
        lz4t_reach(tm, ip, twt, tvt);
        __syncwarp();                         /* table stores of the scalar code (lane 0) are seen by every lane */
        LZ4C_SPAN(LZ4C_START, c_s0);
        LZ4C_T(c_s1);
        const smem_addr_t vda = smem_addr(tm->vd);
        u32 e = (u32)ip % (u32)LZ4T_RING;     /* ring entry of ip: slot (ip >> 5) mod LZ4T_TILES, lane ip & 31 */
        bool given = false;                   /* element 0 is lz4t_search's hit at ip: checked and stored already */
        u32 gpk = 0, gsnap = 0;
        for (;;) {
          /* a window parks at most LZ4T_W records; op only grows inside a chain, so one limitedOutput check per
           * parked batch, before anything is written, is exact (LZ4_FLUSH_CHECKED) */
          if (nrec > 32 - LZ4T_W) {
#ifdef SIMT_EMU
            if (limited && op + 1 + LZ4_LASTLITERALS > olimit) LZ4T_DBG(g_dbg_lz4t_w[LZ4T_W_FULL]);
#endif
            LZ4_FLUSH_CHECKED();
          }
          lz4t_extend(tm, twt, tvt);
          /* 1. path; lane j keeps element j (position, ring entry, verdict) */
          int cnt = 0, q = ip, why;
          u32 ee = e, pk, snap;
          if (given) { pk = gpk; snap = gsnap; } else smem_ld_u32x2(vda, ee << 3, pk, snap);
          int jq = 0;
          u32 je = 0, jpk = 0, jsnap = 0;
          for (;;) {
            if (lane == cnt) { jq = q; je = ee; jpk = pk; jsnap = snap; }
            cnt++;
            const u32 step = ((pk >> 2) & 15u) + 4u;
            u32 en = ee + step;
            if (en >= (u32)LZ4T_RING) en -= (u32)LZ4T_RING;
            u32 npk, nsnap;
            smem_ld_u32x2(vda, en << 3, npk, nsnap);                       /* ahead of the tests: en is inside the ring */
            if (!(pk & 1u)) { why = LZ4C_W_MISS; break; }
            if (step == LZ4T_LONG + 4u) { why = LZ4C_W_LONG; break; }
            q += (int)step; ee = en;
            if (cnt == LZ4T_W) { why = LZ4C_W_CAP; break; }
            if (q + 64 > n) { why = LZ4C_W_END; break; }
            if ((q >> 5) > tvt) { why = LZ4C_W_TILE; break; }
            pk = npk; snap = nsnap;
          }
          /* 2. check: lane m holds S_m */
          u32 jh2 = 0;
          if (lane < cnt) jh2 = smem_ld_u32(vda, (je >= 2u ? je - 2u : je - 2u + LZ4T_RING) << 3) >> LZ4T_HSHIFT;
          const int el = lane >> 1;
          const bool odd = (lane & 1) != 0;
          const u32 sh2 = __shfl_sync(FULLMASK, jh2, el), sh = __shfl_sync(FULLMASK, jpk >> LZ4T_HSHIFT, el);
          const int sq = __shfl_sync(FULLMASK, jq, el);
          const u32 ssnap = __shfl_sync(FULLMASK, jsnap, el);
          const bool act = lane < 2 * cnt && !(given && lane < 2);
          const u32 skey = odd ? sh : sh2;
          const int spos = odd ? sq : sq - 2;
          /* the live entries, and whether two stores of the window share a hash: one bit per hash, set with an atomic */
          int look = 0;
          bool dup = false;
          if (act) {
            if (odd) look = LZ4_TGET(skey);
            const u32 bit = 1u << (skey & 31u);
            dup = (atomicOr(&tm->seen[skey >> 5], bit) & bit) != 0;
          }
          unsigned peers = 1u << lane;                                     /* lanes with my hash: mine alone, unless ... */
          if (__ballot_sync(FULLMASK, dup)) {                              /* (rare) a hash is shared: the nearest lower lane forwards its position */
            peers = __match_any_sync(FULLMASK, act ? skey : 0x80000000u | (u32)lane);   /* hashes have 13 bits */
            const unsigned lower = peers & ((1u << lane) - 1u);
            const int fpos = __shfl_sync(FULLMASK, spos, lower ? 31 - __clz((int)lower) : lane);
            if (act && odd && lower) look = fpos;
#ifdef SIMT_EMU
            const unsigned fwd = __ballot_sync(FULLMASK, act && odd && lower != 0);
            const unsigned cross = __ballot_sync(FULLMASK, act && !odd && ((peers & 0xaaaaaaaau) & ~(2u << lane)) != 0);
            if (fwd) LZ4T_DBG(g_dbg_lz4t_w[LZ4T_W_FWD]);
            if (cross) LZ4T_DBG(g_dbg_lz4t_w[LZ4T_W_CROSS]);
#endif
          }
          const unsigned bad = __ballot_sync(FULLMASK, act && odd && look != (int)ssnap);
          const int nv = bad ? (__ffs((int)bad) - 1) >> 1 : cnt;           /* valid elements: a prefix */
          LZ4T_DBG(g_dbg_lz4t_w[LZ4T_W_WINDOWS]);
          LZ4T_DBGN(g_dbg_lz4t_w[LZ4T_W_ELEMS], nv);
          __syncwarp();                                                    /* every lane has read the table before any store */
          /* 3. commit */
          const unsigned le = nv >= 16 ? FULLMASK : (1u << (2 * nv)) - 1u;
          if (act && lane < 2 * nv && (((peers & le) >> lane) >> 1) == 0) LZ4_TPUT(skey, spos);
          if (act) tm->seen[skey >> 5] = 0u;
          __syncwarp();
          const int nb = nv < cnt || why == LZ4C_W_MISS || why == LZ4C_W_LONG ? (nv < cnt ? nv : cnt - 1) : cnt;
          const u32 rv = (u32)((jpk >> 2) & 15u) | ((u32)(jq - (int)jsnap) << 8);   /* lz4.c:1187-1226 with 0 literals, 4..16 bytes */
          const u32 rmine = __shfl_sync(FULLMASK, rv, (lane - nrec) & 31);
          if (lane >= nrec && lane < nrec + nb) { rec = rmine; recop = op + 3 * (lane - nrec); }
          nrec += nb;
          op += 3 * nb;
          LZ4T_DBGN(g_dbg_lz4t_seqs, nb);
          LZ4C_ADD(LZ4C_CHAIN_SEQS, nb);
          LZ4C_ADD(LZ4C_WINDOWS, 1);
          if (nb < cnt) {                                                  /* the element that ends the window */
            ip = __shfl_sync(FULLMASK, jq, nb);
            e = __shfl_sync(FULLMASK, je, nb);
            snap = __shfl_sync(FULLMASK, jsnap, nb);
          } else { ip = q; e = ee; }
          anchor = ip;
          given = false;
          if (nv < cnt) {                                                  /* its verdict was computed from another candidate */
            LZ4T_DBG(g_dbg_lz4t_stale); LZ4C_ADD(LZ4C_STALE, 1); LZ4C_ADD(LZ4C_W_STALE, 1);
            LZ4T_DBG(g_dbg_lz4t_w[nv ? LZ4T_W_STALEJ : LZ4T_W_STALE0]);
            scalar_post = true; break;                                     /* the plain probe below looks this one up itself */
          }
          LZ4C_ADD(why, 1);
          if (why == LZ4C_W_MISS) {                                        /* lz4.c:1298, then the search */
            LZ4T_DBG(g_dbg_lz4t_x[4]);
            LZ4T_DBG(g_dbg_lz4t_w[nb ? LZ4T_W_MISSJ : LZ4T_W_MISS0]);
            if (!lz4t_search<U16>(tm, vda, tabmem, sb, n, anchor, accel, twt, tvt, gpk, gsnap, ip, hit, match, back, lit, have_mc, mc_carry))
              break;                                                       /* on to the search or the emission below */
            given = true;                                                  /* a literal-free hit at ip = anchor: element 0 of the next window */
            continue;
          }
          if (why == LZ4C_W_LONG) {
            LZ4T_DBG(g_dbg_lz4t_x[0]);
            LZ4T_DBG(g_dbg_lz4t_w[nb ? LZ4T_W_LONGJ : LZ4T_W_LONG0]);
            const int off = ip - (int)snap;
            const int mc = LZ4T_LONG + lz4_count_tail(sb, s, ip + 4 + LZ4T_LONG, ip - off + 4 + LZ4T_LONG, matchlimit, n);   /* ip+64 <= n: far from matchlimit */
            if (mc >= 15 + 255) {                                          /* very long match: general emission below */
              hit = true; imm = true; match = ip - off;
              have_mc = true; mc_carry = mc;
              LZ4T_DBG(g_dbg_lz4t_x[1]);
              LZ4T_DBG(g_dbg_lz4t_w[LZ4T_W_HUGE]);
              break;
            }
            /* token, offset and -- from 19 bytes on -- one length byte (at most 31 records are parked here) */
            const bool ext = mc >= 15;
            LZ4T_DBG(g_dbg_lz4t_seqs);
            LZ4C_ADD(LZ4C_CHAIN_SEQS, 1);
            if (lane == nrec) { rec = (ext ? 15u | ((u32)(mc - 15) << 24) : (u32)mc) | ((u32)off << 8); recop = op; }
            nrec++;
            op += ext ? 4 : 3;
            ip += mc + 4;
            e += (u32)(mc + 4);                                            /* mc + 4 < 15 + 255 + 4 < LZ4T_RING */
            if (e >= (u32)LZ4T_RING) e -= (u32)LZ4T_RING;
            anchor = ip;
          } else if (why == LZ4C_W_CAP) LZ4T_DBG(g_dbg_lz4t_w[LZ4T_W_CAP]);
          else if (why == LZ4C_W_TILE) LZ4T_DBG(g_dbg_lz4t_w[LZ4T_W_TILE]);
          if (ip + 64 > n) {                                               /* a match ended close to the end of the stream */
            if (why == LZ4C_W_END) LZ4T_DBG(g_dbg_lz4t_w[LZ4T_W_END]);
            if (ip >= mfl1) finished = true;                               /* lz4.c:1230-1233 */
            else scalar_post = true;                                       /* the plain probe below takes over */
            break;
          }
          LZ4C_T(c_w);
          lz4t_reach(tm, ip, twt, tvt);                                    /* publishes the tile of ip - 2, waits for that of ip */
          LZ4C_SPAN(LZ4C_FULLWAIT, c_w);
        }
        LZ4C_SPAN(LZ4C_SESSION, c_s1);
        if (finished) break;
      }
      if (!TEAM && post && ip + 64 <= n) {
        scalar_post = false;
        /* ---- chained "test next position" on the lane-cached window: stays in this loop for as
         * long as every match is immediately followed by another one ---- */
        bool room = true;
        for (;;) {
          if (ip - 2 < w0 || ip > w0 + 31) {
            if (nrec >= 24) { LZ4E_HIT(LZ4E_H_WIN_FLUSH); LZ4_FLUSH_CHECKED(); }   /* a window serves at most 8 sequences */
            /* The window that follows (base w0+30: the first ip past this window is >= w0+32) was
             * requested at the previous refill, so its bytes are here by now; only a long match
             * that jumps over it pays for a blocking load. */
            if (ip - 2 >= pb && ip <= pb + 31) {
              LZ4E_HIT(LZ4E_H_WIN_PREFETCHED);
              w0 = pb; ldp_take12(sb, w0 + lane, pq0, pq1, pq2, pq3, wq0, wq1, wq2);
            } else { LZ4E_HIT(LZ4E_H_WIN_BLOCKING); w0 = ip - 2; ldp_win12(sb, w0 + lane, wq0, wq1, wq2); }   /* reaches byte w0+46 < ip+64 <= n */
            wh = lz4_hash_seq<U16>(wq0, wq1);
            pb = w0 + 30;
            if (pb + 31 + 16 <= n) ldp_raw12(sb, pb + lane, pq0, pq1, pq2, pq3);   /* not waited for */
            else { LZ4E_HIT(LZ4E_H_WIN_PB_OFF); pb = -(1 << 30); }
            lz4d_prefetch(s, w0 + 192, lane == 0 ? n : 0);                   /* the line a few refills ahead */
          }
          const int li = ip - w0;                                            /* 2 .. 31 */
          const u32 h2 = __shfl_sync(FULLMASK, wh, li - 2);
          const u32 h = __shfl_sync(FULLMASK, wh, li);
          const u32 seq = __shfl_sync(FULLMASK, wq0, li);
          const u32 n4 = __shfl_sync(FULLMASK, wq1, li);                     /* bytes ip+4 .. ip+7 */
          const u32 n8 = __shfl_sync(FULLMASK, wq2, li);                     /* bytes ip+8 .. ip+11 */
          if (lane == 0) LZ4_TPUT(h2, ip - 2);
          __syncwarp();
          const int cand = LZ4_TGET(h);
          __syncwarp();                    /* every lane has read the old entry before lane 0 overwrites it */
          if (lane == 0) LZ4_TPUT(h, ip);
          u32 c0, c1, c2;
          ldp_win12(sb, cand, c0, c1, c2);   /* cand is a position < ip whatever the table holds: safe even when it is too far back */
          LZ4E_HIT(U16 || c0 != seq ? LZ4E_NHIT : ip - cand == 65535 ? LZ4E_H_CH_D65535 : ip - cand == 65536 ? LZ4E_H_CH_D65536 : LZ4E_NHIT);
          if (!((U16 || cand + 65535 >= ip) && c0 == seq)) { LZ4E_HIT(LZ4E_H_CH_MISS); ip++; break; }  /* lz4.c:1298; on to the search below */
          int mc;
          const u32 x1 = n4 ^ c1, x2 = n8 ^ c2;
          if (x1 | x2) {
            const u32 xx = x1 ? x1 : x2;
            mc = ((__ffs((int)xx) - 1) >> 3) + (x1 ? 0 : 4);
            LZ4E_HIT(LZ4E_H_CH_LEN_REG);
          } else {                                                           /* >= 12 bytes: next 8 from memory */
            u32 p3, p4, q3, q4;
            ldp_win8(sb, ip + 12, p3, p4);
            ldp_win8(sb, cand + 12, q3, q4);
            const u32 x3 = p3 ^ q3, x4 = p4 ^ q4;
            if (x3) { mc = 8 + eq_bytes32(x3); LZ4E_HIT(LZ4E_H_CH_LEN_X3); }
            else if (x4) { mc = 12 + eq_bytes32(x4); LZ4E_HIT(LZ4E_H_CH_LEN_X4); }
            else {
              mc = 16 + lz4_count_tail(sb, s, ip + 20, cand + 20, matchlimit, n);   /* ip+64 <= n: far from matchlimit */
              LZ4E_HIT(mc < 16 + 128 && ip + 20 + 136 <= n ? LZ4E_H_CH_TAIL_BALLOT : LZ4E_H_CH_TAIL_LOOP);
            }
          }
          if (mc >= 15 + 255) {                                              /* very long match: general emission below */
            LZ4E_HIT(LZ4E_H_CH_HUGE);
            hit = true; imm = true; match = cand;
            have_mc = true; mc_carry = mc;
            break;
          }
          /* lz4.c:1187-1226 with 0 literals: token, offset and -- from 19 bytes on -- one length byte.
           * Both limitedOutput checks of such a sequence ask for (op after it) + 6 <= olimit; op only
           * grows inside a chain, so the check is made once per parked batch, before anything is
           * written (LZ4_FLUSH_CHECKED) */
          const bool ext = mc >= 15;
          if (ext) LZ4E_HIT(LZ4E_H_CH_EXT);
          if (PACK && cand >= 65536) LZ4E_HIT(LZ4E_H_PACK_HI);
          const int off = ip - cand;
          if (lane == nrec) { rec = (ext ? 15u | ((u32)(mc - 15) << 24) : (u32)mc) | ((u32)off << 8); recop = op; }
          nrec++;
          op += ext ? 4 : 3;
          ip += mc + 4;
          anchor = ip;
          if (ip + 64 > n) { room = false; break; }
        }
        if (!room) {                                                         /* a match ended close to the end of the stream */
          LZ4E_HIT(ip >= mfl1 ? LZ4E_H_CH_END_LAST : LZ4E_H_CH_END_PROBE);
          if (ip >= mfl1) break;                                             /* lz4.c:1230-1233 */
          continue;                                                          /* post stays true: the plain probe below takes over */
        }
      }
      if (scalar_post) {
        /* ---- fill table at ip-2, test position ip (lz4.c:1236-1294); no literals on a hit ---- */
        LZ4C_TW(c_r);
        u32 b0, b1, b2 = 0;
        const bool wide = ip + 14 <= n;
        LZ4E_HIT(wide ? LZ4E_H_POST_WIDE : LZ4E_H_POST_NARROW);
        if (wide) ldp_win12(sb, ip - 2, b0, b1, b2);
        else { b0 = ld_u32(s + ip - 2); b1 = ld_u32(s + ip + 2); }
        const u32 seq = __funnelshift_r(b0, b1, 16);                       /* bytes ip .. ip+3 */
        const u32 h2 = lz4_hash_seq<U16>(b0, b1);                          /* 5th byte of ip-2 is s[ip+2] */
        const u32 h = lz4_hash_seq<U16>(seq, b1 >> 16);                    /* 5th byte of ip is s[ip+4] */
        if (lane == 0) LZ4_TPUT(h2, ip - 2);
        __syncwarp();
        const int cand = LZ4_TGET(h);
        __syncwarp();                      /* every lane has read the old entry before lane 0 overwrites it */
        if (lane == 0) LZ4_TPUT(h, ip);
        LZ4E_HIT(U16 || ld_u32(s + cand) != seq ? LZ4E_NHIT : ip - cand == 65535 ? LZ4E_H_POST_D65535 : ip - cand == 65536 ? LZ4E_H_POST_D65536 : LZ4E_NHIT);
        if (U16 || cand + 65535 >= ip) {
          u32 c0, c1;
          ldp_win8(sb, cand, c0, c1);
          if (c0 == seq) {
            hit = true; imm = true; match = cand;
            ipn = __funnelshift_r(b1, b2, 16); cn = c1; have_next = wide;
          }
        }
        LZ4E_HIT(hit ? LZ4E_H_POST_HIT : LZ4E_H_POST_MISS);
        if (!hit) ip++;                                                    /* lz4.c:1298 */
        if (TEAM) LZ4C_SPAN(LZ4C_REPROBE, c_r);
      }

      if (!hit) {
        /* ---- find a match (lz4.c:1043-1101): two scalar probes, then 32-wide rounds ---- */
        LZ4C_TW(c_f);
        bool ended = false;
        for (int it = TEAM ? lit : 0; it < LZ4_SCALAR_PROBES; it++) {   /* TEAM: lit = first probe lz4t_search left */
          const int pos = ip + (it ? 1 + (it - 1) * accel : 0);            /* probe offsets 0, 1, 1+accel, 1+2*accel (lz4.c:1043-1053) */
          if (ip + 1 + it * accel > mfl1) { LZ4E_HIT(LZ4E_H_SP_ENDED); ended = true; break; }   /* `goto _last_literals` (lz4.c:1055) */
          u32 b0, b1 = 0, b2 = 0;
          const bool wide = pos + 16 <= n;
          if (wide) ldp_win12(sb, pos, b0, b1, b2);
          else { b0 = ld_u32(s + pos); b1 = (u32)s[pos + 4]; }
          const u32 h = lz4_hash_seq<U16>(b0, b1);
          __syncwarp();                    /* table writes of the previous step are visible */
          const int cand = LZ4_TGET(h);
          __syncwarp();
          if (lane == 0) LZ4_TPUT(h, pos);
          LZ4E_HIT(U16 || ld_u32(s + cand) != b0 ? LZ4E_NHIT : pos - cand == 65535 ? LZ4E_H_SP_D65535 : pos - cand == 65536 ? LZ4E_H_SP_D65536 : LZ4E_NHIT);
          if (U16 || cand + 65535 >= pos) {
            u32 c0, c1;
            ldp_win8(sb, cand, c0, c1);
            if (c0 == b0) {
              LZ4E_HIT(LZ4E_H_SP_HIT0 + it);
              hit = true; ip = pos; match = cand;
              ipn = b1; cn = c1; have_next = wide;
              break;
            }
          }
        }
        if (!hit && !ended) {
          __syncwarp();
          for (int base_it = LZ4_SCALAR_PROBES;; base_it += 32) {
            const int itl = base_it + lane;
            const bool valid = ip + lz4_probe_offset(itl + 1, accel) <= mfl1;
            const int pos = valid ? ip + (int)lz4_probe_offset(itl, accel) : 0;
            u32 h = 0x80000000u | (u32)lane, seq = 0;
            if (valid) { seq = ld_u32(s + pos); h = lz4_hash_at<U16>(s, pos); }
            const unsigned vmask = __ballot_sync(FULLMASK, valid);
            const unsigned peers = __match_any_sync(FULLMASK, h);
            const unsigned lower = peers & ((1u << lane) - 1u);
            int cand = 0;
            bool lhit = false;
            if (valid) {
              cand = lower ? ip + (int)lz4_probe_offset(base_it + (31 - __clz((int)lower)), accel) : LZ4_TGET(h);
              if (U16 || cand + 65535 >= pos) lhit = ld_u32(s + cand) == seq;   /* lz4.c:1090-1101 */
              LZ4E_HITL(lhit ? LZ4E_H_R_FWD_HIT : LZ4E_H_R_FWD_MISS, lower != 0);
              LZ4E_HITL(LZ4E_H_R_STEP64, itl - 1 >= 64);
              LZ4E_HITL(LZ4E_H_R_STEP128, itl - 1 >= 128);
              LZ4E_HITL(LZ4E_H_R_STEP192, itl - 1 >= 192);
            }
            const unsigned found = __ballot_sync(FULLMASK, lhit);
            const int nvalid = __popc(vmask);                       /* valid lanes form a prefix */
            const int f = found ? __ffs((int)found) - 1 : 32;
            const int last = f < nvalid - 1 ? f : nvalid - 1;       /* last probe committed to the table */
            __syncwarp();                                           /* all lookups done before any commit */
            if (valid && lane <= last) {
              const unsigned le = last >= 31 ? FULLMASK : ((1u << (last + 1)) - 1u);
              if ((((peers & le) >> lane) >> 1) == 0) LZ4_TPUT(h, pos);  /* highest committed lane per hash wins */
            }
            __syncwarp();
            if (found) {
              LZ4E_HIT(LZ4E_H_R_HIT);
              ip = __shfl_sync(FULLMASK, pos, f);
              match = __shfl_sync(FULLMASK, cand, f);
              hit = true;
              break;
            }
            if (nvalid < 32) { LZ4E_HIT(LZ4E_H_R_PARTIAL); break; }  /* ran into the end: last literals */
          }
        }
        if (!hit) { if (TEAM) LZ4C_SPAN(LZ4C_SEARCH, c_f); break; }  /* -> last literals */

        /* ---- catch up (lz4.c:1107-1109) ---- */
        if (ip > anchor && match > 0 && s[ip - 1] == s[match - 1]) back = lz4_catch_up(s, ip, match, anchor, 0);
        LZ4E_HIT(back == 0 ? LZ4E_H_CU_NONE : back < 32 ? LZ4E_H_CU_SHORT : LZ4E_H_CU_LONG);
        if (back) LZ4E_HIT(ip - back == anchor ? LZ4E_H_CU_ANCHOR : match - back == 0 ? LZ4E_H_CU_ZERO : LZ4E_NHIT);
        lit = ip - back - anchor;
        if (TEAM) LZ4C_SPAN(LZ4C_SEARCH, c_f);
      }

      /* ---- match length (lz4.c:1182-1184): LZ4_count(start+4, ...) = catch-up bytes + forward bytes.
       * Most matches of shuffled data are 8..20 bytes long: compare that much with scalar
       * (warp-uniform) loads first and only then fall into the 512-bytes-per-round warp loop. ---- */
      int mc;
      if (have_mc) mc = mc_carry;                                    /* already counted by the chained probe */
      else {
        const int room = matchlimit - (ip + 4);                      /* >= 3 because ip < mflimitPlusOne */
        if (have_next) {
          const u32 x = ipn ^ cn;
          if (x) { mc = eq_bytes32(x); LZ4E_HIT(LZ4E_H_ML_NEXT); }
          else if (room > 20) {
            u32 p0, p1, p2, q0, q1, q2;                              /* bytes [ip+8, ip+20) vs [match+8, match+20) */
            ldp_win12(sb, ip + 8, p0, p1, p2);                        /* ip+8+16 <= n because room > 20 */
            ldp_win12(sb, match + 8, q0, q1, q2);
            const u32 x0 = p0 ^ q0, x1 = p1 ^ q1, x2 = p2 ^ q2;
            if (x0) { mc = 4 + eq_bytes32(x0); LZ4E_HIT(LZ4E_H_ML_X0); }
            else if (x1) { mc = 8 + eq_bytes32(x1); LZ4E_HIT(LZ4E_H_ML_X1); }
            else if (x2) { mc = 12 + eq_bytes32(x2); LZ4E_HIT(LZ4E_H_ML_X2); }
            else { mc = 16 + lz4_count_tail(sb, s, ip + 20, match + 20, matchlimit, n); LZ4E_HIT(LZ4E_H_ML_TAIL); }
          } else {
            LZ4E_HIT(room > 4 ? LZ4E_H_ML_ROOM20 : LZ4E_H_ML_ROOM4);
            mc = 4 + (room > 4 ? warp_count_match(s, ip + 8, match + 8, matchlimit) : 0);
          }
          if (mc > room) { LZ4E_HIT(LZ4E_H_ML_CLAMP); mc = room; }
        } else { LZ4E_HIT(LZ4E_H_ML_NARROW); mc = warp_count_match(s, ip + 4, match + 4, matchlimit); }
      }
      const int off = ip - match;
      ip += mc + 4;
      mc += back;

      /* ---- emit (lz4.c:1112-1226) ---- */
      if (TEAM) LZ4C_ADD(LZ4C_SEQS, 1);
      LZ4_FLUSH_CHECKED();
      const int token = op++;
      LZ4E_HIT(imm ? LZ4E_H_EM_IMM : LZ4E_H_EM_LITS);
      if (PACK && match >= 65536) LZ4E_HIT(LZ4E_H_PACK_HI);
      if (!imm) LZ4_LIMIT(op + lit + (2 + 1 + LZ4_LASTLITERALS) + lit / 255, LZ4E_H_LIM_FIRST);
      if (lit < 15 && mc < 15) {
        LZ4E_HIT(LZ4E_H_EM_COMPACT);
        LZ4_LIMIT(op + lit + 2 + (1 + LZ4_LASTLITERALS), LZ4E_H_LIM_COMPACT);
        u32 v;
        if (lane == 0) v = ((u32)lit << 4) | (u32)mc;
        else if (lane <= lit) v = s[anchor + lane - 1];
        else v = lane == lit + 1 ? (u32)off : (u32)off >> 8;
        if (lane <= lit + 2) d[token + lane] = (u8)v;
        op += lit + 2;
      } else {
        u32 tokval;
        if (lit >= 15) {
          const int len = lit - 15, nff = len / 255;
          LZ4E_HIT(LZ4E_H_EM_LIT_FF0 + (nff < 2 ? nff : 2));
          tokval = 15u << 4;
          warp_fill_bytes(d + op, nff, 255);
          if (lane == 0) d[op + nff] = (u8)(len - nff * 255);
          op += nff + 1;
        } else tokval = (u32)lit << 4;
        warp_copy_bytes(d + op, s + anchor, lit);
        op += lit;
        if (lane == 0) { d[op] = (u8)off; d[op + 1] = (u8)(off >> 8); }
        op += 2;
        LZ4_LIMIT(op + (1 + LZ4_LASTLITERALS) + (mc + 240) / 255, LZ4E_H_LIM_LONG);
        if (mc >= 15) {
          tokval += 15;
          const int rest = mc - 15, nff = rest / 255;
          LZ4E_HIT(LZ4E_H_EM_ML_FF0 + (nff < 2 ? nff : 2));
          warp_fill_bytes(d + op, nff, 255);
          if (lane == 0) d[op + nff] = (u8)(rest - nff * 255);
          op += nff + 1;
        } else tokval += (u32)mc;
        if (lane == 0) d[token] = (u8)tokval;
      }

      anchor = ip;
      if (ip >= mfl1) break;                                         /* lz4.c:1230-1233 */
      post = true;
    }
  }

  /* ---- last literals (lz4.c:1302-1329) ---- */
  LZ4_FLUSH_CHECKED();
  const int lastRun = n - anchor;
  if (n < LZ4_MFLIMIT + 1) LZ4E_HIT(LZ4E_H_LAST_NOPARSE);
  LZ4E_HIT(lastRun < 15 ? LZ4E_H_LAST_SHORT : lastRun < 270 ? LZ4E_H_LAST_FF0 : LZ4E_H_LAST_FF1);
  LZ4_LIMIT(op + lastRun + 1 + (lastRun + 255 - 15) / 255, LZ4E_H_LIM_LAST);
  if (lastRun >= 15) {
    const int acc = lastRun - 15, nff = acc / 255;
    if (lane == 0) d[op] = (u8)(15u << 4);
    op++;
    warp_fill_bytes(d + op, nff, 255);
    if (lane == 0) d[op + nff] = (u8)(acc - nff * 255);
    op += nff + 1;
  } else {
    if (lane == 0) d[op] = (u8)(lastRun << 4);
    op++;
  }
  warp_copy_bytes(d + op, s + anchor, lastRun);
  op += lastRun;
  *need_out = need;
  return op;
#undef LZ4_FLUSH_CHECKED
#undef LZ4_FLUSH
#undef LZ4_LIMIT
#undef LZ4_TGET
#undef LZ4_TPUT
}

/* Team mode, walker side, around each stream: the preparers start with wt = 0 and fresh ready words; at
 * the end the walker posts LZ4T_STOP and waits until all three are parked at their GO barriers again,
 * so that the next stream may change the stream fields and clear the ready words.  The kernel ends
 * the preparers after its last stream by posting LZ4T_QUIT and arriving at GO(0..2). */
DEV void lz4t_begin(Lz4Team* tm, const u8* s, int n, bool u16) {
  const int lane = lane_id();
  for (int i = lane; i < LZ4T_TILES; i += 32) tm->rdy[i] = 0;
  for (int i = lane; i < 8192 / 32; i += 32) tm->seen[i] = 0;
  if (lane == 0) { tm->s = s; tm->n = n; tm->u16 = u16 ? 1 : 0; tm->wt = 0; tm->gen = tm->gen + 1; }
  __syncwarp();
  __threadfence_block();
  bar_arrive(LZ4T_BAR_GO(0), 64); bar_arrive(LZ4T_BAR_GO(1), 64); bar_arrive(LZ4T_BAR_GO(2), 64);
}
DEV void lz4t_end(Lz4Team* tm) {
  __syncwarp();                            /* every lane's last store of `wt` (lz4t_reach) lands before LZ4T_STOP */
  if (lane_id() == 0) lz4t_st_i32(&tm->wt, LZ4T_STOP);
  __syncwarp();
  bar_sync(LZ4T_BAR_IDLE(0), 64); bar_sync(LZ4T_BAR_IDLE(1), 64); bar_sync(LZ4T_BAR_IDLE(2), 64);
}

/* Returns the compressed size, or 0 when the stream does not fit in `cap` (see lz4_encode_stream).
 * TEAM: the calling warp is the walker of the team `tm` (one stream from start to end, on every return). */
template <bool U16, bool PACK = false, bool TEAM = false>
DEV int lz4_encode_warp(const u8* __restrict__ s, const int n, u8* __restrict__ d, const int cap,
                        const int accel, void* tabmem, int* need_out, Lz4Team* tm = nullptr) {
  if (TEAM) lz4t_begin(tm, s, n, U16);
  const int c = lz4_encode_stream<U16, PACK, TEAM>(s, n, d, cap, accel, tabmem, need_out, tm);
  if (TEAM) lz4t_end(tm);
  return c;
}

/* ---- decoder ---- */
/* branch ids of the tier walk (lz4_decode_warp and lz4_pair_parse both run it); emulator builds count
 * them so that tests can tell which tier and which match source a stream reached */
enum {
  LZ4D_H_DENSE_SHIFT = 0,                    /* + s: a dense step whose last segment has byte shift s (0..8) */
  LZ4D_H_DENSE_LONGCAP = 9,                  /* the segment loop stopped at LZ4D_DENSE_LONG long matches */
  LZ4D_H_DENSE_BAD,                          /* a sequence that reads the step's own output (or before the block) ends the run */
  LZ4D_H_DENSE_BAD0,                         /* ... already at lane 0 (cnt == 0) */
  LZ4D_H_DENSE_FEW,                          /* fewer than LZ4D_DENSE_MIN short and no long sequence: no dense step */
  LZ4D_H_DENSE_RING, LZ4D_H_DENSE_GLOBAL,    /* a dense sequence's match source */
  LZ4D_H_LONE_RING, LZ4D_H_LONE_GLOBAL, LZ4D_H_LONE_PERIOD,
  LZ4D_H_BATCH_FAST, LZ4D_H_BATCH_WALK,      /* the 0x49249249 chain of 3-byte sequences / the shuffle walk */
  LZ4D_H_BATCH_RING, LZ4D_H_BATCH_GLOBAL,
  LZ4D_H_SINGLE_RING, LZ4D_H_SINGLE_GLOBAL,
  LZ4D_H_GEN_LITBUMP,                        /* a literal run longer than the ring moves ring_lo */
  LZ4D_H_GEN_OFF0, LZ4D_H_GEN_RING, LZ4D_H_GEN_GLOBAL, LZ4D_H_GEN_LONG, LZ4D_H_GEN_LAST,
  LZ4D_NHIT
};
#ifdef SIMT_EMU
static long long g_dbg_lz4d_batch_seqs = 0, g_dbg_lz4d_fast_seqs = 0, g_dbg_lz4d_general_seqs = 0, g_dbg_lz4d_dense_seqs = 0;
#define LZ4D_DBG(x) do { if (lane == 0) (x)++; } while (0)
#define LZ4D_DBGN(x, n) do { if (lane == 0) (x) += (n); } while (0)
static int g_lz4d_fail_line = 0;             /* emulator builds remember the first check that rejected the stream */
#define LZ4D_FAIL (g_lz4d_fail_line = g_lz4d_fail_line ? g_lz4d_fail_line : __LINE__, -1)
static long long g_lz4d_hit[LZ4D_NHIT];
#define LZ4D_HIT(id) do { if (lane == 0) g_lz4d_hit[id]++; } while (0)            /* warp-uniform branch */
#define LZ4D_HITL(id, c) do { if (c) g_lz4d_hit[id]++; } while (0)               /* per lane */
#else
#define LZ4D_DBG(x) do {} while (0)
#define LZ4D_DBGN(x, n) do {} while (0)
#define LZ4D_FAIL (-1)
#define LZ4D_HIT(id) do {} while (0)
#define LZ4D_HITL(id, c) do {} while (0)
#endif
#define LZ4D_RING 16384                      /* bytes of recent output mirrored in shared memory, per warp */
#define LZ4D_RMASK (LZ4D_RING - 1)
#define LZ4D_BATCH_OUT 320                   /* a batch writes < 320 bytes (11 sequences x <= 27) */
#define LZ4D_DENSE_LONG 8                    /* long matches (one extra length byte) a dense step takes inline */
#define LZ4D_DENSE_OUT 2624                  /* a dense step writes <= 24 x 18 + 8 x 273 bytes */
#define LZ4D_DENSE_MIN 4                     /* fewer chained 3-byte sequences than this: the 11-wide batch path is as good */
#define LZ4D_SCRATCH 256                     /* per-warp shared scratch after the ring: the batch table (lz4d_batch_table) */
#define LZ4D_SMEM (LZ4D_RING + LZ4D_SCRATCH)

/* ---- decoder copy routines, one per tier ----
 * lz4_decode_warp calls them inline; the pair decoder's copier warp (dev_lz4dpair.cuh) calls them on the fields of a
 * descriptor.  Each one writes its output both to `out` and to the ring, so that the ring keeps mirroring the most
 * recent output; none ends with a __syncwarp (the caller makes the bytes visible). */
enum { LZ4D_ZERO = 0, LZ4D_FROM_RING = 1, LZ4D_FROM_GLOBAL = 2, LZ4D_LONG = 3 };   /* how a general-path match is copied */
#define LZ4D_TBL_START 22                    /* batch table: 11 x {info, offset}, then 10 start-bit words */

/* dense step: lanes [0, cnt) hold one sequence each (kind 1: 4..18-byte match, kind 2: long match, lanes `longm`),
 * its output at dst and its source off bytes back -- before the step's first output byte */
DEV void lz4d_copy_dense(u8* out, smem_addr_t ring, int dst, int off, int ml, int kind, bool from_ring, int cnt,
                         unsigned longm) {
  const int lane = lane_id();
  const int match = dst - off;
  {
    /* every lane copies its own short match, 4 source bytes per step: from the ring (two aligned
     * words + funnel shift) or, for far offsets, from the output in global memory */
    const int mls = (lane < cnt && kind == 1) ? ml : 0;
    const int mlmax = __ballot_sync(FULLMASK, mls > 16) ? 18 : (__ballot_sync(FULLMASK, mls > 8) ? 16 : 8);
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
  /* the long ones, by the whole warp (their sources also lie before this step's output) */
  for (unsigned tm = longm; tm; tm &= tm - 1u) {
    const int t = __ffs((int)tm) - 1;
    const int td = __shfl_sync(FULLMASK, dst, t), tmt = __shfl_sync(FULLMASK, match, t), tl = __shfl_sync(FULLMASK, ml, t);
    const bool tring = __shfl_sync(FULLMASK, (int)from_ring, t) != 0;
    for (int k = lane; k < tl; k += 32) {
      const u32 v = tring ? smem_ld_u8(ring, (u32)(tmt + k) & LZ4D_RMASK) : (u32)out[tmt + k];
      out[td + k] = (u8)v;
      smem_st_u8(ring, (u32)(td + k) & LZ4D_RMASK, v);
    }
  }
}

/* one long match whose source overlaps its own output (small offsets): period copy by the warp */
DEV void lz4d_copy_lone(u8* out, smem_addr_t ring, int op, int len, int off, bool from_ring) {
  const int match = op - off;
  for (int k = lane_id(); k < len; k += 32) {             /* sources are all before `op`: no lane waits for another */
    const int src = match + (off >= len ? k : k % off);
    const u32 v = from_ring ? smem_ld_u8(ring, (u32)src & LZ4D_RMASK) : (u32)out[src];
    out[op + k] = (u8)v;
    smem_st_u8(ring, (u32)(op + k) & LZ4D_RMASK, v);
  }
}

/* the batch's sequence table (tbl[0..21]: {output offset | literals << 9 | input lane << 13, offset} by rank) and its
 * start bits (tbl[22..31]: bit y = a sequence starts at output byte y of the batch), written by the real lanes */
DEV void lz4d_batch_table(u32* tbl, int my_rank, int my_opre, int lit, int off) {
  const int lane = lane_id();
  if (lane < 10) tbl[LZ4D_TBL_START + lane] = 0;
  __syncwarp();
  if (my_rank >= 0) {
    tbl[2 * my_rank] = (u32)my_opre | ((u32)lit << 9) | ((u32)lane << 13);
    tbl[2 * my_rank + 1] = (u32)off;
    atomicOr(&tbl[LZ4D_TBL_START + (my_opre >> 5)], 1u << (my_opre & 31));
  }
}

/* the batch's `total` output bytes, 32 per instruction: lane y finds its sequence by counting start bits */
DEV void lz4d_copy_batch(const u8* in, u8* out, smem_addr_t ring, int ip, int op, int total, int ring_lo, const u32* tbl) {
  const int lane = lane_id();
  int kbase = 0;
  for (int r = 0; r * 32 < total; r++) {
    const u32 w = tbl[LZ4D_TBL_START + r];
    const int y = r * 32 + lane;
    if (y < total) {
      const int k = kbase + __popc(w & ((2u << lane) - 1u)) - 1;
      const u32 e0 = tbl[2 * k], offk = tbl[2 * k + 1];
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
    kbase += __popc(w);
  }
}

/* one short sequence (lit literals at in[ip+1..], then a match off bytes back), one lane per output byte */
DEV void lz4d_copy_single(const u8* in, u8* out, smem_addr_t ring, int ip, int op, int lit, int total, int off,
                          bool use_ring) {
  const int lane = lane_id();
  const int match = op + lit - off;
  if (lane < total) {
    u32 v;
    if (lane < lit) v = in[ip + 1 + lane];
    else if (use_ring) v = smem_ld_u8(ring, (u32)(match + lane - lit) & LZ4D_RMASK);
    else v = out[match + lane - lit];
    out[op + lane] = (u8)v;
    smem_st_u8(ring, (u32)(op + lane) & LZ4D_RMASK, v);
  }
}

/* len literals from in[lsrc..] to out[op..], then (mlen > 0) a match of mlen bytes off bytes back, copied as `how` says */
DEV void lz4d_copy_general(const u8* in, u8* out, smem_addr_t ring, int lsrc, int op, int len, int mlen, int off, int how) {
  const int lane = lane_id();
  for (int k = lane; k < len; k += 32) {
    const u32 v = in[lsrc + k];
    out[op + k] = (u8)v;
    smem_st_u8(ring, (u32)(op + k) & LZ4D_RMASK, v);
  }
  if (mlen == 0) return;
  op += len;
  const int match = op - off;
  __syncwarp();                                             /* earlier output must be visible to all lanes */
  if (how == LZ4D_ZERO) {
    for (int k = lane; k < mlen; k += 32) out[op + k] = 0;
  } else if (how != LZ4D_LONG) {
    /* sources lie before `op`; inside the ring they are not overwritten by this copy.  Far
     * sources are read from global memory, but the output still goes into the ring so that it
     * stays a mirror of the last 16 KiB */
    const bool from_ring = how == LZ4D_FROM_RING;
    for (int k0 = 0; k0 < mlen; k0 += 32) {
      const int k = k0 + lane;
      if (k < mlen) {
        const int src = match + (off >= mlen ? k : k % off);
        const u32 v = from_ring ? smem_ld_u8(ring, (u32)src & LZ4D_RMASK) : (u32)out[src];
        out[op + k] = (u8)v;
        smem_st_u8(ring, (u32)(op + k) & LZ4D_RMASK, v);
      }
    }
  } else warp_copy_match(out, op, match, mlen);             /* global sources; ring no longer mirrors this span */
}

/* The copies of the single-warp decoder: made on the spot, by the parsing warp.  `ring_ptr` is LZ4D_SMEM bytes of
 * warp-private shared memory: the ring, then the batch table. */
struct Lz4dWarpCopies {
  const u8* in;
  u8* out;
  u8* ring_ptr;
  smem_addr_t ring;
  DEV Lz4dWarpCopies(u8* out_, u8* ring_ptr_) : in(nullptr), out(out_), ring_ptr(ring_ptr_), ring(smem_addr(ring_ptr_)) {}
  DEV void start(const u8* in_) { in = in_; }
  DEV void dense(int dst, int off, int ml, int kind, bool from_ring, int cnt, unsigned longm) {
    lz4d_copy_dense(out, ring, dst, off, ml, kind, from_ring, cnt, longm);
    __syncwarp();
  }
  DEV void lone(int op, int len, int off, bool from_ring) { lz4d_copy_lone(out, ring, op, len, off, from_ring); __syncwarp(); }
  DEV u32* batch_table() { return (u32*)(ring_ptr + LZ4D_RING); }
  DEV void batch(int ip, int op, int total, int ring_lo) {
    __syncwarp();
    lz4d_copy_batch(in, out, ring, ip, op, total, ring_lo, batch_table());
    __syncwarp();
  }
  DEV void single(int ip, int op, int lit, int total, int off, bool use_ring) {
    lz4d_copy_single(in, out, ring, ip, op, lit, total, off, use_ring);
    __syncwarp();
  }
  DEV void literals(int lsrc, int op, int len) { lz4d_copy_general(in, out, ring, lsrc, op, len, 0, 0, LZ4D_ZERO); }
  DEV void match(int op, int mlen, int off, int how) {
    lz4d_copy_general(in, out, ring, 0, op, 0, mlen, off, how);
    __syncwarp();
  }
  DEV void finish() {}
};

/* LZ4_decompress_safe for one stream (lz4.c:2451-2456; safe-loop rules :2234-2436): the tier walk.
 * Returns the number of bytes written or -1.  offset==0 decodes to zeros, as in the reference.
 *
 * The walk keeps ip / op / ring_lo and decides, for every step, what is copied where; `cp` performs the copies
 * (Lz4dWarpCopies: the same warp, now; Lz4dPairCopies in dev_lz4dpair.cuh: a second warp, from a queue).  The ring
 * mirrors the most recent output so that match sources -- a few KiB back in >99% of the sequences of shuffled data --
 * come from shared memory instead of a global load behind the stores that produced them; `ring_lo` is where that
 * mirror begins to be valid: positions [max(ring_lo, op-RING), op) are in the ring. */
template <class Copies>
DEV int lz4d_walk(const u8* __restrict__ in, const int csize, const int cap, Copies& cp) {
  const int iend = csize, oend = cap;
  const int lane = lane_id();
  const StreamBase ib = make_stream_base(in);
  int ip = 0, op = 0, result = 0;
  int ring_lo = 0;
  if (cap == 0) return (csize == 1 && in[0] == 0) ? 0 : LZ4D_FAIL;   /* lz4.c:2062-2066 */
  if (csize == 0) return LZ4D_FAIL;
  cp.start(in);
  int dense_skip = 0, dense_back = 0;
  for (;;) {
    /* ---- dense path: a run of literal-free sequences, one per lane ----
     * The byte-planes of shuffled data decode to long chains of 3-byte sequences (token with
     * 0 literals and a 4..18 byte match, 16-bit offset).  If the sequence at ip is of that form the
     * next one starts at ip+3, so lane l parses the 3 bytes at ip+3l and the leading run of lanes
     * that all see this form are real sequences.  A prefix sum of the match lengths gives every
     * lane its output position; sequences whose source lies entirely before the batch's first
     * output byte are independent, and every lane copies its own match. */
    if (dense_skip > 0) dense_skip--;
    else if (ip + 112 <= iend && op + LZ4D_DENSE_OUT <= oend - LZ4_MFLIMIT) {
      u32 b0, b1, b2;
      ldp_win12(ib, ip + 3 * lane, b0, b1, b2);               /* bytes ip+3l .. ip+3l+11 (touches < ip+109) */
      lz4d_prefetch(in, ip + 256 + 128 * lane, lane < 2 ? iend : 0);
      /* Segments: lanes [c, e) see 3-byte sequences at byte shift s; the sequence that ends a
       * segment is very often a longer literal-free match with one extra length byte (token 0x0F,
       * offset, len): lane e takes it and the next segment starts one byte later (shift s+1). */
      int kind = 0, ml = 0, off = 0, c = 0, sft = 0;
      u32 w = b0;
      for (;;) {
        const u32 tok = w & 0xffu;
        const unsigned okm = __ballot_sync(FULLMASK, lane >= c && (tok >> 4) == 0u && (tok & 15u) != 15u);
        const unsigned stop = ~okm & ~((1u << c) - 1u);        /* first lane >= c that is not such a sequence */
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
      int cnt = c;                                             /* lanes [0, cnt) hold one sequence each */
      int incl = ml;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(FULLMASK, incl, d);
        if (lane >= d) incl += t;
      }
      const int dst = op + incl - ml, match = dst - off;
      /* first sequence that reads its own batch's output (or is invalid: off == 0, match < 0) ends the run;
       * 8 bytes of slack because the word-wise copy reads up to 7 bytes past the end of its source */
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
        cp.dense(dst, off, ml, kind, from_ring, cnt, longm);
        ip += 3 * cnt + __popc(longm); op += total;
        LZ4D_DBGN(g_dbg_lz4d_dense_seqs, cnt);
        dense_back = 0;
        continue;
      }
      /* a lone long match whose source overlaps its own output (small offsets) */
      {
        const u32 tw = __shfl_sync(FULLMASK, b0, 0);
        const int tlen = 19 + (int)(tw >> 24), toff = (int)((tw >> 8) & 0xffffu), tmatch = op - toff;
        if ((tw & 0xffu) == 0x0fu && (tw >> 24) != 255u && toff != 0 && tmatch >= 0 && op + tlen <= oend - LZ4_MFLIMIT) {
          const bool tring = toff <= LZ4D_RING - 512 && tmatch >= ring_lo;
          LZ4D_HIT(tring ? LZ4D_H_LONE_RING : LZ4D_H_LONE_GLOBAL);
          if (toff < tlen) LZ4D_HIT(LZ4D_H_LONE_PERIOD);
          cp.lone(op, tlen, toff, tring);
          ip += 4; op += tlen;
          LZ4D_DBG(g_dbg_lz4d_dense_seqs);
          dense_back = 0;
          continue;
        }
      }
      if (cnt > 0) LZ4D_HIT(LZ4D_H_DENSE_FEW);
      dense_back = dense_back < 8 ? dense_back + 1 : 8;   /* not that kind of data right here: back off */
      dense_skip = dense_back;
    }
    /* ---- batch path: up to 11 short sequences per round ----
     * Lane l speculates that a sequence starts at input byte ip+l and parses it from its own
     * 12-byte window.  Sequences whose offset reaches back past everything this batch can write
     * (>= LZ4D_BATCH_OUT) cannot depend on each other, so once the chain of real starts is known
     * (one ballot when every sequence is the 3-byte literal-free form, a shuffle walk otherwise)
     * all their output bytes are produced 32 per instruction. */
    if (ip + 49 <= iend && op + LZ4D_BATCH_OUT <= oend - LZ4_MFLIMIT) {   /* a 9-literal sequence of lane 31 ends at ip+41 <= iend-8 (lz4.c:2289) */
      u32 b0, b1, b2;
      ldp_win12(ib, ip + lane, b0, b1, b2);
      const u32 token = b0 & 0xffu;
      const int lit = (int)(token >> 4), mln = (int)(token & 15u);
      const int ob = 1 + lit;                                  /* window byte of the 16-bit offset (valid for lit <= 9: token, literals and offset fit the 12-byte window) */
      const u32 ow = ob < 4 ? __funnelshift_r(b0, b1, 8u * ob) : (ob < 8 ? __funnelshift_r(b1, b2, 8u * (ob - 4)) : b2 >> (8u * ((ob - 8) & 3)));
      const int off = (int)(ow & 0xffffu);
      const int L = 3 + lit, O = lit + mln + 4;
      const bool good = lit <= 9 && mln != 15 && off >= LZ4D_BATCH_OUT;
      int nseq = 0, consumed = 0, total = 0, my_rank = -1, my_opre = 0;
      const unsigned g3 = __ballot_sync(FULLMASK, good && lit == 0);
      if ((g3 & 0x49249249u) == 0x49249249u) {                 /* starts at lanes 0,3,...,30 */
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
        const int match = op + my_opre + lit - off;            /* meaningful on real lanes */
        if (__ballot_sync(FULLMASK, my_rank >= 0 && match < 0)) { result = LZ4D_FAIL; break; }   /* lz4.c:2356 */
        LZ4D_HIT((g3 & 0x49249249u) == 0x49249249u ? LZ4D_H_BATCH_FAST : LZ4D_H_BATCH_WALK);
        LZ4D_HITL(off <= LZ4D_RING - LZ4D_BATCH_OUT - 64 && match >= ring_lo ? LZ4D_H_BATCH_RING : LZ4D_H_BATCH_GLOBAL, my_rank >= 0);
        lz4d_batch_table(cp.batch_table(), my_rank, my_opre, lit, off);
        cp.batch(ip, op, total, ring_lo);
        ip += consumed; op += total;
        LZ4D_DBGN(g_dbg_lz4d_batch_seqs, nseq);
        continue;
      }
    }
    /* ---- single-sequence fast path: short sequence, source strictly before its own output ----
     * Token, literals (<= 9) and offset are parsed from one 12-byte register window, and the whole
     * sequence (<= 27 bytes) is produced by one predicated load/store step, one lane per output byte. */
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
        if (off >= total && op + total <= oend - LZ4_MFLIMIT) { /* no self-overlap; far from the end of the block */
          if (match < 0) { result = LZ4D_FAIL; break; }        /* lz4.c:2356 (off == 0 cannot get here: off >= total >= 4) */
          const bool use_ring = off <= LZ4D_RING - 64 && match >= ring_lo;
          LZ4D_HIT(use_ring ? LZ4D_H_SINGLE_RING : LZ4D_H_SINGLE_GLOBAL);
          cp.single(ip, op, lit, total, off, use_ring);
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
        if (len > oend) { result = LZ4D_FAIL; break; }        /* same verdict as the cpy>oend test below, no int overflow */
      } while (sb == 255);
      if (result < 0) break;
    }
    int cpy = op + len;
    const bool last = cpy > oend - LZ4_MFLIMIT || ip + len > iend - (2 + 1 + LZ4_LASTLITERALS);   /* lz4.c:2289-2331 */
    if (last && (ip + len != iend || cpy > oend)) { result = LZ4D_FAIL; break; }
    cp.literals(ip, op, len);                                 /* written even if the match turns out to be refused */
    if (len > LZ4D_RING - 64) { ring_lo = cpy - (LZ4D_RING - 64) > ring_lo ? cpy - (LZ4D_RING - 64) : ring_lo; LZ4D_HIT(LZ4D_H_GEN_LITBUMP); }
    if (last) { LZ4D_HIT(LZ4D_H_GEN_LAST); result = cpy; break; }
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
        if (mlen > oend) { result = LZ4D_FAIL; break; }       /* keeps `mlen` from overflowing on hostile input */
      } while (sb == 255);
      if (result < 0) break;
    }
    mlen += 4;
    if (match < 0) { result = LZ4D_FAIL; break; }             /* lz4.c:2356 */
    cpy = op + mlen;
    if (cpy > oend - LZ4_LASTLITERALS) { result = LZ4D_FAIL; break; }   /* lz4.c:2423 */
    int how = LZ4D_ZERO;
    if (off == 0) {
      /* not a valid stream, but LZ4_decompress_safe accepts it: every copy routine first clears the
       * destination word ("silence msan warning when offset==0", lz4.c:2386-2390; LZ4_memcpy_using_offset_base)
       * and then replicates it, so the match decodes to zeros */
      ring_lo = cpy;
      LZ4D_HIT(LZ4D_H_GEN_OFF0);
    } else if (mlen <= 2048) {
      how = off <= LZ4D_RING - 2048 - 64 && match >= ring_lo ? LZ4D_FROM_RING : LZ4D_FROM_GLOBAL;
      LZ4D_HIT(how == LZ4D_FROM_RING ? LZ4D_H_GEN_RING : LZ4D_H_GEN_GLOBAL);
    } else {
      how = LZ4D_LONG;
      ring_lo = cpy;
      LZ4D_HIT(LZ4D_H_GEN_LONG);
    }
    cp.match(op, mlen, off, how);
    op = cpy;
  }
  cp.finish();
  __syncwarp();
  return result;
}

/* one warp per stream; `ring_ptr`: LZ4D_SMEM bytes of warp-private shared memory */
DEV int lz4_decode_warp(const u8* __restrict__ in, const int csize, u8* out, const int cap, u8* ring_ptr) {
  Lz4dWarpCopies cp(out, ring_ptr);
  return lz4d_walk(in, csize, cap, cp);
}

/*
 * dev_lz4dpair.cuh -- LZ4 block decoder as a PAIR of warps per stream, sm_90a.
 *
 * lz4_decode_warp (dev_lz4.cuh) is one warp per stream and, on the hard byte-plane of shuffled data, a chain of
 * ~150 k dependent instructions: every step parses up to 32 sequences and then copies them, and a lone warp issues
 * one instruction every ~6 cycles.  Parsing step k+1 needs nothing from the copies of step k -- only the byte counts,
 * which the parse itself produces -- so the two halves run in two warps:
 *
 *   parser  runs the tier walk of dev_lz4.cuh (lz4d_walk: every tier, threshold and LZ4_decompress_safe check),
 *           keeps ip / op / ring_lo, and instead of copying writes a descriptor of the step (the arguments of the
 *           tier's copy routine) into a queue of LZ4P_Q slots in shared memory;
 *   copier  owns the output and the 16 KiB ring that mirrors it, takes the descriptors in order and calls the copy
 *           routines of dev_lz4.cuh on them -- the very functions the single-warp decoder calls inline.
 *
 * Hand-over with named barriers (bar.sync / bar.arrive, 64 threads): FULL(s) parser -> copier, EMPTY(s) back.
 * This file holds only that machinery: the slot layout, the barriers, the parser's side of the queue and the copier.
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
  u32 w[64];                                   /* DENSE: two words per lane; BATCH: the batch table (lz4d_batch_table) */
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

/* The copies of the pair, as lz4d_walk hands them over: one descriptor each, for the copier warp.  k counts the
 * descriptors of the current stream.  A general-path sequence is one descriptor: its literals wait (lsrc, lop, llen)
 * for its match, or for the end of the stream. */
struct Lz4dPairCopies {
  u8* out;
  Lz4pSlot* slots;
  int k;
  int lsrc, lop, llen;
  DEV Lz4dPairCopies(u8* out_, Lz4pSlot* slots_) : out(out_), slots(slots_), k(0), lsrc(0), lop(0), llen(0) {}
  /* one descriptor of scalars; lane 0 writes it */
  DEV void post(u32 type, u32 p0 = 0, u32 p1 = 0, u32 p2 = 0, u32 p3 = 0, u32 p4 = 0, u32 p5 = 0) {
    Lz4pSlot* q = lz4p_acquire(slots, k);
    if (lane_id() == 0) { q->type = type; q->p[0] = p0; q->p[1] = p1; q->p[2] = p2; q->p[3] = p3; q->p[4] = p4; q->p[5] = p5; }
    lz4p_publish(k);
  }
  DEV void start(const u8* in) {
    post(LZ4P_START, (u32)(u64)(uintptr_t)in, (u32)((u64)(uintptr_t)in >> 32), (u32)(u64)(uintptr_t)out, (u32)((u64)(uintptr_t)out >> 32));
  }
  /* lane l: w[2l] = dst, w[2l+1] = off | ml << 16 | kind << 28 | from_ring << 31 */
  DEV void dense(int dst, int off, int ml, int kind, bool from_ring, int cnt, unsigned longm) {
    Lz4pSlot* q = lz4p_acquire(slots, k);
    const int lane = lane_id();
    q->w[2 * lane] = (u32)dst;
    q->w[2 * lane + 1] = (u32)off | ((u32)ml << 16) | ((u32)kind << 28) | (from_ring ? 0x80000000u : 0u);
    if (lane == 0) { q->type = LZ4P_DENSE; q->p[0] = (u32)cnt; q->p[1] = longm; }
    lz4p_publish(k);
  }
  DEV void lone(int op, int len, int off, bool from_ring) { post(LZ4P_LONE, (u32)op, (u32)len, (u32)off, from_ring ? 1u : 0u); }
  /* the walk writes the batch table straight into the next slot */
  DEV u32* batch_table() { return lz4p_acquire(slots, k)->w; }
  DEV void batch(int ip, int op, int total, int ring_lo) {
    Lz4pSlot* q = &slots[k & (LZ4P_Q - 1)];                  /* acquired by batch_table */
    if (lane_id() == 0) { q->type = LZ4P_BATCH; q->p[0] = (u32)ip; q->p[1] = (u32)op; q->p[2] = (u32)total; q->p[3] = (u32)ring_lo; }
    lz4p_publish(k);
  }
  DEV void single(int ip, int op, int lit, int total, int off, bool use_ring) {
    post(LZ4P_SINGLE, (u32)ip, (u32)op, (u32)lit, (u32)total, (u32)off, use_ring ? 1u : 0u);
  }
  DEV void literals(int src, int op, int len) { lsrc = src; lop = op; llen = len; }
  DEV void match(int op, int mlen, int off, int how) {
    post(LZ4P_GENERAL, (u32)lsrc, (u32)lop, (u32)llen, (u32)mlen, (u32)off, (u32)how);
    llen = 0;
  }
  /* end of the stream: literals still waiting (the last ones, or those of a refused match) go out alone; the copier
   * takes END, and the parser waits until everything before it has been copied */
  DEV void finish() {
    if (llen > 0) post(LZ4P_GENERAL, (u32)lsrc, (u32)lop, (u32)llen);
    post(LZ4P_END);
    lz4p_drain(k);
  }
};

/* ---- copier: takes the descriptors in order and runs the copy routine each one names ---- */
DEV void lz4_pair_copier(u8* ring_ptr, Lz4pSlot* slots) {
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
      const int lane = lane_id();
      const u32 wd = *(const volatile u32*)&q->w[2 * lane], wx = *(const volatile u32*)&q->w[2 * lane + 1];
      lz4d_copy_dense(out, ring, (int)wd, (int)(wx & 0xffffu), (int)((wx >> 16) & 0xfffu), (int)((wx >> 28) & 3u),
                      (wx >> 31) != 0u, (int)p0, p1);
    } else if (type == LZ4P_LONE) {
      lz4d_copy_lone(out, ring, (int)p0, (int)p1, (int)p2, p3 != 0u);
    } else if (type == LZ4P_BATCH) {
      lz4d_copy_batch(in, out, ring, (int)p0, (int)p1, (int)p2, (int)p3, q->w);
    } else if (type == LZ4P_SINGLE) {
      lz4d_copy_single(in, out, ring, (int)p0, (int)p1, (int)p2, (int)p3, (int)p4, p5 != 0u);
    } else if (type == LZ4P_GENERAL) {
      lz4d_copy_general(in, out, ring, (int)p0, (int)p1, (int)p2, (int)p3, (int)p4, (int)p5);
    }
    __syncwarp();
    bar_arrive(LZ4P_BAR_EMPTY(s), 64);
    k = type == LZ4P_END ? 0 : k + 1;
  }
}

/* the parser warp: LZ4_decompress_safe for one stream, copies delegated.  Returns the number of bytes the stream decodes
 * to or -1; the copier has finished with the stream when this returns. */
DEV int lz4_pair_parse(const u8* __restrict__ in, const int csize, u8* out, const int cap, Lz4pSlot* slots) {
  Lz4dPairCopies cp(out, slots);
  return lz4d_walk(in, csize, cap, cp);
}

/* tell the copier that there are no more streams */
DEV void lz4_pair_quit(Lz4pSlot* slots) {
  if (lane_id() == 0) slots[0].type = LZ4P_QUIT;
  __syncwarp();
  __threadfence_block();
  bar_arrive(LZ4P_BAR_FULL(0), 64);
}

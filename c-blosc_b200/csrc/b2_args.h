/*
 * b2_args.h -- plain-C argument blocks shared by the host framing code
 * (blosc_b200.c), the CUDA backend (backend_cuda.cu) and the device kernels.
 */
#ifndef B2_ARGS_H
#define B2_ARGS_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { FILT_SHUFFLE = 0, FILT_UNSHUFFLE = 1, FILT_BITSHUFFLE = 2, FILT_BITUNSHUFFLE = 3 };
enum { B2_CODEC_BLOSCLZ = 0, B2_CODEC_LZ4 = 1, B2_CODEC_ZLIB = 2, B2_CODEC_ZSTD = 3, B2_CODEC_SNAPPY = 4 };

typedef struct FilterArgs {
  const uint8_t* src;
  uint8_t* dst;
  long long nbytes;       /* total bytes */
  int blocksize;          /* Blosc block size (last block may be shorter) */
  int typesize;
  int mode;
} FilterArgs;

typedef struct StreamMap {
  long long nbytes;      /* uncompressed size of the whole buffer */
  int blocksize;
  int nsplits;           /* streams per full block */
  int first_block;       /* first selected block (getitem decodes a sub-range) */
  int nfull;             /* number of selected full-size blocks */
  int leftover;          /* bytes of the (selected) short last block, 0 if none */
  int nstreams;          /* nfull*nsplits + (leftover ? 1 : 0) */
} StreamMap;

/* the per-workspace int32 words behind `result` / `queue` / `done` / `status` (zero between calls: the
 * last warp of every encode / decode launch puts the counters back) */
enum { B2_R_CBYTES = 0, B2_R_FITS = 1, B2_R_STATUS = 2, B2_R_QUEUE = 3, B2_R_DONE = 4, B2_R_STATUS_OUT = 5, B2_R_WORDS = 16 };
#define B2_FOLD_SCAN_MAX_BLOCKS 65536   /* above this the 1024-thread scan_kernel is launched instead of the in-kernel scan */

typedef struct ScanArgs {
  const int* csizes;
  const int* needs;
  int* bstarts;          /* [nblocks] out */
  int* result;           /* [0] = total cbytes (clamped to INT_MAX), [1] = fits */
  int nsplits, nfull, has_leftover;
  int blocksize, leftover;
  int serial;            /* 1: reproduce serial_blosc's per-split maxout clamp (blosc.c:646-651); 0: t_blosc's total-fit rule */
  long long destsize;
} ScanArgs;

typedef struct EncodeArgs {
  StreamMap map;
  const uint8_t* in;     /* filtered (or original) bytes, block-major */
  uint8_t* slots;        /* per-stream output slots at the same offsets as `in` */
  int* csizes;           /* [nstreams] compressed size; == stream length means "stored raw" */
  int* needs;            /* [nstreams] smallest `maxout` with which the codec would still have succeeded */
  int codec, clevel, accel, split_flag;
  int table_bytes;       /* shared-memory bytes per warp */
  int num_sms;           /* filled in by the backend (team kernel: spreads the walker warps over the SM sub-partitions) */
  int many;              /* other chunks are in flight on this device (frames): streams per SM matter more than latency */
  int* queue;            /* work counter: warps pull stream numbers from it.  It only ever counts up: a launch
                          * adds exactly nstreams + (warps launched) tickets, the backend keeps the running base */
  unsigned queue_base;   /* first ticket of this launch (filled in by the backend) */
  unsigned* queue_base_host;   /* HOST word behind it, owned by the workspace */
  int* done;             /* zero-initialised count of finished streams: the warp that completes it runs the scan */
  int fold_scan;         /* 1: that warp computes bstarts / cbytes / the fit verdict (scan) in this launch */
  ScanArgs scan;
} EncodeArgs;

/* ---- segment-parallel LZ4 parse (dev_lz4fast.cuh) ---- */
#ifndef B2_FAST_SEG
#define B2_FAST_SEG 256     /* bytes per segment (dev_lz4fast.cuh FAST_SEG) */
#endif
#define B2_FAST_WIN_MAX (64 * 1024)   /* bytes of a stream that one parse CTA keeps in shared memory */
typedef struct FastSeg {   /* one record per segment of FAST_SEG bytes */
  uint16_t nbytes;         /* bytes in the segment's slot (0: no match, the segment is all literals) */
  uint16_t l1;             /* literals in front of the segment's first match */
  uint16_t tail;           /* literals after its last match (the whole segment when nbytes == 0) */
  uint16_t lt;             /* slot position of the last sequence's token */
  uint16_t lm, lo;         /* length and offset of the last match (its length bytes are not in the slot) */
  uint16_t pad0, pad1;
  uint32_t dst;            /* by the stream scan: offset of the merged output inside the stream's LZ4 block,
                            * 0xffffffff when the segment only continues the previous segment's last match */
  uint32_t pin;            /* by the stream scan: literals pending in front of this segment */
  uint32_t run;            /* by the stream scan: final length of the last match (with the segments it swallowed) */
  uint32_t pad2;
} FastSeg;

typedef struct FastArgs {
  StreamMap map;
  const uint8_t* in;       /* filtered (or original) bytes, block-major */
  uint8_t* slots;
  uint16_t* prev;          /* [nbytes] hash-chain index written by index_kernel */
  FastSeg* segs;           /* stream-major: stream idx starts at idx * segs_full (the leftover stream comes last) */
  int* ptail;              /* [nstreams] literals after the stream's last match */
  int* csizes;
  int* needs;
  int segs_full, segs_left;        /* segments per full stream / of the leftover stream */
  int win_bytes;                   /* bytes per parse window (one CTA): multiple of 32 segments */
  int threads;                     /* threads of a parse CTA (<= segments per window; they draw segments from a counter) */
  int groups_full, groups_left;    /* windows per full stream / of the leftover stream */
  int depth, accel;
  int hash_mask;                   /* 0xffff: chains over 6-byte hashes (lz4); 0: over 4-byte hashes (lz4hc) */
  int lazy;                        /* matches shorter than this are weighed against the next position's match (lz4hc) */
  int* queue;
  unsigned queue_base;
  unsigned* queue_base_host;
  int* done;
  int fold_scan;
  ScanArgs scan;
  /* B2_CODEC_LZ4: the parse writes LZ4 bytes and segs, one warp per stream merges them (fscan_kernel).  The others
   * parse into sequence records (recs / nrec; segs and ptail are not used), then one warp per stream writes it:
   *   B2_CODEC_ZSTD    a zstd frame (dev_zstdenc.cuh);
   *   B2_CODEC_ZLIB    a zlib stream, from records with offsets <= 32768 (dev_deflate.cuh);
   *   B2_CODEC_SNAPPY  a snappy stream (dev_snappy.cuh); the last warp's block scan applies blosc_c's snappy maxout rule */
  int codec;
  uint32_t* recs;                  /* 64 records per segment, segment-major as segs */
  uint32_t* nrec;                  /* records per segment */
  int flevel;                      /* zlib's FLEVEL for the clevel (deflate.c), in the stream header */
  int ebsize;                      /* blocksize + 4 typesize: the per-block maxbytes of t_blosc's pool (blosc.c:1745) */
} FastArgs;

typedef struct CompactArgs {
  StreamMap map;
  const uint8_t* in;     /* raw splits are copied from here */
  const uint8_t* slots;
  const int* csizes;
  const int* bstarts;
  const int* result;
  uint8_t* dest;
  uint32_t hdr0;         /* version | versionlz<<8 | flags<<16 | typesize<<24 */
  int nbytes32, nblocks;
  const FastSeg* segs;   /* non-NULL: the compressed streams are fast-parsed segments to be stitched (dev_lz4fast.cuh) */
  const int* ptail;
  int segs_full, segs_left;
} CompactArgs;

typedef struct DecodeArgs {
  StreamMap map;
  const uint8_t* chunk;  /* whole compressed chunk */
  int cbytes;            /* header cbytes (bounds for every read) */
  uint8_t* out;          /* uncompressed (still filtered) bytes */
  long long out_shift;   /* subtracted from the buffer offset (getitem decodes into a small scratch) */
  int codec;
  int* status;           /* zero-initialised accumulator: 0 ok, else min of the negative error codes */
  int* queue;            /* work counter, see EncodeArgs */
  unsigned queue_base;
  unsigned* queue_base_host;
  int* done;             /* zero-initialised count of finished streams */
  int* status_out;       /* the last warp publishes the verdict here and zeroes the three words above */
  int many;              /* other calls are running on this device: streams per SM matter more than latency */
  const int* blocks;     /* NULL: the selected blocks are [first_block, first_block + nfull (+1)) of map.  Otherwise a
                          * device list of block numbers (getitems; map.first_block and out_shift are 0): the j-th
                          * listed block decodes to j * blocksize of a compact output, and a short last block can
                          * only be the last entry.  It is not part of StreamMap so that the encoders' arguments,
                          * and the code compiled from them, stay as they are. */
} DecodeArgs;

/* One item range of a getitems request: `len` = next.pos - pos bytes from src + `src` to dst + `dst`.  `pos` is the
 * exclusive prefix of the lengths, so the gather splits its work by bytes; the table ends with an entry whose pos is
 * the total.  The host plan lists only non-empty ranges; the GPU plan keeps empty ones, which copy nothing (next.pos ==
 * pos). */
typedef struct GatherRange {
  long long src, dst, pos;
} GatherRange;

typedef struct GatherArgs {
  const uint8_t* src;         /* decoded (unfiltered) scratch, or a memcpyed chunk's payload */
  uint8_t* dst;
  const GatherRange* ranges;  /* [nranges + 1] */
  int nranges;
  long long total;            /* bytes to copy = ranges[nranges].pos */
  const int* status;          /* NULL, or the decode verdict: the gather writes nothing when it is negative */
} GatherArgs;

/* blosc_getitem's bounds checks of one range (blosc.c:1633-1644), the one statement of them: the host plan of getitems
 * (blosc_b200.c getitem_range) and its GPU plan (dev_chunk.cuh plan_check_kernel) both call it.  0: the range is
 * valid and covers bytes [*b_lo, *b_hi), empty when b_hi <= b_lo; 1: `start` is out of bounds; 2: `start`+`nitems` is.
 * The stop wraps as the reference's int sum does. */
#ifdef __CUDACC__
#define B2_HD __host__ __device__
#else
#define B2_HD
#endif
static inline B2_HD int b2_range_check(int start, int nitems, int typesize, long long nbytes, long long* b_lo,
                                       long long* b_hi) {
  const int stop = (int)((unsigned)start + (unsigned)nitems);
  if (start < 0 || (long long)start * typesize > nbytes) return 1;
  if (stop < 0 || (long long)stop * typesize > nbytes) return 2;
  *b_lo = (long long)start * typesize; *b_hi = (long long)stop * typesize;
  return 0;
}

/* The frame's check of one range against its `total` items, the one statement of it: the host plan of frame getitems
 * (blosc_b200.c frame_getitems_host) and its GPU plan (dev_chunk.cuh fplan_check_kernel) both call it.  Nonzero: the
 * range is out of bounds.  No sum is formed, so nothing wraps at the u64 extremes. */
static inline B2_HD int b2_frame_range_bad(unsigned long long start, unsigned long long nitems,
                                           unsigned long long total) {
  return start > total || nitems > total - start;
}

/* What the GPU plan of getitems leaves for the host, read back with one small copy */
typedef struct GetitemsPlan {
  unsigned bad;          /* index of the first failing range; 0xffffffff when every range is valid */
  int nlisted;           /* touched blocks, listed in ascending order */
  int has_left;          /* whether the chunk's short last block is one of them */
  int pad;
  long long total;       /* bytes of all ranges */
  unsigned long long bad_box;   /* getslices: the first box whose corner fails (box_check_kernel); all ones when none */
} GetitemsPlan;

/* The tile state of one device-wide scan (dev_chunk.cuh plan_scan_kernel, single pass with decoupled look-back) */
typedef struct PlanScan {
  unsigned* ticket;      /* zeroed: CTAs take tiles in the order they start, so a tile only waits for running ones */
  unsigned* flag;        /* [tiles], zeroed: 1 when the tile's aggregate is published, 2 when its inclusive prefix is */
  void* agg;             /* [tiles] of the scan's value type */
  void* inc;             /* [tiles] */
} PlanScan;

/* getitems planned on the GPU from device-resident range lists: the gather table and the touched-block list the host
 * plan would build.  Kernels: plan_check_kernel, then (unless in_place) the block scans PLAN_COVER and PLAN_SLOT over
 * nblocks, then PLAN_POS over the ranges, which also fills the table. */
typedef struct PlanArgs {
  const int* starts;
  const int* nitems;
  int nranges;
  int typesize, blocksize, nblocks;
  int leftover;          /* the chunk has a short last block */
  long long nbytes;
  int in_place;          /* a memcpyed chunk in device memory: the gather reads the payload itself, no block list */
  long long* len;        /* [nranges] bytes of each range; 0 when it is empty or fails */
  int* cover;            /* [nblocks + 1], zeroed: +1 at each range's first block, -1 after its last; then coverage */
  int* slot;             /* [nblocks] position of a touched block in the list */
  int* blocks;           /* [nblocks] the touched blocks, ascending */
  GatherRange* ranges;   /* [nranges + 1] the gather table, in request order, empty ranges included */
  GetitemsPlan* rec;     /* zeroed but for rec->bad = 0xffffffff */
  PlanScan scan[3];      /* PLAN_COVER, PLAN_SLOT, PLAN_POS */
  const long long* dsts; /* NULL: range r lands at its position in dest; else at dsts[r] (frame pieces) */
} PlanArgs;
enum { PLAN_COVER = 0, PLAN_SLOT = 1, PLAN_POS = 2 };
#define PLAN_THREADS 256
#define PLAN_ITEMS 8
#define PLAN_TILE (PLAN_THREADS * PLAN_ITEMS)

/* What the GPU plan of frame getitems leaves for the host, read back with one small copy */
typedef struct FramePlan {
  unsigned long long bad;    /* index of the first failing range; all ones when every range is valid */
  long long total;           /* bytes of all ranges */
  long long npieces;         /* pieces of all chunks */
  long long ntouched;        /* chunks with at least one piece */
} FramePlan;

/* One touched chunk: its pieces are [base, base + count) of the piece lists */
typedef struct FrameTouch {
  long long chunk, base, count;
} FrameTouch;

/* frame getitems planned on the GPU from device-resident range lists: every range is cut at the chunk boundaries into
 * pieces, and each chunk's pieces are gathered into one bucket of the piece lists, which the chunk plan (PlanArgs with
 * dsts) then reads like range lists of its own.  Kernels: fplan_check_kernel, the scans FPLAN_DST over the ranges and
 * FPLAN_COUNT, FPLAN_BASE, FPLAN_TOUCH over the chunks, then (once the host knows how many pieces there are)
 * fplan_scatter_kernel. */
typedef struct FramePlanArgs {
  const unsigned long long* starts;   /* NULL: every start is 0 (only the counts are checked) */
  const unsigned long long* nitems;
  long long nranges;
  unsigned long long total_items;     /* the frame's nbytes / typesize */
  long long ipc;                      /* items per chunk */
  int typesize;
  long long nchunks;
  long long* dst;          /* [nranges] bytes of each range (0 when it fails), then its offset in dest */
  long long* count;        /* [nchunks + 1], zeroed: +1 at each range's first chunk, -1 after its last; then pieces */
  long long* cursor;       /* [nchunks] the first free slot of each chunk's bucket */
  FrameTouch* touched;     /* [nchunks] the touched chunks, ascending */
  int* pstart;             /* [npieces] first item of each piece inside its chunk */
  int* pnitems;            /* [npieces] its items */
  long long* pdst;         /* [npieces] its offset in dest */
  FramePlan* rec;          /* zeroed but for rec->bad = all ones */
  PlanScan scan[4];        /* FPLAN_DST .. FPLAN_TOUCH, at [mode - FPLAN_DST] */
} FramePlanArgs;
enum { FPLAN_DST = 3, FPLAN_COUNT = 4, FPLAN_BASE = 5, FPLAN_TOUCH = 6 };

/* A box of an N-d C-order array (blosc_b200_getslice): items start[k], start[k] + step[k], ... below stop[k] of each
 * dimension, none of them empty.  The host builds it normalised (blosc_b200.c box_build): each stop is the last
 * selected coordinate + 1, a dimension that selects one coordinate has step 1, and every dimension that the box covers
 * whole with step 1 is merged into the dimension before it when that one's step is 1 too, so the innermost run of
 * consecutive flat items is as long as the box allows.  A box whose steps are all 1 is then `stepped` 0.  Its
 * arithmetic is the three functions below, shared by the host (which touched chunks, where their output starts) and
 * the kernels (which blocks a chunk's part touches, where each output byte comes from).  Each takes `stepped`, which
 * the kernels pass as a template constant: with 0 the step code folds away and step / ext are never read.  Every loop
 * runs over the fixed B2_BOX_MAXDIM with a guard, so the kernels index the box with constants only. */
#define B2_BOX_MAXDIM 8
typedef struct B2Box {
  int ndim;                           /* dimensions after merging, 1..B2_BOX_MAXDIM */
  int stepped;                        /* some step[k] > 1 */
  long long start[B2_BOX_MAXDIM];
  long long stop[B2_BOX_MAXDIM];      /* the last selected coordinate + 1 */
  long long stride[B2_BOX_MAXDIM];    /* flat items per step of dimension k: the product of the shape after k */
  long long inner[B2_BOX_MAXDIM];     /* box items per step of dimension k: the product of the extents after k */
  long long run;                      /* items of one innermost run: the extent of the last dimension, or 1 when its
                                       * step is > 1 */
  long long nitems;                   /* items of the whole array: b2_box_next's end sentinel */
  long long count;                    /* items of the box */
  long long step[B2_BOX_MAXDIM];      /* >= 1 */
  long long ext[B2_BOX_MAXDIM];       /* selected coordinates of dimension k */
} B2Box;

/* a / b for a >= 0, b > 0.  On the device it makes no call to the 64-bit division routine, whose saved registers
 * would spill in the box kernels: a 32-bit division when both fit, else a double estimate refined once in double and
 * corrected by one in exact integer arithmetic (the remainders are below 2^63, so the unsigned products are exact). */
static inline B2_HD long long b2_box_div(long long a, long long b) {
#ifdef __CUDA_ARCH__
  long long q, r;
  if ((((unsigned long long)a | (unsigned long long)b) >> 32) == 0) return (long long)((unsigned)a / (unsigned)b);
  q = (long long)((double)a / (double)b);
  r = (long long)((unsigned long long)a - (unsigned long long)q * (unsigned long long)b);
  q += (long long)((double)r / (double)b);
  r = (long long)((unsigned long long)a - (unsigned long long)q * (unsigned long long)b);
  return r < 0 ? q - 1 : r >= b ? q + 1 : q;
#else
  return a / b;
#endif
}

/* The smallest flat index >= x (0 <= x <= nitems) that lies in the box; nitems when there is none.  A coordinate
 * inside [start, stop) but off its dimension's lattice moves up to the next lattice point, or carries past the last. */
static inline B2_HD long long b2_box_next(const B2Box* b, long long x, int stepped) {
  long long c[B2_BOX_MAXDIM], r = x, v = 0, lift = 0;
  int k, bad = -1, below = 0, p = -1;
#pragma unroll
  for (k = 0; k < B2_BOX_MAXDIM; k++) {
    c[k] = 0;
    if (k < b->ndim) {
      c[k] = b2_box_div(r, b->stride[k]);
      r -= c[k] * b->stride[k];
      if (bad < 0 && (c[k] < b->start[k] || c[k] >= b->stop[k])) { bad = k; below = c[k] < b->start[k]; }
      else if (stepped && bad < 0) {
        const long long o = c[k] - b->start[k], q = b2_box_div(o, b->step[k]);
        if (o != q * b->step[k]) {    /* off the lattice: up to the next point (>= 1) when it is below stop */
          bad = k; lift = b->start[k] + (q + 1) * b->step[k]; below = lift < b->stop[k];
        }
      }
    }
  }
  if (bad < 0) return x;
  if (below) {                      /* dimension `bad` moves up to its start (or lift), the ones after it to theirs */
    p = bad;
#pragma unroll
    for (k = 0; k < B2_BOX_MAXDIM; k++) if (k == bad) v = b->start[k];
    if (stepped && lift) v = lift;
  } else {                          /* past the box in `bad`: carry into the last dimension before it that has room */
#pragma unroll
    for (k = B2_BOX_MAXDIM - 1; k >= 0; k--) {
      const long long s = stepped ? b->step[k] : 1;
      if (p < 0 && k < bad && c[k] + s < b->stop[k]) { p = k; v = c[k] + s; }
    }
    if (p < 0) return b->nitems;
  }
  r = 0;
#pragma unroll
  for (k = 0; k < B2_BOX_MAXDIM; k++)
    if (k < b->ndim) r += (k < p ? c[k] : k == p ? v : b->start[k]) * b->stride[k];
  return r;
}

/* How many box items have a flat index < x (0 <= x <= nitems) */
static inline B2_HD long long b2_box_rank(const B2Box* b, long long x, int stepped) {
  long long r = x, rank = 0;
  int k;
#pragma unroll
  for (k = 0; k < B2_BOX_MAXDIM; k++) {
    if (k < b->ndim) {
      const long long c = b2_box_div(r, b->stride[k]);
      r -= c * b->stride[k];
      if (c < b->start[k]) return rank;
      if (stepped) {
        long long o, q;
        if (c >= b->stop[k]) return rank + b->ext[k] * b->inner[k];
        o = c - b->start[k]; q = b2_box_div(o, b->step[k]);
        rank += q * b->inner[k];
        if (o != q * b->step[k]) return rank + b->inner[k];   /* off the lattice: lattice point q lies before x */
      } else {
        if (c >= b->stop[k]) return rank + (b->stop[k] - b->start[k]) * b->inner[k];
        rank += (c - b->start[k]) * b->inner[k];
      }
    }
  }
  return rank;
}

/* The flat index of box item p (0 <= p < count, C order inside the box) */
static inline B2_HD long long b2_box_unrank(const B2Box* b, long long p, int stepped) {
  long long f = 0;
  int k;
#pragma unroll
  for (k = B2_BOX_MAXDIM - 1; k >= 0; k--) {
    if (k < b->ndim) {
      long long q = p;
      if (k > 0) {
        const long long e = stepped ? b->ext[k] : b->stop[k] - b->start[k];
        p = b2_box_div(p, e);
        q -= p * e;
      }
      f += (b->start[k] + (stepped ? q * b->step[k] : q)) * b->stride[k];
    }
  }
  return f;
}

/* The plan of one chunk's part of a box: box_touch_kernel marks in plan.cover every block that holds a byte of it, then
 * the PLAN_SLOT scan of the getitems plan (plan.cover, slot, blocks, rec, leftover, scan[PLAN_SLOT]) lists them.  The
 * chunk holds the array's flat items [window, window + nbytes / typesize). */
typedef struct BoxPlanArgs {
  B2Box box;
  long long window;
  PlanArgs plan;
} BoxPlanArgs;

/* box_gather_kernel: box items [p0, p0 + total / typesize) in C order, all inside the chunk's window, to dst.  slot
 * NULL: src is the chunk's bytes in place (a memcpyed payload); else block b of the chunk is at src + slot[b] *
 * blocksize (the compact scratch of the listed blocks). */
typedef struct BoxGatherArgs {
  B2Box box;
  long long window;
  long long p0;
  long long total;            /* bytes to write */
  int typesize, blocksize;
  const int* slot;
  const uint8_t* src;
  uint8_t* dst;
  const int* status;          /* NULL, or the decode verdict: the gather writes nothing when it is negative */
} BoxGatherArgs;

/* A batch of boxes of one extent (blosc_b200_getslices).  The box at the origin, `box` (start 0, stop = extent, after
 * the same merge), is shared by all of them: box i is that box moved by the flat offset off[i] = sum of corner[k] *
 * stride[k], so its items, ranks and unranks are the origin box's shifted by off[i] (box_next_at and the gather, in
 * dev_chunk.cuh).  span: flat items from a box's first item to its last, the same for every box.
 *
 * box_check_kernel, one thread per box: box i's corner is starts[i][0..ndim) in the caller's dimensions, and it fails
 * when a coordinate is below 0 or above hi[k] = shape[k] - extent[k].  The first failing box goes to *bad by
 * atomicMin; every box's offset goes to off[i] (0 for a failing box, so the launches that follow stay in bounds).
 * Frame only (touched != NULL): touched[c] = 1 for every chunk c, of ipc items, that holds an item of some box. */
typedef struct BoxCheckArgs {
  B2Box box;
  const long long* starts;
  long long nboxes, span;
  int ndim, pad;
  long long hi[B2_BOX_MAXDIM];
  long long stride[B2_BOX_MAXDIM];    /* flat items per step of the caller's dimension k */
  long long* off;
  unsigned long long* bad;
  int* touched;
  long long ipc, nchunks;
} BoxCheckArgs;

/* The plan of one chunk's part of a batch: boxes_touch_kernel marks in plan.cover every block that holds a byte of some
 * box (it only stores 1s; plan.cover starts zeroed), then the PLAN_SLOT scan lists them, as for one box.  Work item
 * (i, j), j < per_box, tests the j-th block of box i's span inside the chunk, which holds the array's flat items
 * [window, window + nbytes / typesize).  part != NULL (a frame): item (i, 0) also writes box i's part of the chunk,
 * the bytes [part[2i], part[2i + 1]) of the box's output whose items lie in the chunk, for the gather. */
typedef struct BoxesPlanArgs {
  B2Box box;
  const long long* off;
  long long nboxes, per_box, span, window;
  long long* part;
  int in_place, pad;          /* a memcpyed device chunk: the parts only, no block is marked */
  PlanArgs plan;
} BoxesPlanArgs;

/* boxes_gather_kernel: the batch's output, box i's C-order items at i * count * typesize, total bytes in all, to dst.
 * part != NULL: the chunk holds only part of each box (a frame, BoxesPlanArgs.part), and box i's bytes outside it are
 * skipped; NULL: the chunk holds every box.  slot / src / status as in BoxGatherArgs. */
typedef struct BoxesGatherArgs {
  B2Box box;
  const long long* off;
  const long long* part;
  long long window, total;
  int typesize, blocksize;
  const int* slot;
  const uint8_t* src;
  uint8_t* dst;
  const int* status;
} BoxesGatherArgs;

/* An orthogonal index selection of an N-d C-order array (blosc_b200_getoindex): numpy's a[np.ix_(...)], where each
 * dimension is either a slice (start, step, ext coordinates) or a list of coordinates in device memory, in any order
 * and with repeats.  The host builds it (blosc_b200.c osel_build) with B2Box's merging of the slice dimensions: a whole
 * step-1 slice merges into the dimension before it when that one is a step-1 slice too; a list never merges.  The run
 * is the innermost extent when the innermost dimension is a step-1 slice, else one item.  Position q of dimension k is
 * the coordinate list[k][q], or start[k] + q * step[k]. */
typedef struct B2OSel {
  int ndim;                           /* dimensions after merging, 1..B2_BOX_MAXDIM */
  int kdim[B2_BOX_MAXDIM];            /* the caller's dimension of each list, for the bad-entry key */
  long long start[B2_BOX_MAXDIM];
  long long step[B2_BOX_MAXDIM];
  long long ext[B2_BOX_MAXDIM];       /* positions of dimension k: n_k */
  long long shape[B2_BOX_MAXDIM];     /* the dimension's extent in the array: a list entry must lie in [0, shape) */
  long long stride[B2_BOX_MAXDIM];    /* flat items per coordinate of dimension k */
  const long long* list[B2_BOX_MAXDIM];   /* NULL for a slice */
  long long lbase[B2_BOX_MAXDIM];     /* entries of the lists before list k, in the check's numbering */
  long long run;                      /* items of one run */
  long long slab;                     /* items of the selection per position of dimension 0 */
  long long count;                    /* items of the selection */
  long long nruns;                    /* count / run */
  long long nentries;                 /* entries of all lists */
} B2OSel;

/* The flat index of selection item p (0 <= p < count), or -1 when a list entry it reads lies outside its dimension
 * (the check reports those; the plan must not index with them).  Only the kernels call it: the lists are device
 * memory. */
static inline B2_HD long long b2_osel_unrank(const B2OSel* s, long long p) {
  long long f = 0;
  int k, bad = 0;
#pragma unroll
  for (k = B2_BOX_MAXDIM - 1; k >= 0; k--) {
    if (k < s->ndim) {
      long long q = p, c;
      if (k > 0) {
        p = b2_box_div(p, s->ext[k]);
        q -= p * s->ext[k];
      }
      c = s->list[k] ? s->list[k][q] : s->start[k] + q * s->step[k];
      bad |= c < 0 || c >= s->shape[k];
      f += c * s->stride[k];
    }
  }
  return bad ? -1 : f;
}

/* oindex_touch_kernel over work items [0, (check ? nentries : 0) + r1 - r0).  The first nentries check the list
 * entries: an entry outside its dimension puts the key (caller's dimension << 56 | position) to *bad by atomicMin, so
 * the first bad entry wins.  The rest take one run each, the runs [r0, r1) (a frame's chunk: those of the output
 * bytes its gather walks).  touched != NULL (a frame): the run flags every
 * chunk, of ipc items, that holds one of its items.  Else the run marks in plan.cover every block of the chunk, which
 * holds the array's flat items [window, window + nbytes / typesize), that holds a byte of it (it only stores 1s; cover
 * starts zeroed), and the PLAN_SLOT scan lists them. */
typedef struct OIndexPlanArgs {
  B2OSel sel;
  long long window;
  int check, pad;
  long long r0, r1;
  unsigned long long* bad;
  int* touched;
  long long ipc;
  PlanArgs plan;
} OIndexPlanArgs;

/* oindex_gather_kernel: the output bytes [g0, g1) of the selection (each a multiple of the run's bytes), at dst + byte.
 * clip (a frame): only the items inside the chunk's window [window, wend) are written; a position of dimension 0
 * whose coordinate's flat span misses the window is skipped whole.  slot / src / status as in BoxGatherArgs. */
typedef struct OIndexGatherArgs {
  B2OSel sel;
  long long window, wend;
  long long g0, g1;
  int typesize, blocksize;
  int clip, pad;
  const int* slot;
  const uint8_t* src;
  uint8_t* dst;
  const int* status;
} OIndexGatherArgs;

/* One touched chunk of a chunk grid (blosc_b200_grid_getslice) and its part of the selection, as two boxes with the
 * same extents: `box` in the chunk's own coordinates (over the chunk shape, with the selection's steps) and `out` in
 * the output array's (step 1), so box item p of the one is box item p of the other.  placed_gather_kernel copies run q
 * of `run` items from box's unrank of q * run in the chunk to out's unrank of q * run in dst; `run` is the shorter of
 * the two boxes' runs (each is a product of trailing extents, so it divides the longer).  placed_fill_kernel (a missing
 * chunk; box, slot, src and status unused) writes the itemsize-byte pattern `fill`, or zeros when it is NULL, over out
 * instead.  slot / src / status as in BoxGatherArgs. */
typedef struct PlacedGatherArgs {
  B2Box box;
  B2Box out;
  long long run;
  long long total;            /* bytes of the part: out.count * itemsize */
  long long itemsize;
  int blocksize, pad;
  const int* slot;
  const uint8_t* src;
  const uint8_t* fill;        /* device memory */
  uint8_t* dst;
  const int* status;
} PlacedGatherArgs;

#ifdef __cplusplus
}
#endif
#endif

/*
 * blosc_b200.h -- C ABI of libblosc_b200.so, a CUDA (H100, sm_90a) drop-in for the hot path
 * of c-blosc 1.21: the blocked shuffle -> LZ compress / LZ decompress -> unshuffle
 * pipeline behind blosc_compress_ctx() / blosc_decompress_ctx() / blosc_getitem().
 *
 * Every declaration below replaces the reference declaration cited next to it
 * (paths are relative to the reference checkout, blosc/blosc.h) and keeps its name,
 * argument meaning, return codes and on-wire chunk format (README_CHUNK_FORMAT.rst).
 * Differences a caller can observe:
 *   - `src` / `dest` may be host pointers (as in the reference; the library stages them
 *     over PCIe) OR CUDA device pointers (detected with cudaPointerGetAttributes), so a
 *     GPU-resident caller never leaves HBM;
 *   - `numinternalthreads` is validated like the reference but otherwise ignored: the
 *     CUDA grid is the thread pool (reference blosc.c:1706-1949);
 *   - "blosclz" and "lz4" chunks are byte-identical to the reference's; "lz4hc" is accepted and
 *     written in its (= LZ4's, blosc.h:96) format by a hash-chain parser run with LZ4HC's search
 *     effort -- every reference build decodes the chunks, the header is the reference's, the
 *     bytes are not LZ4_compress_HC's; other compressors report -5 exactly like a reference built
 *     with -DDEACTIVATE_ZLIB/ZSTD/SNAPPY (blosc.c:573,1197-1208).  Decoding is wider: zlib and
 *     zstd chunks decode too (serial GPU decoders, one lane per stream); snappy chunks report -5 unless
 *     BLOSC_B200_SNAPPY=1;
 *   - with the environment variable BLOSC_B200_ZSTD=1 (read on every call) the library behaves
 *     like a reference built with zstd: "zstd" is listed, named and encoded (segment-parallel GPU
 *     encoder, one zstd frame per block).  The header is the reference's and every reference build
 *     with zstd decodes the chunks, but the frames are not ZSTD_compress's bytes;
 *   - with BLOSC_B200_ZLIB=1 (read on every call, independent of BLOSC_B200_ZSTD) it behaves like a
 *     reference built with zlib: "zlib" is listed, named and encoded (segment-parallel GPU encoder,
 *     one zlib stream per split).  Every zlib reads the streams, but they are not compress2's bytes
 *     and their sizes differ;
 *   - with BLOSC_B200_SNAPPY=1 (read on every call, independent of the other two) it behaves like a reference built
 *     with snappy: "snappy" is listed, named, encoded and decoded on the GPU (one snappy stream per split, valid snappy
 *     but no snappy release's bytes; blosc_get_complib_info reports version "unknown");
 *   - there is no CPU codec: without a CUDA device every compress/decompress call
 *     prints a message on stderr and returns -1.
 */
#ifndef BLOSC_B200_H
#define BLOSC_B200_H

#include <limits.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- constants, blosc.h:20-117 ---- */
#define BLOSC_VERSION_MAJOR 1
#define BLOSC_VERSION_MINOR 21
#define BLOSC_VERSION_RELEASE 7
#define BLOSC_VERSION_STRING "1.21.7.dev-b200"
#define BLOSC_VERSION_DATE "$Date:: 2024-06-24 #$"
#define BLOSC_VERSION_FORMAT 2
#define BLOSC_MIN_HEADER_LENGTH 16
#define BLOSC_MAX_OVERHEAD BLOSC_MIN_HEADER_LENGTH
#define BLOSC_MAX_BUFFERSIZE (INT_MAX - BLOSC_MAX_OVERHEAD)
#define BLOSC_MAX_TYPESIZE 255
#define BLOSC_MAX_BLOCKSIZE ((INT_MAX - BLOSC_MAX_TYPESIZE * sizeof(int32_t)) / 3)
#define BLOSC_MAX_THREADS 256
#define BLOSC_NOSHUFFLE 0
#define BLOSC_SHUFFLE 1
#define BLOSC_BITSHUFFLE 2
#define BLOSC_DOSHUFFLE 0x1
#define BLOSC_MEMCPYED 0x2
#define BLOSC_DOBITSHUFFLE 0x4
#define BLOSC_BLOSCLZ 0
#define BLOSC_LZ4 1
#define BLOSC_LZ4HC 2
#define BLOSC_SNAPPY 3
#define BLOSC_ZLIB 4
#define BLOSC_ZSTD 5
#define BLOSC_BLOSCLZ_COMPNAME "blosclz"
#define BLOSC_LZ4_COMPNAME "lz4"
#define BLOSC_LZ4HC_COMPNAME "lz4hc"
#define BLOSC_SNAPPY_COMPNAME "snappy"
#define BLOSC_ZLIB_COMPNAME "zlib"
#define BLOSC_ZSTD_COMPNAME "zstd"
#define BLOSC_BLOSCLZ_LIB 0
#define BLOSC_LZ4_LIB 1
#define BLOSC_SNAPPY_LIB 2
#define BLOSC_ZLIB_LIB 3
#define BLOSC_ZSTD_LIB 4
#define BLOSC_BLOSCLZ_FORMAT BLOSC_BLOSCLZ_LIB
#define BLOSC_LZ4_FORMAT BLOSC_LZ4_LIB
#define BLOSC_LZ4HC_FORMAT BLOSC_LZ4_LIB
#define BLOSC_SNAPPY_FORMAT BLOSC_SNAPPY_LIB
#define BLOSC_ZLIB_FORMAT BLOSC_ZLIB_LIB
#define BLOSC_ZSTD_FORMAT BLOSC_ZSTD_LIB
#define BLOSC_BLOSCLZ_VERSION_FORMAT 1
#define BLOSC_LZ4_VERSION_FORMAT 1
#define BLOSC_SNAPPY_VERSION_FORMAT 1
#define BLOSC_ZLIB_VERSION_FORMAT 1
#define BLOSC_ZSTD_VERSION_FORMAT 1
#define BLOSC_ALWAYS_SPLIT 1
#define BLOSC_NEVER_SPLIT 2
#define BLOSC_AUTO_SPLIT 3
#define BLOSC_FORWARD_COMPAT_SPLIT 4

/* ---- the hot path (the drop-in boundary) ---- */

/* replaces blosc.h:245-248 / blosc.c:1282-1308.  >0 compressed bytes; 0 does not fit in
 * destsize / input too large / destsize < 16; -10 bad clevel|doshuffle|typesize; -5 codec not
 * available; -1 internal / no device. */
int blosc_compress_ctx(int clevel, int doshuffle, size_t typesize, size_t nbytes, const void* src,
                       void* dest, size_t destsize, const char* compressor, size_t blocksize,
                       int numinternalthreads);

/* replaces blosc.h:301-302 / blosc.c:1520-1535.  >=0 decompressed bytes; -1 malformed chunk or
 * destsize too small; -5 / -9 unknown codec / codec format version. */
int blosc_decompress_ctx(const void* src, void* dest, size_t destsize, int numinternalthreads);

/* replaces blosc.h:312 / blosc.c:1574-1703.  `start`, `nitems` in elements of the chunk's typesize. */
int blosc_getitem(const void* src, int start, int nitems, void* dest);

/* ---- global-state front-end over the ctx path (blosc.h:127-222,256-299,321-352) ---- */
void blosc_init(void);                                                   /* blosc.h:142 */
void blosc_destroy(void);                                                /* blosc.h:151 */
int  blosc_compress(int clevel, int doshuffle, size_t typesize, size_t nbytes, const void* src,
                    void* dest, size_t destsize);                        /* blosc.h:221-222 */
int  blosc_decompress(const void* src, void* dest, size_t destsize);     /* blosc.h:279 */
int  blosc_get_nthreads(void);                                           /* blosc.h:321 */
int  blosc_set_nthreads(int nthreads);                                   /* blosc.h:332 */
const char* blosc_get_compressor(void);                                  /* blosc.h:338 */
int  blosc_set_compressor(const char* compname);                         /* blosc.h:352 */
int  blosc_get_blocksize(void);                                          /* blosc.h:494 */
void blosc_set_blocksize(size_t blocksize);                              /* blosc.h:506 */
void blosc_set_splitmode(int splitmode);                                 /* blosc.h:527 */
int  blosc_free_resources(void);                                         /* blosc.h:411 */

/* ---- names / introspection (host-only header readers) ---- */
int  blosc_compcode_to_compname(int compcode, const char** compname);    /* blosc.h:364 */
int  blosc_compname_to_compcode(const char* compname);                   /* blosc.h:374 */
const char* blosc_list_compressors(void);                                /* blosc.h:388 */
const char* blosc_get_version_string(void);                              /* blosc.h:396 */
int  blosc_get_complib_info(const char* compname, char** complib, char** version);   /* blosc.h:417 */
void blosc_cbuffer_sizes(const void* cbuffer, size_t* nbytes, size_t* cbytes, size_t* blocksize);  /* blosc.h:431 */
int  blosc_cbuffer_validate(const void* cbuffer, size_t cbytes, size_t* nbytes);                   /* blosc.h:441 */
void blosc_cbuffer_metainfo(const void* cbuffer, size_t* typesize, int* flags);                    /* blosc.h:459 */
void blosc_cbuffer_versions(const void* cbuffer, int* version, int* compversion);                  /* blosc.h:468 */
const char* blosc_cbuffer_complib(const void* cbuffer);                                            /* blosc.h:477 */

/* ---- blosc_b200 extensions (not in the reference) ---- */

/* One filter over one block, the GPU counterpart of the reference's internal
 * blosc_internal_{shuffle,unshuffle,bitshuffle,bitunshuffle} (blosc/shuffle.c:367-443) that
 * its unit tests call.  mode: 0 shuffle, 1 unshuffle, 2 bitshuffle, 3 bitunshuffle.
 * src/dest host or device.  Returns 0, or -1 on device failure. */
int blosc_b200_filter(int mode, size_t typesize, size_t blocksize, const void* src, void* dest);

/* Many item ranges of one chunk in one call.  Range r covers items [starts[r], starts[r] + nitems[r]) in elements of
 * the chunk's typesize.  Each range is validated exactly as blosc_getitem validates one.  Ranges may be unsorted,
 * overlap or repeat.  They are written back to back into dest in request order.  src / dest are host or device.
 * Every block that some range overlaps is decoded once, by one decode launch, however many ranges touch it.  Returns
 * the total bytes written, or the code blosc_getitem would return for the first range that fails (with its stderr
 * message); in that case nothing is written to dest.  nranges == 0 returns 0 and reads neither list.
 *
 * starts / nitems may each be host or device memory.  When either is device memory the read is planned on the GPU
 * (a host list is uploaded with the other), so the lists never come back to the host; the results are the same as
 * with host lists.  Device lists must be on the device the call runs on: that of src or dest when either is device
 * memory, else the one chosen with blosc_b200_set_device; otherwise the call returns -1 before anything is read or
 * written.  The call runs on blocking streams, ordered after work on the legacy default stream; lists produced on
 * other non-blocking streams must be synchronised first, as src must. */
long long blosc_b200_getitems(const void* src, int nranges, const int* starts, const int* nitems, void* dest);

/* A box of an N-d array in one call.  The chunk holds a C-order array of `shape` (ndim entries, 1..8) in items of the
 * chunk's typesize; items [start[k], stop[k]) of each dimension k are written to dest as one contiguous C-order array
 * of extents stop - start (numpy: a[start[0]:stop[0], ..., start[ndim-1]:stop[ndim-1]], made contiguous).  shape /
 * start / stop are host memory; src / dest are host or device memory, and the call runs on the device getitems would
 * use.  Only the blocks that hold a byte of the box are decoded, and the read is planned on the GPU from the box
 * alone: the launches do not grow with the number of innermost runs.  Returns the bytes written, prod(stop - start) *
 * typesize; 0 for an empty box, with nothing launched.  -1 with a message on stderr, before anything is launched or
 * written, when ndim is not in 1..8, a shape entry is negative or their product overflows int64, the product times the
 * typesize is not the chunk's nbytes, or start[k] > stop[k] or stop[k] > shape[k] (or start[k] < 0).  The chunk header
 * is checked as blosc_getitem checks it, with its codes.  A touched block that fails to decode returns blosc_d's code
 * and leaves dest untouched. */
long long blosc_b200_getslice(const void* src, int ndim, const int64_t* shape, const int64_t* start,
                              const int64_t* stop, void* dest);

/* blosc_b200_getslice with a positive step per dimension: the items start[k], start[k] + step[k], ... below stop[k] of
 * each dimension k, written to dest as one contiguous C-order array (numpy: a[start[0]:stop[0]:step[0], ...,
 * start[ndim-1]:stop[ndim-1]:step[ndim-1]], made contiguous).  Dimension k selects n_k = ceil((stop[k] - start[k]) /
 * step[k]) items.  step is host memory, ndim entries; step == NULL means all ones, which is blosc_b200_getslice.
 * Returns the bytes written, prod(n_k) * typesize; 0 for an empty box, with nothing launched.  Every check of
 * blosc_b200_getslice applies, and a step[k] < 1 also returns -1 with a message on stderr before anything is launched
 * or written (negative steps are not supported).  Only the blocks that hold a byte of a selected item are decoded, so
 * a step that jumps over whole blocks skips them, and the launches do not grow with the number of selected items. */
long long blosc_b200_getslice_step(const void* src, int ndim, const int64_t* shape, const int64_t* start,
                                   const int64_t* stop, const int64_t* step, void* dest);

/* A batch of equal-sized boxes in one call: nboxes boxes of extents extent[0..ndim) (host memory), box i at the corner
 * starts[i][0..ndim) (starts: nboxes x ndim int64, row-major), covering items [starts[i][k], starts[i][k] + extent[k])
 * of each dimension k of the chunk's C-order array of `shape`.  Box i is written to dest + i * B, B = prod(extent) *
 * typesize, as one contiguous C-order array, so dest is numpy's np.stack of the K slices.  Boxes may overlap, repeat
 * and come in any order.  src / dest are host or device memory as in blosc_b200_getslice.  starts may be host memory
 * (uploaded) or device memory on the call's device, chosen as blosc_b200_getitems chooses it (otherwise -1 with a
 * message before anything is read).  The corners are checked and every box planned on the GPU: each touched block is
 * decoded once, and the launches, read-backs and syncs do not grow with nboxes.  Returns the bytes written, nboxes * B;
 * 0 when nboxes is 0 or an extent is 0, with nothing launched and starts never read.  -1 with a message on stderr,
 * before anything is launched, when ndim is not in 1..8, a shape or extent entry is negative, extent[k] > shape[k],
 * the shape's product overflows int64 or times the typesize is not the chunk's nbytes, nboxes < 0, or nboxes * B
 * overflows int64.  A corner with starts[i][k] < 0 or > shape[k] - extent[k] returns -1 with one message naming the
 * first such box, and nothing is decoded or written.  The chunk header is checked as blosc_getitem checks it, with its
 * codes.  A touched block that fails to decode returns blosc_d's code and leaves dest untouched. */
long long blosc_b200_getslices(const void* src, int ndim, const int64_t* shape, const int64_t* extent,
                               long long nboxes, const int64_t* starts, void* dest);

/* An orthogonal index selection (numpy: a[np.ix_(...)] with slices kept as slices, made contiguous in C order; zarr's
 * oindex): dimension k is a list when index != NULL and index[k] != NULL, selecting the coordinates index[k][0 ..
 * nindex[k]), in any order and with repeats; start[k] / stop[k] / step[k] are then not read.  Every other dimension is
 * a slice, as in blosc_b200_getslice_step (step == NULL: all ones).  Dimension k contributes n_k = nindex[k] entries for
 * a list, ceil((stop[k] - start[k]) / step[k]) for a slice, and the result is written to dest as one contiguous C-order
 * array.  shape, start, stop, step, nindex and the index pointer array are host memory; each list may be host memory
 * (uploaded once) or device memory on the call's device, chosen as blosc_b200_getitems chooses it, and a device list is
 * never copied to the host.  src / dest are host or device memory as in blosc_b200_getslice.  With no list (index ==
 * NULL or all NULL) this is blosc_b200_getslice_step.  Returns the bytes written, prod(n_k) * typesize; 0 when some n_k
 * is 0, with nothing launched and no list read.  -1 with a message on stderr, before anything is launched, on every
 * failing check of blosc_b200_getslice_step on the shape and the slice dimensions, nindex[k] < 0, an output size that
 * overflows int64, or a device list on another device.  The list entries are checked on the GPU by the planning
 * launch: an entry < 0 or >= shape[k] returns -1 with one message naming the first bad entry (lowest k, then lowest
 * position), and nothing is decoded or written (negative indices are not wrapped).  The header codes and decode
 * failures are those of blosc_b200_getslice.  Only the blocks that hold a byte of a selected item are decoded, and the
 * launches, read-backs and syncs do not grow with the list lengths. */
long long blosc_b200_getoindex(const void* src, int ndim, const int64_t* shape, const int64_t* start,
                               const int64_t* stop, const int64_t* step, const int64_t* const* index,
                               const int64_t* nindex, void* dest);

/* Frames: buffers larger than one chunk (a Blosc-1 chunk holds at most BLOSC_MAX_BUFFERSIZE
 * bytes, blosc.h:40).  The buffer is cut into `chunksize`-byte pieces (0 = 256 MiB; rounded down
 * to a multiple of typesize), each compressed exactly as blosc_compress_ctx() would with
 * destsize = piece + 16, several in flight at once so that PCIe transfers overlap the kernels.
 * The result is a 32-byte header + u64 offset table + ordinary Blosc-1 chunks (layout in
 * blosc_b200.c); blosc_b200_frame_chunk() locates chunk i so that any Blosc-1 library can decode
 * it.  src/dest/frame may be host or device memory.  Returns: compress -> frame bytes, 0 if it
 * does not fit in destsize (always fits in blosc_b200_frame_bound()), <0 like blosc_compress_ctx;
 * decompress -> nbytes or -1; getitem -> bytes copied or <0 (items may span chunks). */
size_t    blosc_b200_frame_bound(size_t nbytes, size_t typesize, size_t chunksize);
long long blosc_b200_frame_compress(int clevel, int doshuffle, size_t typesize, size_t nbytes, const void* src,
                                    void* dest, size_t destsize, const char* compressor, size_t blocksize,
                                    size_t chunksize, int numinternalthreads);
long long blosc_b200_frame_decompress(const void* frame, size_t framesize, void* dest, size_t destsize,
                                      int numinternalthreads);
long long blosc_b200_frame_getitem(const void* frame, size_t framesize, size_t start, size_t nitems, void* dest);
/* blosc_b200_getitems over a frame: ranges may cross chunk boundaries, as in blosc_b200_frame_getitem, and are
 * written back to back into dest in request order.  Every range is checked before anything is read.  starts / nitems
 * may be host or device memory.  When either is device memory and every device list is on the call's device (that of
 * frame or dest when either is device memory, else the one chosen with blosc_b200_set_device), the frame is planned on
 * the GPU: the ranges are cut into one piece list per chunk there, and neither list is copied to the host.  Device
 * lists on another device are copied to the host, where the frame is planned. */
long long blosc_b200_frame_getitems(const void* frame, size_t framesize, size_t nranges, const size_t* starts,
                                    const size_t* nitems, void* dest);
/* blosc_b200_getslice over a frame: the whole frame holds the C-order array, in items of chunk 0's typesize (as
 * frame_getitems reads them).  The box may cross chunk boundaries; the chunks it touches are read in ascending order,
 * each as one blosc_b200_getslice part, and the first failure decides the result: its header code, blosc_d's code, or
 * -1 for a touched chunk whose typesize differs from chunk 0's.  On a failure a host dest is untouched; a device dest
 * may hold the parts of earlier chunks.  The geometry is checked as in blosc_b200_getslice, against the frame's
 * nbytes. */
long long blosc_b200_frame_getslice(const void* frame, size_t framesize, int ndim, const int64_t* shape,
                                    const int64_t* start, const int64_t* stop, void* dest);
/* blosc_b200_getslice_step over a frame, with the failures and ordering of blosc_b200_frame_getslice: chunks that
 * hold no selected item are neither read nor decoded. */
long long blosc_b200_frame_getslice_step(const void* frame, size_t framesize, int ndim, const int64_t* shape,
                                         const int64_t* start, const int64_t* stop, const int64_t* step, void* dest);
/* blosc_b200_getslices over a frame: the whole frame holds the C-order array, as in blosc_b200_frame_getslice, and a
 * box may cross chunk boundaries.  The corners are checked once; the chunks that hold an item of some box are then
 * read in ascending order, each decoding its touched blocks once for all boxes.  The first failure decides the result,
 * as in blosc_b200_frame_getslice: on a failure a host dest is untouched; a device dest may hold parts of earlier
 * chunks. */
long long blosc_b200_frame_getslices(const void* frame, size_t framesize, int ndim, const int64_t* shape,
                                     const int64_t* extent, long long nboxes, const int64_t* starts, void* dest);
/* blosc_b200_getoindex over a frame, with the failures and ordering of blosc_b200_frame_getslice_step: the list
 * entries are checked once, by one launch that also flags the chunks holding a selected item; chunks that hold none
 * are neither read nor decoded. */
long long blosc_b200_frame_getoindex(const void* frame, size_t framesize, int ndim, const int64_t* shape,
                                     const int64_t* start, const int64_t* stop, const int64_t* step,
                                     const int64_t* const* index, const int64_t* nindex, void* dest);
int       blosc_b200_frame_info(const void* frame, size_t framesize, size_t* nbytes, size_t* cbytes,
                                size_t* chunksize, size_t* nchunks);
long long blosc_b200_frame_chunk(const void* frame, size_t framesize, size_t i, size_t* chunk_cbytes);

/* blosc_b200_getslice_step over an N-d array stored as a regular grid of chunks (zarr v2, the HDF5 blosc filter,
 * PyTables): the C-order array of `shape`, items of `itemsize` bytes, is cut into grid[k] = ceil(shape[k] /
 * chunkshape[k]) chunks per dimension.  chunks is a host array of prod(grid) pointers in C order of the grid, each a
 * Blosc-1 chunk in host or device memory holding its sub-array of prod(chunkshape) * itemsize bytes in C order (edge
 * chunks at full shape; their padding is never read), or NULL for a missing chunk, whose items are the itemsize bytes
 * at `fill` (host memory; NULL: zero bytes).  The selection is blosc_b200_getslice_step's, written to dest (host or
 * device memory) as one contiguous C-order array.  Only the table entries of touched chunks (those holding a selected
 * item) are read, and in a touched chunk only the blocks holding a byte of a selected item are decoded.  The item size
 * is the caller's: a chunk's header typesize may differ (it is used for unshuffling alone), and chunks may differ in
 * codec, filter and typesize; only the header's nbytes must be prod(chunkshape) * itemsize.  Each touched chunk's part
 * is gathered straight into its place in dest, and touched chunks are read by up to BLOSC_B200_FRAME_WORKERS threads
 * (default 4) at once.  Returns the bytes written, prod(n_k) * itemsize; 0 for an empty selection, with nothing launched
 * or read (chunks may then be NULL).  -1 with a message on stderr, before anything is launched or read, on every
 * failing check of blosc_b200_getslice_step against `shape`, chunkshape[k] < 1, itemsize < 1, a chunk larger than
 * BLOSC_MAX_BUFFERSIZE bytes, an output size that overflows int64, chunks == NULL, or a touched device chunk on another
 * device than the call's: dest's when dest is device memory, else the first touched device chunk's, else the one
 * chosen with blosc_b200_set_device.  A touched chunk's header failure returns blosc_getitem's code, an nbytes other
 * than prod(chunkshape) * itemsize returns -1 with a message naming its grid coordinates, and a touched block that
 * fails to decode returns blosc_d's code; when several touched chunks fail, the lowest in grid C order decides, whatever
 * the number of workers.  On a failure a host dest is untouched; a device dest may hold the parts of other chunks. */
long long blosc_b200_grid_getslice(int ndim, const int64_t* shape, const int64_t* chunkshape, size_t itemsize,
                                   const void* const* chunks, const void* fill, const int64_t* start,
                                   const int64_t* stop, const int64_t* step, void* dest);

/* Select the CUDA device used by the calling thread's subsequent calls with HOST pointers
 * (device pointers carry their device).  Multi-GPU callers run one process (or thread) per GPU. */
int blosc_b200_set_device(int dev);

/* Per-kernel CUDA-event timing of the calls made since the last reset (bench.py's roofline
 * leg).  kind: 0 filter, 1 encode, 2 scan, 3 compact, 4 decode, 5 unfilter, 6 index, 7 parse, 8 zenc, 9 denc,
 * 10 senc, 11 gather, 12 plan (getitems planned on the GPU). */
void blosc_b200_set_profiling(int on);
void blosc_b200_prof_reset(void);
int  blosc_b200_prof_get(int kind, double* ms_total, long long* launches);
long long blosc_b200_launch_count(void);      /* kernels launched by this library so far */

#ifdef __cplusplus
}
#endif
#endif

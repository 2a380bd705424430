/*
 * b2_backend.h -- the thin device layer the host framing code (blosc_b200.c, plain C)
 * talks to.  The product implements it with CUDA (backend_cuda.cu, sm_90a kernels);
 * the CPU test-suite links the same host code against tests/emu/backend_emu.cpp, which
 * runs the very same kernels in a lock-step SIMT emulator.  There is no CPU codec
 * behind this interface: without a CUDA device every call fails.
 */
#ifndef B2_BACKEND_H
#define B2_BACKEND_H
#include <stddef.h>
#include "b2_args.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2_stream_s* b2_stream_t;

int  b2_backend_init(void);                         /* 0 ok; <0 no usable device (message on stderr) */
int  b2_get_device(void);                           /* current CUDA device of the calling thread */
int  b2_set_device(int dev);
int  b2_device_prepare(void);                       /* per-device one-time kernel attribute setup */
int  b2_stream_create(b2_stream_t* s);
void b2_stream_destroy(b2_stream_t s);
int  b2_stream_sync(b2_stream_t s);

int  b2_dev_alloc(void** p, size_t n);
void b2_dev_free(void* p);
int  b2_pinned_alloc(void** p, size_t n);           /* host memory the device can DMA from/to */
void b2_pinned_free(void* p);
int  b2_ptr_is_device(const void* p);               /* 1 device/managed, 0 host */
int  b2_ptr_is_pinned(const void* p);               /* 1 page-locked / registered host memory */
int  b2_ptr_device(const void* p);                  /* the device that holds device memory p; -1 for host memory */

typedef struct b2_event_s* b2_event_t;
int  b2_event_create(b2_event_t* e);
void b2_event_destroy(b2_event_t e);
int  b2_event_record(b2_event_t e, b2_stream_t s);
int  b2_event_sync(b2_event_t e);

int  b2_copy_h2d(void* d, const void* h, size_t n, b2_stream_t s);
int  b2_copy_d2h(void* h, const void* d, size_t n, b2_stream_t s);
int  b2_copy_d2d(void* d, const void* s_, size_t n, b2_stream_t s);
int  b2_memset_dev(void* d, int v, size_t n, b2_stream_t s);

int  b2_launch_filter(const FilterArgs* a, b2_stream_t s);
int  b2_launch_encode(const EncodeArgs* a, b2_stream_t s);
int  b2_launch_scan(const ScanArgs* a, b2_stream_t s);
int  b2_launch_compact(const CompactArgs* a, b2_stream_t s);
int  b2_launch_decode(const DecodeArgs* a, b2_stream_t s);
int  b2_launch_fast(const FastArgs* a, b2_stream_t s);      /* by a->codec, index_kernel and then:
                                                             * B2_CODEC_LZ4: parse_kernel + fscan_kernel (segment-parallel LZ4);
                                                             * B2_CODEC_ZSTD: zparse_kernel + zenc_kernel (zstd);
                                                             * B2_CODEC_ZLIB: dparse_kernel + denc_kernel (zlib);
                                                             * B2_CODEC_SNAPPY: zparse_kernel + senc_kernel */
int  b2_launch_gather(const GatherArgs* a, b2_stream_t s);  /* gather_kernel (getitems) */
int  b2_launch_plan(const PlanArgs* a, b2_stream_t s);      /* plan_check_kernel + plan_scan_kernel x 3 (x 1 in place):
                                                             * getitems planned from device-resident range lists */
int  b2_launch_fplan(const FramePlanArgs* a, b2_stream_t s);           /* fplan_check_kernel + plan_scan_kernel x 2
                                                                        * (x 4 when the frame has chunks) */
int  b2_launch_fplan_scatter(const FramePlanArgs* a, b2_stream_t s);   /* fplan_scatter_kernel: the piece lists */
int  b2_launch_box_plan(const BoxPlanArgs* a, b2_stream_t s);          /* box_touch_kernel + plan_scan_kernel<PLAN_SLOT>:
                                                                        * the blocks a chunk's part of a box touches */
int  b2_launch_box_gather(const BoxGatherArgs* a, b2_stream_t s);      /* box_gather_kernel (getslice) */
int  b2_launch_box_check(const BoxCheckArgs* a, b2_stream_t s);        /* box_check_kernel: getslices' corners */
int  b2_launch_boxes_plan(const BoxesPlanArgs* a, b2_stream_t s);      /* boxes_touch_kernel + plan_scan_kernel<PLAN_SLOT>:
                                                                        * the blocks a chunk's part of a batch touches */
int  b2_launch_boxes_gather(const BoxesGatherArgs* a, b2_stream_t s);  /* boxes_gather_kernel (getslices) */
int  b2_launch_oindex_plan(const OIndexPlanArgs* a, b2_stream_t s);    /* oindex_touch_kernel (+ plan_scan_kernel<PLAN_SLOT>
                                                                        * when it marks blocks): getoindex's list check and
                                                                        * touched blocks, or a frame's touched chunks */
int  b2_launch_oindex_gather(const OIndexGatherArgs* a, b2_stream_t s);   /* oindex_gather_kernel (getoindex) */
int  b2_launch_placed_gather(const PlacedGatherArgs* a, b2_stream_t s);   /* placed_gather_kernel (grid_getslice) */
int  b2_launch_placed_fill(const PlacedGatherArgs* a, b2_stream_t s);     /* placed_fill_kernel (grid_getslice) */

/* profiling: per-kernel-kind CUDA-event timing (off by default) */
enum { B2_K_FILTER = 0, B2_K_ENCODE, B2_K_SCAN, B2_K_COMPACT, B2_K_DECODE, B2_K_UNFILTER, B2_K_INDEX, B2_K_PARSE, B2_K_ZENC, B2_K_DENC, B2_K_SENC, B2_K_GATHER, B2_K_PLAN, B2_K_COUNT };
void b2_prof_enable(int on);
void b2_prof_reset(void);
int  b2_prof_get(int kind, double* ms_total, long long* launches);
long long b2_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif

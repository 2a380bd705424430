/*
 * blosc_b200.c -- host side of libblosc_b200: the c-blosc 1.x C API and the chunk
 * framing / planning, in plain C, over the device layer of b2_backend.h.
 *
 * What stays on the host (it is the format contract, a few dozen integer operations per
 * call): argument validation and return codes (reference blosc/blosc.c:1062-1145,
 * 1435-1518), compute_blocksize (:962-1060), split_block (:929-959), the 16-byte header
 * (:1148-1247) and the MEMCPYED decisions (:1219-1229, :1264-1272).  Everything that
 * touches the payload -- filters, codecs, the block scheduler and the compaction of
 * variable-size blocks -- runs as CUDA kernels (dev_*.cuh); there is no CPU codec here.
 */
#include "../../include/blosc_b200.h"

#include <errno.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "b2_backend.h"

#define MIN_BUFFERSIZE 128        /* blosc.c:73 */
#define MAX_SPLITS 16             /* blosc.c:76 */
#define L1_SIZE (32 * 1024)       /* blosc.c:79 */

/* ---- process-global state of the non-ctx API (blosc.c:143-150) ---- */
static int g_compressor = BLOSC_BLOSCLZ;
static int g_threads = 1;
static int g_force_blocksize = 0;
static int g_initlib = 0;
static int g_splitmode = BLOSC_FORWARD_COMPAT_SPLIT;
static pthread_mutex_t g_global_mutex = PTHREAD_MUTEX_INITIALIZER;

/* ---- little-endian header accessors (blosc.c:243-289) ---- */
static int32_t rd_i32(const uint8_t* p) {
  return (int32_t)((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24));
}
static void wr_i32(uint8_t* p, int32_t v) {
  uint32_t u = (uint32_t)v;
  p[0] = (uint8_t)u; p[1] = (uint8_t)(u >> 8); p[2] = (uint8_t)(u >> 16); p[3] = (uint8_t)(u >> 24);
}

/* ------------------------------------------------------------------------- */
/* pageable-host staging: a small pool of copy threads + pinned bounce slices */
/* ------------------------------------------------------------------------- */
/* Callers of the C API usually hand in malloc'ed (pageable) buffers.  cudaMemcpy from pageable
 * memory runs at a fraction of the PCIe rate, so such buffers go through page-locked bounce
 * slices instead: a few host threads copy slice i+1 while the DMA engine moves slice i. */
#define B2_STAGE_SLICE ((size_t)8 << 20)
#define B2_STAGE_DEPTH 4
#define B2_COPY_THREADS_MAX 16

typedef struct {
  pthread_mutex_t mu;
  pthread_cond_t cv_work, cv_done;
  int nthreads, started, generation, pending, stop;
  uint8_t* dst;
  const uint8_t* src;
  size_t len;
  pthread_t th[B2_COPY_THREADS_MAX];
  int ids[B2_COPY_THREADS_MAX];
} b2_copy_pool;

static b2_copy_pool g_cp = {PTHREAD_MUTEX_INITIALIZER, PTHREAD_COND_INITIALIZER, PTHREAD_COND_INITIALIZER, 0, 0, 0, 0, 0, NULL, NULL, 0, {0}, {0}};
static pthread_mutex_t g_cp_user = PTHREAD_MUTEX_INITIALIZER;      /* one parallel copy at a time */

static void* copy_worker(void* arg) {
  const int id = *(int*)arg;
  int seen = 0;
  pthread_mutex_lock(&g_cp.mu);
  for (;;) {
    while (!g_cp.stop && g_cp.generation == seen) pthread_cond_wait(&g_cp.cv_work, &g_cp.mu);
    if (g_cp.stop) break;
    seen = g_cp.generation;
    {
      const size_t per = ((g_cp.len + g_cp.nthreads - 1) / g_cp.nthreads + 63) & ~(size_t)63;
      const size_t lo = per * (size_t)id, hi = lo + per < g_cp.len ? lo + per : g_cp.len;
      uint8_t* d = g_cp.dst;
      const uint8_t* s = g_cp.src;
      pthread_mutex_unlock(&g_cp.mu);
      if (lo < hi) memcpy(d + lo, s + lo, hi - lo);
      pthread_mutex_lock(&g_cp.mu);
    }
    if (--g_cp.pending == 0) pthread_cond_signal(&g_cp.cv_done);
  }
  pthread_mutex_unlock(&g_cp.mu);
  return NULL;
}

static void parallel_memcpy(void* dst, const void* src, size_t len) {
  int i;
  if (len < ((size_t)1 << 20)) { memcpy(dst, src, len); return; }
  pthread_mutex_lock(&g_cp_user);
  pthread_mutex_lock(&g_cp.mu);
  if (!g_cp.started) {
    const char* e = getenv("BLOSC_B200_COPY_THREADS");
    int n = e ? atoi(e) : 8;
    if (n < 1) n = 1;
    if (n > B2_COPY_THREADS_MAX) n = B2_COPY_THREADS_MAX;
    g_cp.nthreads = 0;
    for (i = 0; i < n; i++) {
      g_cp.ids[i] = i;
      if (pthread_create(&g_cp.th[i], NULL, copy_worker, &g_cp.ids[i]) != 0) break;
      g_cp.nthreads++;
    }
    g_cp.started = 1;
  }
  if (g_cp.nthreads == 0) {
    pthread_mutex_unlock(&g_cp.mu);
    memcpy(dst, src, len);
  } else {
    g_cp.dst = (uint8_t*)dst; g_cp.src = (const uint8_t*)src; g_cp.len = len;
    g_cp.pending = g_cp.nthreads;
    g_cp.generation++;
    pthread_cond_broadcast(&g_cp.cv_work);
    while (g_cp.pending) pthread_cond_wait(&g_cp.cv_done, &g_cp.mu);
    pthread_mutex_unlock(&g_cp.mu);
  }
  pthread_mutex_unlock(&g_cp_user);
}

/* ------------------------------------------------------------------------- */
/* workspace pool: device scratch + one stream per concurrent call            */
/* ------------------------------------------------------------------------- */
typedef struct {
  void* p;
  size_t cap;
} b2_buf;

typedef struct {
  int in_use, ready, dev;
  b2_stream_t stream;
  b2_buf in, filt, slots, out, csizes, needs, bstarts;
  b2_buf prev, segs, ptail;   /* segment-parallel LZ4 parse (dev_lz4fast.cuh) */
  b2_buf plan;          /* getitems planned on the GPU: its scratch */
  int* d_result;        /* B2_R_* words (b2_args.h): cbytes, fits, status, work-queue and done counters */
  int* h_result;        /* pinned mirror */
  unsigned queue_base;  /* tickets drawn from the B2_R_QUEUE counter so far (dev_chunk.cuh next_stream) */
  uint8_t* stage[B2_STAGE_DEPTH];   /* pinned bounce slices for pageable host buffers (lazy) */
  b2_event_t stage_ev[B2_STAGE_DEPTH];
  int stage_ok;         /* all DEPTH slices and events exist */
} b2_ws;

#define B2_MAX_WS 16
static b2_ws g_ws[B2_MAX_WS];
static pthread_mutex_t g_ws_mutex = PTHREAD_MUTEX_INITIALIZER;
static pthread_cond_t g_ws_cv = PTHREAD_COND_INITIALIZER;
static int g_backend_state = 0;   /* 0 untried, 1 ok, -1 failed */

static int backend_ready(void) {
  int st;
  pthread_mutex_lock(&g_ws_mutex);
  if (g_backend_state == 0) g_backend_state = b2_backend_init() == 0 ? 1 : -1;
  st = g_backend_state;
  pthread_mutex_unlock(&g_ws_mutex);
  if (st < 0) fprintf(stderr, "blosc_b200: no usable CUDA device -- this library has no CPU codec\n");
  return st > 0;
}

static void buf_free(b2_buf* b) { if (b->p) b2_dev_free(b->p); b->p = NULL; b->cap = 0; }

/* Everything a slot owns; the caller holds the slot (in_use) and the slot's device need not be current
 * (device and page-locked allocations are freed by address) */
static void ws_teardown(b2_ws* w) {
  int k;
  buf_free(&w->in); buf_free(&w->filt); buf_free(&w->slots); buf_free(&w->out);
  buf_free(&w->csizes); buf_free(&w->needs); buf_free(&w->bstarts);
  buf_free(&w->prev); buf_free(&w->segs); buf_free(&w->ptail); buf_free(&w->plan);
  for (k = 0; k < B2_STAGE_DEPTH; k++) {
    if (w->stage[k]) b2_pinned_free(w->stage[k]);
    if (w->stage_ev[k]) b2_event_destroy(w->stage_ev[k]);
    w->stage[k] = NULL; w->stage_ev[k] = NULL;
  }
  w->stage_ok = 0;
  if (w->d_result) b2_dev_free(w->d_result);
  if (w->h_result) b2_pinned_free(w->h_result);
  if (w->stream) b2_stream_destroy(w->stream);
  w->d_result = NULL; w->h_result = NULL; w->stream = NULL;
  w->ready = 0;
}

/* error paths only: wait for whatever was launched and zero the counter words */
static void ws_reset_counters(b2_ws* w) {
  b2_stream_sync(w->stream);
  b2_memset_dev(w->d_result, 0, 4 * B2_R_WORDS, w->stream);
  b2_stream_sync(w->stream);
  w->queue_base = 0;
}

/* calls in flight on `dev` right now (the caller's own included) */
static int ws_busy(int dev) {
  int i, n = 0;
  pthread_mutex_lock(&g_ws_mutex);
  for (i = 0; i < B2_MAX_WS; i++) if (g_ws[i].in_use && g_ws[i].ready && g_ws[i].dev == dev) n++;
  pthread_mutex_unlock(&g_ws_mutex);
  return n;
}

static void ws_release(b2_ws* w) {
  pthread_mutex_lock(&g_ws_mutex);
  w->in_use = 0;
  pthread_cond_signal(&g_ws_cv);
  pthread_mutex_unlock(&g_ws_mutex);
}

/* A workspace = one stream + scratch on one device.  The reference's _ctx calls have no limit on the
 * number of concurrent callers (each allocates its own context, blosc.c:1287-1309); here the 17th
 * concurrent call WAITS for a slot instead of failing, and an idle slot that was made on another
 * device is rebuilt for the caller's device when no matching or unused slot is left. */
static b2_ws* ws_acquire(void) {
  b2_ws* w = NULL;
  int i, dev, rebuild = 0;
  if (!backend_ready()) return NULL;
  dev = b2_get_device();
  pthread_mutex_lock(&g_ws_mutex);
  for (;;) {
    for (i = 0; i < B2_MAX_WS && !w; i++)
      if (!g_ws[i].in_use && g_ws[i].ready && g_ws[i].dev == dev) w = &g_ws[i];
    for (i = 0; i < B2_MAX_WS && !w; i++)
      if (!g_ws[i].in_use && !g_ws[i].ready) w = &g_ws[i];
    for (i = 0; i < B2_MAX_WS && !w; i++)
      if (!g_ws[i].in_use) { w = &g_ws[i]; rebuild = 1; }
    if (w) { w->in_use = 1; break; }
    pthread_cond_wait(&g_ws_cv, &g_ws_mutex);
  }
  pthread_mutex_unlock(&g_ws_mutex);
  if (rebuild) ws_teardown(w);
  if (!w->ready) {
    void* p = NULL;
    int ok = 0;
    do {
      if (b2_device_prepare() || b2_stream_create(&w->stream)) break;
      if (b2_dev_alloc(&p, 4 * B2_R_WORDS)) break;
      w->d_result = (int*)p;
      if (b2_pinned_alloc(&p, 4 * B2_R_WORDS)) break;
      w->h_result = (int*)p;
      /* the work counters start at zero and every launch leaves them at zero again (dev_chunk.cuh) */
      if (b2_memset_dev(w->d_result, 0, 4 * B2_R_WORDS, w->stream) || b2_stream_sync(w->stream)) break;
      w->queue_base = 0;
      ok = 1;
    } while (0);
    if (!ok) { ws_teardown(w); ws_release(w); return NULL; }
    w->dev = dev;
    w->ready = 1;
  }
  return w;
}

static int buf_ensure(b2_buf* b, size_t need) {
  if (need <= b->cap) return 0;
  if (b->p) b2_dev_free(b->p);
  b->p = NULL; b->cap = 0;
  need = (need + (need >> 3) + 4095) & ~(size_t)4095;    /* slack so slowly growing sizes do not thrash */
  if (b2_dev_alloc(&b->p, need)) { fprintf(stderr, "blosc_b200: device allocation of %zu bytes failed\n", need); return -1; }
  b->cap = need;
  return 0;
}

int blosc_free_resources(void) {                              /* blosc.h:411 */
  int i;
  pthread_mutex_lock(&g_ws_mutex);
  for (i = 0; i < B2_MAX_WS; i++) {
    b2_ws* w = &g_ws[i];
    if (w->in_use || !w->ready) continue;
    buf_free(&w->in); buf_free(&w->filt); buf_free(&w->slots); buf_free(&w->out);
    buf_free(&w->csizes); buf_free(&w->needs); buf_free(&w->bstarts);
    buf_free(&w->prev); buf_free(&w->segs); buf_free(&w->ptail); buf_free(&w->plan);
  }
  pthread_mutex_unlock(&g_ws_mutex);
  return 0;
}

/* ------------------------------------------------------------------------- */
/* names                                                                      */
/* ------------------------------------------------------------------------- */
/* BLOSC_B200_ZSTD=1 (read on every call) makes the library behave like a reference built with zstd: "zstd" chunks
 * are then written (dev_zstdenc.cuh).  Unset, it is a reference built without zstd, which still reads them. */
static int zstd_enabled(void) {
  const char* e = getenv("BLOSC_B200_ZSTD");
  return e && *e && atoi(e) != 0;
}

/* BLOSC_B200_ZLIB=1 (read on every call, independent of the zstd switch) does the same for zlib: "zlib" chunks are
 * then written (dev_deflate.cuh).  Unset, it is a reference built with -DDEACTIVATE_ZLIB, which still reads them. */
static int zlib_enabled(void) {
  const char* e = getenv("BLOSC_B200_ZLIB");
  return e && *e && atoi(e) != 0;
}

/* BLOSC_B200_SNAPPY=1 (read on every call, independent of the other two) does the same for snappy: "snappy" chunks are
 * written (dev_snappy.cuh) and read.  Unset, it is a reference built without snappy, which neither writes nor reads
 * them (blosc.c:547-553). */
static int snappy_enabled(void) {
  const char* e = getenv("BLOSC_B200_SNAPPY");
  return e && *e && atoi(e) != 0;
}

int blosc_compcode_to_compname(int compcode, const char** compname) {    /* blosc.c:329-374 */
  static const char* names[6] = {BLOSC_BLOSCLZ_COMPNAME, BLOSC_LZ4_COMPNAME, BLOSC_LZ4HC_COMPNAME,
                                 BLOSC_SNAPPY_COMPNAME, BLOSC_ZLIB_COMPNAME, BLOSC_ZSTD_COMPNAME};
  *compname = (compcode >= 0 && compcode < 6) ? names[compcode] : NULL;
  /* codecs this build can ENCODE; like a reference built without the others */
  if (compcode == BLOSC_BLOSCLZ || compcode == BLOSC_LZ4 || compcode == BLOSC_LZ4HC) return compcode;
  if (compcode == BLOSC_SNAPPY && snappy_enabled()) return compcode;
  if (compcode == BLOSC_ZLIB && zlib_enabled()) return compcode;
  if (compcode == BLOSC_ZSTD && zstd_enabled()) return compcode;
  return -1;
}

int blosc_compname_to_compcode(const char* compname) {                    /* blosc.c:377-409 */
  if (strcmp(compname, BLOSC_BLOSCLZ_COMPNAME) == 0) return BLOSC_BLOSCLZ;
  if (strcmp(compname, BLOSC_LZ4_COMPNAME) == 0) return BLOSC_LZ4;
  if (strcmp(compname, BLOSC_LZ4HC_COMPNAME) == 0) return BLOSC_LZ4HC;
  if (strcmp(compname, BLOSC_SNAPPY_COMPNAME) == 0 && snappy_enabled()) return BLOSC_SNAPPY;
  if (strcmp(compname, BLOSC_ZLIB_COMPNAME) == 0 && zlib_enabled()) return BLOSC_ZLIB;
  if (strcmp(compname, BLOSC_ZSTD_COMPNAME) == 0 && zstd_enabled()) return BLOSC_ZSTD;
  return -1;
}

/* the reference's order, minus the codecs that are switched off: one string per combination of the three switches
 * (snappy | zlib << 1 | zstd << 2), built once, so that a returned pointer stays valid whatever the switches do later */
static char g_complists[8][64];
static pthread_once_t g_complists_once = PTHREAD_ONCE_INIT;
static void build_complists(void) {
  for (int m = 0; m < 8; m++)
    snprintf(g_complists[m], sizeof g_complists[m], "%s,%s,%s%s%s%s", BLOSC_BLOSCLZ_COMPNAME, BLOSC_LZ4_COMPNAME,
             BLOSC_LZ4HC_COMPNAME, (m & 1) ? "," BLOSC_SNAPPY_COMPNAME : "", (m & 2) ? "," BLOSC_ZLIB_COMPNAME : "",
             (m & 4) ? "," BLOSC_ZSTD_COMPNAME : "");
}
const char* blosc_list_compressors(void) {                                  /* blosc.c:2029-2042 */
  pthread_once(&g_complists_once, build_complists);
  return g_complists[snappy_enabled() | zlib_enabled() << 1 | zstd_enabled() << 2];
}
const char* blosc_get_version_string(void) { return BLOSC_VERSION_STRING; }

int blosc_get_complib_info(const char* compname, char** complib, char** version) {   /* blosc.c:2063-2124 */
  int code = -1;
  const char *lib = NULL, *ver = NULL;
  if (strcmp(compname, BLOSC_BLOSCLZ_COMPNAME) == 0) { code = BLOSC_BLOSCLZ_LIB; lib = "BloscLZ"; ver = "2.5.1"; }
  else if (strcmp(compname, BLOSC_LZ4_COMPNAME) == 0 || strcmp(compname, BLOSC_LZ4HC_COMPNAME) == 0) {
    code = BLOSC_LZ4_LIB; lib = "LZ4"; ver = "1.10.0";
  } else if (strcmp(compname, BLOSC_SNAPPY_COMPNAME) == 0 && snappy_enabled()) {
    /* what the reference reports when its snappy does not define SNAPPY_VERSION (blosc.c:2056,2078-2084): these
     * streams are no snappy release's */
    code = BLOSC_SNAPPY_LIB; lib = "Snappy"; ver = "unknown";
  } else if (strcmp(compname, BLOSC_ZLIB_COMPNAME) == 0 && zlib_enabled()) {
    code = BLOSC_ZLIB_LIB; lib = "Zlib"; ver = "1.3.1";          /* the zlib release the streams are checked against */
  } else if (strcmp(compname, BLOSC_ZSTD_COMPNAME) == 0 && zstd_enabled()) {
    code = BLOSC_ZSTD_LIB; lib = "Zstd"; ver = "1.5.6";         /* the zstd release the frames are checked against */
  }
  if (code < 0) {
    if (complib) *complib = NULL;
    if (version) *version = NULL;
    return -1;
  }
  if (complib) *complib = strdup(lib);
  if (version) *version = strdup(ver);
  return code;
}

static const char* clib_name(int clibcode) {                               /* blosc.c:315-322 */
  static const char* n[5] = {"BloscLZ", "LZ4", "Snappy", "Zlib", "Zstd"};
  return (clibcode >= 0 && clibcode < 5) ? n[clibcode] : NULL;
}

/* ------------------------------------------------------------------------- */
/* header introspection (host pointers, as in the reference)                   */
/* ------------------------------------------------------------------------- */
void blosc_cbuffer_sizes(const void* cbuffer, size_t* nbytes, size_t* cbytes, size_t* blocksize) {   /* blosc.c:2127-2141 */
  const uint8_t* s = (const uint8_t*)cbuffer;
  if (s[0] != BLOSC_VERSION_FORMAT) { *nbytes = *blocksize = *cbytes = 0; return; }
  *nbytes = (size_t)rd_i32(s + 4);
  *blocksize = (size_t)rd_i32(s + 8);
  *cbytes = (size_t)rd_i32(s + 12);
}

int blosc_cbuffer_validate(const void* cbuffer, size_t cbytes, size_t* nbytes) {   /* blosc.c:2143-2150 */
  size_t hc, hb;
  if (cbytes < BLOSC_MIN_HEADER_LENGTH) return -1;
  blosc_cbuffer_sizes(cbuffer, nbytes, &hc, &hb);
  if (hc != cbytes) return -1;
  if (*nbytes > BLOSC_MAX_BUFFERSIZE) return -1;
  return 0;
}

void blosc_cbuffer_metainfo(const void* cbuffer, size_t* typesize, int* flags) {   /* blosc.c:2153-2168 */
  const uint8_t* s = (const uint8_t*)cbuffer;
  if (s[0] != BLOSC_VERSION_FORMAT) { *flags = 0; *typesize = 0; return; }
  *flags = (int)s[2] & 7;
  *typesize = (size_t)s[3];
}

void blosc_cbuffer_versions(const void* cbuffer, int* version, int* versionlz) {   /* blosc.c:2172-2180 */
  const uint8_t* s = (const uint8_t*)cbuffer;
  *version = (int)s[0];
  *versionlz = (int)s[1];
}

const char* blosc_cbuffer_complib(const void* cbuffer) {                            /* blosc.c:2184-2195 */
  const uint8_t* s = (const uint8_t*)cbuffer;
  return clib_name((s[2] & 0xe0) >> 5);
}

/* ------------------------------------------------------------------------- */
/* planning                                                                   */
/* ------------------------------------------------------------------------- */
static int is_hcr(int compcode) { return compcode == BLOSC_LZ4HC || compcode == BLOSC_ZLIB || compcode == BLOSC_ZSTD; }

static int split_block(int compcode, int typesize, int blocksize) {       /* blosc.c:929-959 */
  switch (g_splitmode) {
    case BLOSC_ALWAYS_SPLIT: return 1;
    case BLOSC_NEVER_SPLIT: return 0;
    case BLOSC_AUTO_SPLIT:
      return (compcode == BLOSC_BLOSCLZ || compcode == BLOSC_SNAPPY) && typesize <= MAX_SPLITS &&
             blocksize / typesize >= MIN_BUFFERSIZE;
    case BLOSC_FORWARD_COMPAT_SPLIT:
      return compcode != BLOSC_ZSTD && typesize <= MAX_SPLITS && blocksize / typesize >= MIN_BUFFERSIZE;
    default:
      fprintf(stderr, "Split mode %d not supported", g_splitmode);
      return -1;
  }
}

static int32_t compute_blocksize(int compcode, int clevel, int32_t typesize, int32_t nbytes, int32_t forced) {   /* blosc.c:962-1060 */
  int32_t bs = nbytes;
  if (nbytes < typesize) return 1;
  if (forced) {
    bs = forced;
    if (bs < MIN_BUFFERSIZE) bs = MIN_BUFFERSIZE;
    if (bs > (int32_t)BLOSC_MAX_BLOCKSIZE) bs = (int32_t)BLOSC_MAX_BLOCKSIZE;
  } else if (nbytes >= L1_SIZE) {
    bs = L1_SIZE;
    if (is_hcr(compcode)) bs *= 2;
    switch (clevel) {
      case 0: bs /= 4; break;
      case 1: bs /= 2; break;
      case 2: break;
      case 3: bs *= 2; break;
      case 4: case 5: bs *= 4; break;
      case 6: case 7: case 8: bs *= 8; break;
      default: bs *= 8; if (is_hcr(compcode)) bs *= 2; break;
    }
  }
  if (clevel > 0 && split_block(compcode, typesize, bs)) {
    if (bs > (1 << 18)) bs = 1 << 18;
    bs *= typesize;
    if (bs < (1 << 16)) bs = 1 << 16;
    if (bs > 1024 * 1024) bs = 1024 * 1024;
  }
  if (bs > nbytes) bs = nbytes;
  if (bs > typesize) bs = bs / typesize * typesize;
  return bs;
}

static int check_threads(int nthreads, int32_t nbytes, int32_t blocksize) {
  /* do_job takes the pool path (and so validates nthreads, blosc.c:1977-1986) only when
   * nthreads != 1 and the buffer has more than one block (blosc.c:910) */
  if (nthreads == 1 || nbytes / blocksize <= 1) return 0;
  if (nthreads > BLOSC_MAX_THREADS) {
    fprintf(stderr, "Error.  nthreads cannot be larger than BLOSC_MAX_THREADS (%d)", BLOSC_MAX_THREADS);
    return -1;
  }
  if (nthreads <= 0) { fprintf(stderr, "Error.  nthreads must be a positive integer"); return -1; }
  return 0;
}

/* copy between any combination of host / device memory */
static int copy_any(void* dst, int dst_dev, const void* src, int src_dev, size_t n, b2_stream_t s) {
  int rc = 0;
  if (n == 0) return 0;
  if (!dst_dev && !src_dev) { memcpy(dst, src, n); return 0; }
  if (dst_dev && src_dev) rc = b2_copy_d2d(dst, src, n, s);
  else if (dst_dev) rc = b2_copy_h2d(dst, src, n, s);
  else rc = b2_copy_d2h(dst, src, n, s);
  if (rc == 0) rc = b2_stream_sync(s);
  return rc;
}

/* copy_any outside a call's workspace: one is taken for the copy only when either side is device memory */
static int copy_some(void* dst, int dst_dev, const void* src, int src_dev, size_t n) {
  b2_ws* w = NULL;
  int rc;
  if ((dst_dev || src_dev) && !(w = ws_acquire())) return -1;
  rc = copy_any(dst, dst_dev, src, src_dev, n, w ? w->stream : NULL);
  if (w) ws_release(w);
  return rc;
}

static int stage_ready(b2_ws* w) {
  int k;
  if (w->stage_ok) return 0;
  for (k = 0; k < B2_STAGE_DEPTH; k++) {
    void* p = NULL;
    if (!w->stage[k]) { if (b2_pinned_alloc(&p, B2_STAGE_SLICE)) break; w->stage[k] = (uint8_t*)p; }
    if (!w->stage_ev[k] && b2_event_create(&w->stage_ev[k])) { w->stage_ev[k] = NULL; break; }
  }
  if (k < B2_STAGE_DEPTH) {                 /* partial: give everything back, callers fall back to a direct copy */
    for (k = 0; k < B2_STAGE_DEPTH; k++) {
      if (w->stage[k]) b2_pinned_free(w->stage[k]);
      if (w->stage_ev[k]) b2_event_destroy(w->stage_ev[k]);
      w->stage[k] = NULL; w->stage_ev[k] = NULL;
    }
    return -1;
  }
  w->stage_ok = 1;
  return 0;
}

/* host -> device; pageable sources go through the bounce slices */
static int h2d_any(b2_ws* w, void* dst, const void* src, size_t n) {
  size_t off;
  int i = 0;
  if (n == 0) return 0;
  if (n < B2_STAGE_SLICE / 4 || b2_ptr_is_pinned(src) || stage_ready(w)) return b2_copy_h2d(dst, src, n, w->stream);
  for (off = 0; off < n; off += B2_STAGE_SLICE, i++) {
    const int k = i % B2_STAGE_DEPTH;
    const size_t len = n - off < B2_STAGE_SLICE ? n - off : B2_STAGE_SLICE;
    if (i >= B2_STAGE_DEPTH && b2_event_sync(w->stage_ev[k])) return -1;     /* slice k's previous DMA has drained */
    parallel_memcpy(w->stage[k], (const uint8_t*)src + off, len);
    if (b2_copy_h2d((uint8_t*)dst + off, w->stage[k], len, w->stream)) return -1;
    if (b2_event_record(w->stage_ev[k], w->stream)) return -1;
  }
  return 0;
}

/* device -> host, completes before returning; pageable destinations go through the bounce slices */
static int d2h_any(b2_ws* w, void* dst, const void* src, size_t n) {
  size_t off;
  int i = 0, nsl;
  if (n == 0) return 0;
  if (n < B2_STAGE_SLICE / 4 || b2_ptr_is_pinned(dst) || stage_ready(w)) {
    if (b2_copy_d2h(dst, src, n, w->stream)) return -1;
    return b2_stream_sync(w->stream);
  }
  nsl = (int)((n + B2_STAGE_SLICE - 1) / B2_STAGE_SLICE);
  for (i = 0; i < nsl + B2_STAGE_DEPTH - 1; i++) {
    if (i < nsl) {                                   /* issue the DMA of slice i */
      const int k = i % B2_STAGE_DEPTH;
      off = (size_t)i * B2_STAGE_SLICE;
      if (b2_copy_d2h(w->stage[k], (const uint8_t*)src + off, n - off < B2_STAGE_SLICE ? n - off : B2_STAGE_SLICE, w->stream)) return -1;
      if (b2_event_record(w->stage_ev[k], w->stream)) return -1;
    }
    if (i >= B2_STAGE_DEPTH - 1) {                   /* drain slice j = i - (DEPTH-1) to the caller's buffer */
      const int j = i - (B2_STAGE_DEPTH - 1), k = j % B2_STAGE_DEPTH;
      off = (size_t)j * B2_STAGE_SLICE;
      if (b2_event_sync(w->stage_ev[k])) return -1;
      parallel_memcpy((uint8_t*)dst + off, w->stage[k], n - off < B2_STAGE_SLICE ? n - off : B2_STAGE_SLICE);
    }
  }
  return 0;
}

static void make_header(uint8_t* h, int versionlz, int flags, int typesize, int32_t nbytes, int32_t blocksize,
                        int32_t cbytes) {                                  /* blosc.c:1154-1215,1275 */
  h[0] = BLOSC_VERSION_FORMAT; h[1] = (uint8_t)versionlz; h[2] = (uint8_t)flags; h[3] = (uint8_t)typesize;
  wr_i32(h + 4, nbytes); wr_i32(h + 8, blocksize); wr_i32(h + 12, cbytes);
}

/* Where a finished chunk goes.  The plain API writes at `dest`; a frame (below) learns the
 * chunk's offset only once every earlier chunk has announced its size, so the compressor asks
 * for the final location at the moment `cbytes` is known. */
typedef struct b2_frame_job b2_frame_job;
typedef struct {
  b2_frame_job* job;
  int index, placed;
  int many;             /* other chunks are in flight with this one: favour streams per SM over latency */
} b2_place;
static void* frame_place(b2_place* pl, int32_t cbytes);

/* Opt-in (BLOSC_B200_LZ4_PACK=1): on the 8 GiB frames workload it can help typesize 2 and 8, but at
 * typesize 4 the extra instructions per probe outweigh the doubled number of streams per SM -- so it
 * is not the default. */
static int lz4_pack_wanted(const b2_place* pl) {
  const char* e = getenv("BLOSC_B200_LZ4_PACK");
  (void)pl;
  return e && *e && atoi(e) != 0;
}

/* BLOSC_B200_PARSE selects the LZ4 encoder: "exact" (default) replays LZ4_compress_fast bit for bit, chunks are
 * byte-identical to the reference's; "fast" (alias "segmented") is the segment-parallel parser of dev_lz4fast.cuh:
 * chunks are valid Blosc-1 / LZ4 that any reference build decodes, but not the reference's bytes. */
static int lz4_fast_wanted(void) {
  const char* e = getenv("BLOSC_B200_PARSE");
  return e && (strcmp(e, "fast") == 0 || strcmp(e, "segmented") == 0);
}

/* header + raw payload (blosc.c:825-830) */
static int emit_memcpyed(const uint8_t* hdr, const void* src, int src_dev, void* dest, int dest_dev, int32_t nbytes) {
  if (copy_some(dest, dest_dev, hdr, 0, 16) || copy_some((uint8_t*)dest + 16, dest_dev, src, src_dev, (size_t)nbytes))
    return -1;
  return nbytes + 16;
}

/* ------------------------------------------------------------------------- */
/* compression                                                                */
/* ------------------------------------------------------------------------- */
static int compress_impl(int clevel, int doshuffle, size_t typesize, size_t nbytes, const void* src, void* dest,
                         size_t destsize, const char* compressor, size_t blocksize, int numinternalthreads,
                         b2_place* pl, int pl_dest_dev) {
  const int compcode = blosc_compname_to_compcode(compressor);
  int32_t ts, nb, bs, nblocks, leftover, dsz;
  int flags = 0, compformat, dont_split, src_dev, dest_dev, dofilter, fmode = 0, nsplits, result = -1, launched = 0;
  uint8_t hdr[16];
  b2_ws* w;
  const uint8_t* d_src;
  const uint8_t* d_codec_in;
  uint8_t* d_dest;

  /* initialize_context_compression, blosc.c:1062-1145 */
  if (nbytes > BLOSC_MAX_BUFFERSIZE) return 0;
  if (destsize < BLOSC_MAX_OVERHEAD) return 0;
  if (destsize - BLOSC_MAX_OVERHEAD > nbytes) destsize = nbytes + BLOSC_MAX_OVERHEAD;
  if (clevel < 0 || clevel > 9) return -10;
  if (doshuffle != 0 && doshuffle != 1 && doshuffle != 2) return -10;
  if (typesize == 0) return -10;
  if (typesize > BLOSC_MAX_TYPESIZE) typesize = 1;
  ts = (int32_t)typesize; nb = (int32_t)nbytes; dsz = (int32_t)destsize;
  bs = compute_blocksize(compcode, clevel, ts, nb, (int32_t)blocksize);
  nblocks = nb / bs; leftover = nb % bs;
  if (leftover > 0) nblocks++;

  /* write_compression_header, blosc.c:1148-1247 */
  if (compcode == BLOSC_BLOSCLZ) compformat = BLOSC_BLOSCLZ_FORMAT;
  else if (compcode == BLOSC_LZ4) compformat = BLOSC_LZ4_FORMAT;
  else if (compcode == BLOSC_LZ4HC) compformat = BLOSC_LZ4HC_FORMAT;     /* blosc.c:1170-1172: the LZ4 format */
  else if (compcode == BLOSC_SNAPPY) compformat = BLOSC_SNAPPY_FORMAT;   /* blosc.c:1176-1181 */
  else if (compcode == BLOSC_ZLIB) compformat = BLOSC_ZLIB_FORMAT;       /* blosc.c:1183-1188 */
  else if (compcode == BLOSC_ZSTD) compformat = BLOSC_ZSTD_FORMAT;       /* blosc.c:1190-1196 */
  else {
    fprintf(stderr, "Blosc has not been compiled with '%s' ", compressor ? compressor : "(null)");
    fprintf(stderr, "compression support.  Please use one having it.");
    return -5;
  }
  if (clevel == 0) flags |= BLOSC_MEMCPYED;
  if (nb < MIN_BUFFERSIZE) flags |= BLOSC_MEMCPYED;
  if (doshuffle == BLOSC_SHUFFLE) flags |= BLOSC_DOSHUFFLE;
  if (doshuffle == BLOSC_BITSHUFFLE) flags |= BLOSC_DOBITSHUFFLE;
  dont_split = !split_block(compcode, ts, bs);
  flags |= dont_split << 4;
  flags |= compformat << 5;

  src_dev = (nb > 0) ? b2_ptr_is_device(src) : 0;
  dest_dev = pl ? pl_dest_dev : b2_ptr_is_device(dest);

  /* blosc_compress_context, blosc.c:1250-1279 */
  if ((flags & BLOSC_MEMCPYED) && nb + BLOSC_MAX_OVERHEAD > dsz) return 0;
  if (check_threads(numinternalthreads, nb, bs) < 0) return -1;
  if (flags & BLOSC_MEMCPYED) {
    make_header(hdr, 1, flags, ts, nb, bs, nb + 16);
    if (pl && !(dest = frame_place(pl, nb + 16))) return 0;
    return emit_memcpyed(hdr, src, src_dev, dest, dest_dev, nb);
  }

  w = ws_acquire();
  if (!w) return -1;
  do {
    FilterArgs fa;
    EncodeArgs ea;
    ScanArgs sa;
    CompactArgs ca;
    const int32_t nfull = nb / bs;
    /* stage the input on the device if it lives in host memory */
    if (src_dev) d_src = (const uint8_t*)src;
    else {
      if (buf_ensure(&w->in, (size_t)nb + 64)) break;
      if (h2d_any(w, w->in.p, src, (size_t)nb)) break;
      d_src = (const uint8_t*)w->in.p;
    }
    /* filter (blosc.c:607-622): byte shuffle needs typesize > 1; bitshuffle applies per block when bsize >= typesize */
    dofilter = ((flags & BLOSC_DOSHUFFLE) && ts > 1) || (flags & BLOSC_DOBITSHUFFLE);
    if ((flags & BLOSC_DOSHUFFLE) && ts > 1) fmode = FILT_SHUFFLE; else fmode = FILT_BITSHUFFLE;
    d_codec_in = d_src;
    if (dofilter) {
      if (buf_ensure(&w->filt, (size_t)nb + 64)) break;
      fa.src = d_src; fa.dst = (uint8_t*)w->filt.p; fa.nbytes = nb; fa.blocksize = bs; fa.typesize = ts; fa.mode = fmode;
      if (b2_launch_filter(&fa, w->stream)) break;
      d_codec_in = (const uint8_t*)w->filt.p;
    }
    /* one LZ stream per split (blosc.c:628-634) */
    nsplits = dont_split ? 1 : ts;
    memset(&ea, 0, sizeof ea);
    ea.map.nbytes = nb; ea.map.blocksize = bs; ea.map.nsplits = nsplits; ea.map.first_block = 0;
    ea.map.nfull = nfull; ea.map.leftover = leftover; ea.map.nstreams = nfull * nsplits + (leftover ? 1 : 0);
    if (buf_ensure(&w->slots, (size_t)nb + 64)) break;
    if (buf_ensure(&w->csizes, (size_t)ea.map.nstreams * 4 + 64)) break;
    if (buf_ensure(&w->needs, (size_t)ea.map.nstreams * 4 + 64)) break;
    if (buf_ensure(&w->bstarts, (size_t)nblocks * 4 + 64)) break;
    ea.in = d_codec_in; ea.slots = (uint8_t*)w->slots.p; ea.csizes = (int*)w->csizes.p; ea.needs = (int*)w->needs.p;
    ea.codec = (compcode == BLOSC_LZ4 || compcode == BLOSC_LZ4HC) ? B2_CODEC_LZ4 : B2_CODEC_BLOSCLZ;
    ea.clevel = clevel; ea.accel = 10 - clevel;                          /* blosc.c:577-587 */
    ea.split_flag = !dont_split;
    ea.many = (pl && pl->many) || ws_busy(w->dev) > 1;      /* a frame, or other _ctx calls running on this device */
    ea.table_bytes = ea.codec == B2_CODEC_LZ4 ? 16384 : (4 << (clevel == 1 ? 12 : (clevel == 2 ? 13 : 14)));
    /* BloscLZ at clevel >= 3: 17-bit packed table (34 KiB instead of 64 KiB) when every stream is <= 128 KiB */
    if (ea.codec == B2_CODEC_BLOSCLZ && clevel >= 3 && bs / nsplits <= 131072 && leftover <= 131072) ea.table_bytes = 32768 + 2048;
    /* LZ4, on request: 17-bit packed table, 8.5 KiB instead of 16 KiB per stream (twice the streams per SM),
     * when every stream is long enough for the 4096-entry table (lz4.c:710) and at most 128 KiB */
    if (ea.codec == B2_CODEC_LZ4 && lz4_pack_wanted(pl) && leftover == 0 && bs / nsplits >= 65547 && bs / nsplits <= 131072)
      ea.table_bytes = 8192 + 512;
    ea.queue = w->d_result + B2_R_QUEUE; ea.queue_base_host = &w->queue_base; ea.done = w->d_result + B2_R_DONE;
    sa.csizes = ea.csizes; sa.needs = ea.needs; sa.blocksize = bs; sa.leftover = leftover;
    /* do_job runs serial_blosc when nthreads == 1 or there is at most one block (blosc.c:910) */
    sa.serial = (numinternalthreads == 1 || nb / bs <= 1);
    sa.bstarts = (int*)w->bstarts.p; sa.result = w->d_result;
    sa.nsplits = nsplits; sa.nfull = nfull; sa.has_leftover = leftover > 0; sa.destsize = dsz;
    /* the warp that finishes the last stream also does the block scan (no separate 1-CTA launch) */
    ea.fold_scan = nblocks <= B2_FOLD_SCAN_MAX_BLOCKS || compcode == BLOSC_SNAPPY;   /* snappy's scan is always folded */
    ea.scan = sa;
    launched = 1;
    memset(&ca, 0, sizeof ca);
    if (compcode == BLOSC_ZSTD || compcode == BLOSC_ZLIB || compcode == BLOSC_SNAPPY || compcode == BLOSC_LZ4HC ||
        (compcode == BLOSC_LZ4 && lz4_fast_wanted())) {
      /* The segment-parallel encoders (b2_launch_fast): a hash-chain index, one parse CTA per window with one lane per
       * segment, then one warp per stream.  LZ4 and lz4hc parse into LZ4 bytes that compaction stitches together; the
       * zstd (dev_zstdenc.cuh), DEFLATE (dev_deflate.cuh, offsets <= 32768) and snappy (dev_snappy.cuh) encoders parse
       * into sequence records, then one warp writes each stream. */
      FastArgs fx;
      const int neblock = bs / nsplits;
      const int longest = neblock > leftover ? neblock : leftover;
      /* a window is the whole stream when it fits in B2_FAST_WIN_MAX, rounded up to whole warps of segments */
      int win = (longest + 32 * B2_FAST_SEG - 1) / (32 * B2_FAST_SEG) * (32 * B2_FAST_SEG);
      long long nsegs;
      if (win > B2_FAST_WIN_MAX) win = B2_FAST_WIN_MAX;
      memset(&fx, 0, sizeof fx);
      fx.map = ea.map; fx.in = ea.in; fx.slots = ea.slots; fx.csizes = ea.csizes; fx.needs = ea.needs;
      fx.segs_full = (neblock + B2_FAST_SEG - 1) / B2_FAST_SEG; fx.segs_left = (leftover + B2_FAST_SEG - 1) / B2_FAST_SEG;
      fx.win_bytes = win; fx.threads = win / B2_FAST_SEG;
      fx.groups_full = (neblock + win - 1) / win; fx.groups_left = (leftover + win - 1) / win;
      nsegs = (long long)nfull * nsplits * fx.segs_full + fx.segs_left;
      fx.codec = compcode == BLOSC_ZSTD ? B2_CODEC_ZSTD : compcode == BLOSC_ZLIB ? B2_CODEC_ZLIB
               : compcode == BLOSC_SNAPPY ? B2_CODEC_SNAPPY : B2_CODEC_LZ4;
      /* effort (chain depth, accel, lazy matching).  "lz4hc" (blosc.c:422-433 hands clevel to LZ4_compress_HC) takes
       * LZ4HC's search effort -- 2^(level-1) candidates, capped -- and no skipping over literals; so do zstd
       * (blosc.c:499-511 maps clevel to zstd levels 1..22) and zlib.  Snappy is a speed codec: fast LZ4's effort. */
      fx.hash_mask = 0xffff;
      if (compcode == BLOSC_LZ4) { fx.depth = 3 * clevel + 1; fx.accel = ea.accel; fx.lazy = 0; }
      else if (compcode == BLOSC_SNAPPY) { fx.depth = 3 * clevel + 1; fx.accel = 1; fx.lazy = 0; }
      else { fx.depth = clevel <= 2 ? 4 : (clevel >= 8 ? 128 : (1 << (clevel - 1))); fx.accel = 1; fx.lazy = 64; }
      /* zlib's FLEVEL for compress2(.., clevel) (blosc.c:472-483, deflate.c) */
      fx.flevel = clevel < 2 ? 0 : (clevel < 6 ? 1 : (clevel == 6 ? 2 : 3));
      fx.ebsize = bs + 4 * ts;
      if (buf_ensure(&w->prev, 2 * (size_t)nb + 64)) break;
      fx.prev = (uint16_t*)w->prev.p;
      if (fx.codec == B2_CODEC_LZ4) {
        if (buf_ensure(&w->segs, ((size_t)nsegs + 8) * sizeof(FastSeg))) break;
        if (buf_ensure(&w->ptail, (size_t)ea.map.nstreams * 4 + 64)) break;
        fx.segs = (FastSeg*)w->segs.p; fx.ptail = (int*)w->ptail.p;
        ca.segs = fx.segs; ca.ptail = fx.ptail; ca.segs_full = fx.segs_full; ca.segs_left = fx.segs_left;
      } else {
        /* the records need 256 bytes per segment; whichever of the staging / filter buffers does not hold the
         * codec input is free for them */
        b2_buf* recs = d_codec_in == (const uint8_t*)w->in.p ? &w->filt : &w->in;
        if (buf_ensure(recs, (size_t)nsegs * B2_FAST_SEG + 64)) break;
        if (buf_ensure(&w->segs, (size_t)nsegs * 4 + 64)) break;
        fx.recs = (uint32_t*)recs->p; fx.nrec = (uint32_t*)w->segs.p;
      }
      fx.queue = ea.queue; fx.queue_base_host = ea.queue_base_host; fx.done = ea.done;
      fx.fold_scan = ea.fold_scan; fx.scan = sa;
      if (b2_launch_fast(&fx, w->stream)) break;
    } else if (b2_launch_encode(&ea, w->stream)) break;
    if (!ea.fold_scan && b2_launch_scan(&sa, w->stream)) break;
    if (dest_dev && !pl) d_dest = (uint8_t*)dest;
    else { if (buf_ensure(&w->out, (size_t)dsz + 64)) break; d_dest = (uint8_t*)w->out.p; }
    ca.map = ea.map; ca.in = d_codec_in; ca.slots = ea.slots; ca.csizes = ea.csizes; ca.bstarts = sa.bstarts;
    ca.result = w->d_result; ca.dest = d_dest;
    ca.hdr0 = (uint32_t)BLOSC_VERSION_FORMAT | (1u << 8) | ((uint32_t)flags << 16) | ((uint32_t)ts << 24);
    ca.nbytes32 = nb; ca.nblocks = nblocks;
    if (b2_launch_compact(&ca, w->stream)) break;
    if (b2_copy_d2h(w->h_result, w->d_result, 8, w->stream)) break;
    if (b2_stream_sync(w->stream)) break;
    if (w->h_result[1]) {                                                 /* fits */
      const int32_t cbytes = w->h_result[0];
      if (pl && !(dest = frame_place(pl, cbytes))) { result = 0; break; }
      if (!dest_dev) {
        if (d2h_any(w, dest, d_dest, (size_t)cbytes)) break;
      } else if (pl) {
        if (copy_any(dest, 1, d_dest, 1, (size_t)cbytes, w->stream)) break;
      }
      result = cbytes;
    } else if (nb + BLOSC_MAX_OVERHEAD <= dsz) {                          /* blosc.c:1264-1272 */
      result = -2;   /* marker: redo as MEMCPYED after releasing the workspace */
    } else {
      make_header(hdr, 1, flags, ts, nb, bs, 0);                          /* blosc.c:1275 with ntbytes == 0 */
      if (!pl && copy_any(dest, dest_dev, hdr, 0, 16, w->stream)) break;
      result = 0;
    }
  } while (0);
  if (result == -1 && launched) ws_reset_counters(w);                      /* a failed call must not leave the counters dirty */
  ws_release(w);
  if (result == -2) {
    flags |= BLOSC_MEMCPYED;
    make_header(hdr, 1, flags, ts, nb, bs, nb + 16);
    if (pl && !(dest = frame_place(pl, nb + 16))) return 0;
    return emit_memcpyed(hdr, src, src_dev, dest, dest_dev, nb);
  }
  return result;
}

int blosc_compress_ctx(int clevel, int doshuffle, size_t typesize, size_t nbytes, const void* src, void* dest,
                       size_t destsize, const char* compressor, size_t blocksize, int numinternalthreads) {
  return compress_impl(clevel, doshuffle, typesize, nbytes, src, dest, destsize, compressor, blocksize,
                       numinternalthreads, NULL, 0);
}

/* ------------------------------------------------------------------------- */
/* decompression                                                              */
/* ------------------------------------------------------------------------- */
typedef struct {
  int version, versionlz, flags, typesize;
  int32_t nbytes, blocksize, cbytes, nblocks, leftover;
} b2_hdr;

static void parse_header(const uint8_t* h, b2_hdr* o) {                    /* blosc.c:1453-1461 */
  o->version = h[0]; o->versionlz = h[1]; o->flags = h[2]; o->typesize = h[3];
  o->nbytes = rd_i32(h + 4); o->blocksize = rd_i32(h + 8); o->cbytes = rd_i32(h + 12);
  o->nblocks = 0; o->leftover = 0;
}

static int codec_from_header(const b2_hdr* h, int* codec) {                /* blosc.c:525-574 */
  const int fmt = (h->flags & 0xe0) >> 5;
  if (fmt == BLOSC_BLOSCLZ_FORMAT) { if (h->versionlz != BLOSC_BLOSCLZ_VERSION_FORMAT) return -9; *codec = B2_CODEC_BLOSCLZ; return 0; }
  if (fmt == BLOSC_LZ4_FORMAT) { if (h->versionlz != BLOSC_LZ4_VERSION_FORMAT) return -9; *codec = B2_CODEC_LZ4; return 0; }
  if (fmt == BLOSC_SNAPPY_FORMAT && snappy_enabled()) {               /* blosc.c:545-553 */
    if (h->versionlz != BLOSC_SNAPPY_VERSION_FORMAT) return -9;
    *codec = B2_CODEC_SNAPPY;
    return 0;
  }
  if (fmt == BLOSC_ZLIB_FORMAT) { if (h->versionlz != BLOSC_ZLIB_VERSION_FORMAT) return -9; *codec = B2_CODEC_ZLIB; return 0; }   /* blosc.c:556-561 */
  if (fmt == BLOSC_ZSTD_FORMAT) { if (h->versionlz != BLOSC_ZSTD_VERSION_FORMAT) return -9; *codec = B2_CODEC_ZSTD; return 0; }   /* blosc.c:565-571 */
  return -5;
}

/* Launch the decode (and unfilter) of `count` blocks of a chunk that is already on the device into `d_out` (device).
 * d_blocks NULL: blocks [first, first+count), and d_out represents buffer offsets [first*blocksize, ...).  Otherwise
 * d_blocks is a device list of `count` ascending block numbers and the j-th decodes to d_out + j*blocksize; has_left
 * says whether the last of them is the chunk's short last block.  The verdict lands in B2_R_STATUS_OUT. */
static int launch_decode_blocks(b2_ws* w, const b2_hdr* h, int codec, const uint8_t* d_chunk, int first, int count,
                                const int* d_blocks, int has_left, uint8_t* d_out) {
  DecodeArgs da;
  FilterArgs fa;
  const int ts = h->typesize, bs = h->blocksize;
  const int dont_split = (h->flags & 0x10) >> 4;
  const int doshuffle = (h->flags & BLOSC_DOSHUFFLE) && ts > 1;
  const int dobitshuffle = !doshuffle && (h->flags & BLOSC_DOBITSHUFFLE);
  const int nfull = count - has_left;
  const long long span = (long long)nfull * bs + (has_left ? h->leftover : 0);
  uint8_t* d_codec_out = d_out;
  memset(&da, 0, sizeof da);
  /* blosc.c:749-757: split only if typesize <= 16 and >= 128 elements per block */
  da.map.nsplits = (!dont_split && ts <= MAX_SPLITS && bs / ts >= MIN_BUFFERSIZE) ? ts : 1;
  da.map.nbytes = h->nbytes; da.map.blocksize = bs; da.map.first_block = d_blocks ? 0 : first; da.map.nfull = nfull;
  da.map.leftover = has_left ? h->leftover : 0;
  da.map.nstreams = nfull * da.map.nsplits + (has_left ? 1 : 0);
  da.blocks = d_blocks;
  if (doshuffle || dobitshuffle) {
    if (buf_ensure(&w->filt, (size_t)span + 64)) return -1;
    d_codec_out = (uint8_t*)w->filt.p;
  }
  da.chunk = d_chunk; da.cbytes = h->cbytes; da.out = d_codec_out; da.out_shift = d_blocks ? 0 : (long long)first * bs;
  da.codec = codec; da.status = w->d_result + B2_R_STATUS; da.queue = w->d_result + B2_R_QUEUE;
  da.queue_base_host = &w->queue_base;
  da.done = w->d_result + B2_R_DONE; da.status_out = w->d_result + B2_R_STATUS_OUT;
  da.many = ws_busy(w->dev) > 1;
  if (b2_launch_decode(&da, w->stream)) { ws_reset_counters(w); return -1; }
  if (doshuffle || dobitshuffle) {
    fa.src = d_codec_out; fa.dst = d_out; fa.nbytes = span; fa.blocksize = bs; fa.typesize = ts;
    fa.mode = doshuffle ? FILT_UNSHUFFLE : FILT_BITUNSHUFFLE;
    if (b2_launch_filter(&fa, w->stream)) { ws_reset_counters(w); return -1; }
  }
  return 0;
}

/* Decode blocks [first, first+count) of a chunk that is already on the device into `d_out`
 * (device), which represents buffer offsets [first*blocksize, ...).  Shared by decompress and a one-range read. */
static int decode_blocks(b2_ws* w, const b2_hdr* h, int codec, const uint8_t* d_chunk, int first, int count,
                         uint8_t* d_out) {
  const int has_left = h->leftover > 0 && first + count == h->nblocks;
  if (launch_decode_blocks(w, h, codec, d_chunk, first, count, NULL, has_left, d_out)) return -1;
  if (b2_copy_d2h(w->h_result + B2_R_STATUS_OUT, w->d_result + B2_R_STATUS_OUT, 4, w->stream) || b2_stream_sync(w->stream)) {
    ws_reset_counters(w);
    return -1;
  }
  return w->h_result[B2_R_STATUS_OUT] < 0 ? w->h_result[B2_R_STATUS_OUT] : 0;
}

/* max_cbytes >= 0 (frames): the chunk lives in a slot of that many bytes and must decode to exactly
 * expect_nbytes -- a chunk header that claims more is refused before anything is copied */
static int decompress_impl(const void* src, void* dest, size_t destsize, int numinternalthreads, long long max_cbytes,
                           long long expect_nbytes) {
  uint8_t hb[16];
  b2_hdr h;
  int src_dev, dest_dev, codec = 0, rc, result = -1;
  b2_ws* w;

  src_dev = b2_ptr_is_device(src);
  if (copy_some(hb, 0, src, src_dev, 16)) return -1;
  parse_header(hb, &h);
  if (max_cbytes >= 0 && (h.cbytes < BLOSC_MAX_OVERHEAD || h.cbytes > max_cbytes || h.nbytes != expect_nbytes)) return -1;

  /* blosc_run_decompression_with_context, blosc.c:1463-1508 */
  if (h.nbytes == 0) return 0;
  if (h.blocksize <= 0 || (size_t)h.blocksize > destsize || (size_t)h.blocksize > BLOSC_MAX_BLOCKSIZE || h.typesize <= 0)
    return -1;
  if (h.version != BLOSC_VERSION_FORMAT) return -1;
  if (h.flags & 0x08) return -1;
  h.nblocks = h.nbytes / h.blocksize; h.leftover = h.nbytes % h.blocksize;
  if (h.leftover > 0) h.nblocks++;
  if (h.nbytes > (int32_t)destsize) return -1;
  dest_dev = b2_ptr_is_device(dest);
  if (h.flags & BLOSC_MEMCPYED) {
    if (h.nbytes + BLOSC_MAX_OVERHEAD != h.cbytes) return -1;
  } else {
    rc = codec_from_header(&h, &codec);
    if (rc) return rc;
    if (h.nblocks > (h.cbytes - 16) / 4) return -1;
  }
  /* A negative header nbytes passes every check above in the reference too; its block loop then runs
   * zero times (nblocks <= 0, blosc.c:815, :910) and the call returns 0 without touching memory. */
  if (h.nblocks <= 0) return 0;
  if (check_threads(numinternalthreads, h.nbytes, h.blocksize) < 0) return -1;

  if (h.flags & BLOSC_MEMCPYED)                                            /* blosc.c:843-848 */
    return copy_some(dest, dest_dev, (const uint8_t*)src + 16, src_dev, (size_t)h.nbytes) ? -1 : h.nbytes;

  w = ws_acquire();
  if (!w) return -1;
  do {
    const uint8_t* d_chunk;
    uint8_t* d_out;
    if (src_dev) d_chunk = (const uint8_t*)src;
    else {
      if (buf_ensure(&w->in, (size_t)h.cbytes + 64)) break;
      if (h2d_any(w, w->in.p, src, (size_t)h.cbytes)) break;
      d_chunk = (const uint8_t*)w->in.p;
    }
    if (dest_dev) d_out = (uint8_t*)dest;
    else { if (buf_ensure(&w->out, (size_t)h.nbytes + 64)) break; d_out = (uint8_t*)w->out.p; }
    rc = decode_blocks(w, &h, codec, d_chunk, 0, h.nblocks, d_out);
    if (rc < 0) { result = -1; break; }                                    /* blosc.c:1511-1514 */
    if (!dest_dev) {
      if (d2h_any(w, dest, d_out, (size_t)h.nbytes)) break;
    }
    result = h.nbytes;
  } while (0);
  ws_release(w);
  return result;
}

int blosc_decompress_ctx(const void* src, void* dest, size_t destsize, int numinternalthreads) {
  return decompress_impl(src, dest, destsize, numinternalthreads, -1, -1);
}

/* the chunk-header checks of blosc_getitem (blosc.c:1574-1631), with its return codes; 0 when the chunk is readable */
static int getitem_header(const void* src, int src_dev, long long max_cbytes, b2_hdr* h, int* codec) {
  uint8_t hb[16];
  int rc;
  if (copy_some(hb, 0, src, src_dev, 16)) return -1;
  parse_header(hb, h);
  if (max_cbytes >= 0 && (h->cbytes < BLOSC_MAX_OVERHEAD || h->cbytes > max_cbytes)) return -1;
  if (h->version != BLOSC_VERSION_FORMAT) return -9;
  if (h->blocksize <= 0 || h->blocksize > h->nbytes || (size_t)h->blocksize > BLOSC_MAX_BLOCKSIZE || h->typesize <= 0)
    return -1;
  h->nblocks = h->nbytes / h->blocksize; h->leftover = h->nbytes % h->blocksize;
  if (h->leftover > 0) h->nblocks++;
  if (h->flags & BLOSC_MEMCPYED) {
    if (h->nbytes + BLOSC_MAX_OVERHEAD != h->cbytes) return -1;
  } else {
    rc = codec_from_header(h, codec);
    if (rc) return rc;
    if (h->nblocks >= (h->cbytes - 16) / 4) return -1;                     /* :1630 */
  }
  return 0;
}

/* blosc_getitem's bounds checks of one range (blosc.c:1633-1644): its bytes [*b_lo, *b_hi), empty when b_hi <= b_lo */
static int getitem_range(const b2_hdr* h, int start, int nitems, long long* b_lo, long long* b_hi) {
  const int rc = b2_range_check(start, nitems, h->typesize, h->nbytes, b_lo, b_hi);
  if (rc == 1) { fprintf(stderr, "`start` out of bounds"); return -1; }
  if (rc == 2) { fprintf(stderr, "`start`+`nitems` out of bounds"); return -1; }
  return 0;
}

/* ------------------------------------------------------------------------- */
/* item ranges of one chunk in one pass (blosc_getitem, blosc_b200_getitems)  */
/* ------------------------------------------------------------------------- */
/* Every block that some range overlaps is decoded exactly once, by one decode launch over the sorted list of those
 * blocks: the j-th listed block decodes to j * blocksize of a compact scratch (StreamMap.blocks).  A range covers a
 * run of consecutive blocks, which stay adjacent in the list, so it is one contiguous span of the scratch.  One
 * unfilter launch and one gather launch (gather_kernel) then copy every range to its place in dest.  A single range
 * needs neither the list nor the gather: its blocks decode as one run and one copy moves it to dest. */
typedef struct { long long lo, hi; } b2_iv;

static int cmp_iv(const void* a, const void* b) {
  const b2_iv *x = (const b2_iv*)a, *y = (const b2_iv*)b;
  return x->lo < y->lo ? -1 : x->lo > y->lo;
}
static int cmp_i32(const void* a, const void* b) {
  const int32_t x = *(const int32_t*)a, y = *(const int32_t*)b;
  return x < y ? -1 : x > y;
}

/* sorts iv[0..n) by lo and merges the intervals that overlap or touch (hi is exclusive); returns the new count */
static int merge_ivs(b2_iv* iv, int n) {
  int k = 0, i;
  if (n == 0) return 0;
  qsort(iv, (size_t)n, sizeof *iv, cmp_iv);
  for (i = 1; i < n; i++) {
    if (iv[i].lo <= iv[k].hi) { if (iv[i].hi > iv[k].hi) iv[k].hi = iv[i].hi; }
    else iv[++k] = iv[i];
  }
  return k + 1;
}

/* Stage what the decoder reads of a host-resident chunk: the header with bstarts[] and, for every listed block (the
 * list is ascending), its bytes from its bstart to the next bstart above it; adjacent spans are copied as one.  -1 when
 * a listed block's bstart is out of bounds (blosc_d would refuse it, blosc.c:761). */
static int stage_blocks(b2_ws* w, const b2_hdr* h, const uint8_t* hs, const int* blocks, int count) {
  const size_t index_end = 16 + 4 * (size_t)h->nblocks;
  const int run = blocks[count - 1] - blocks[0] == count - 1;              /* consecutive block numbers */
  int32_t* sorted = run ? NULL : (int32_t*)malloc(4 * (size_t)h->nblocks + 4);
  b2_iv* iv = (b2_iv*)malloc(sizeof(b2_iv) * (size_t)count + sizeof(b2_iv));
  int i, n = 0, rc = -1;
  do {
    if ((!run && !sorted) || !iv) break;
    if (run) {
      /* one span, from the lowest of their bstarts to the next bstart above the highest: two linear passes over
       * bstarts[], no sort, whatever the chunk's number of blocks */
      int32_t lo = h->cbytes, hi = 0, cut = h->cbytes;
      for (i = 0; i < count; i++) {
        const int32_t bs_b = rd_i32(hs + 16 + 4 * (size_t)(blocks[0] + i));
        if (bs_b < (int32_t)index_end || bs_b > h->cbytes) break;
        if (bs_b < lo) lo = bs_b;
        if (bs_b > hi) hi = bs_b;
      }
      if (i < count) break;
      for (i = 0; i < h->nblocks; i++) {
        const int32_t bs_b = rd_i32(hs + 16 + 4 * (size_t)i);
        if (bs_b > hi && bs_b < cut) cut = bs_b;
      }
      iv[0].lo = lo; iv[0].hi = cut; n = 1;
    } else {
      for (i = 0; i < h->nblocks; i++) sorted[i] = rd_i32(hs + 16 + 4 * (size_t)i);
      qsort(sorted, (size_t)h->nblocks, 4, cmp_i32);
      for (i = 0; i < count; i++) {
        const int32_t bs_b = rd_i32(hs + 16 + 4 * (size_t)blocks[i]);
        int lo = 0, hi = h->nblocks;
        if (bs_b < (int32_t)index_end || bs_b > h->cbytes) break;
        while (lo < hi) { const int m = (lo + hi) / 2; if (sorted[m] <= bs_b) lo = m + 1; else hi = m; }   /* first above */
        iv[n].lo = bs_b;
        iv[n].hi = (lo < h->nblocks && sorted[lo] < h->cbytes) ? sorted[lo] : h->cbytes;
        n++;
      }
      if (i < count) break;
      n = merge_ivs(iv, n);
    }
    if (buf_ensure(&w->in, (size_t)h->cbytes + 64)) break;
    if (h2d_any(w, w->in.p, hs, index_end)) break;
    for (i = 0; i < n; i++)
      if (h2d_any(w, (uint8_t*)w->in.p + iv[i].lo, hs + iv[i].lo, (size_t)(iv[i].hi - iv[i].lo))) break;
    rc = i < n ? -1 : 0;
  } while (0);
  free(sorted); free(iv);
  return rc;
}

/* The range table of the gather, in one copy.  A host dest receives the ranges packed, from a device staging buffer
 * (w->slots), so their destinations become their positions in it. */
static int upload_ranges(b2_ws* w, GatherRange* tab, int nr, long long total, int dest_dev) {
  int r;
  if (!dest_dev) {
    for (r = 0; r < nr; r++) tab[r].dst = tab[r].pos;
    if (buf_ensure(&w->slots, (size_t)total + 64)) return -1;
  }
  if (buf_ensure(&w->segs, sizeof(GatherRange) * ((size_t)nr + 1) + 64)) return -1;
  return b2_copy_h2d(w->segs.p, tab, sizeof(GatherRange) * ((size_t)nr + 1), w->stream);
}

/* The execution tail of getitems, shared by its host plan and its GPU plan.  On entry the gather table (nr + 1
 * entries; dst = pos when dest is host memory) is in w->segs, and w->slots has room for `total` bytes when dest is host
 * memory.  d_src is the gather's source when it is already on the device (a memcpyed chunk); when it is NULL the
 * `count` blocks listed in w->bstarts (ascending; has_left: the last is the chunk's short last block) are decoded and
 * unfiltered from d_chunk into a compact scratch.  A host dest then receives the ranges from w->slots: at dest +
 * at_b[0] when `contiguous`, else range r at dest + at_b[r] (tab: the table on the host).  Returns total, or blosc_d's
 * code when a stream fails to decode (dest is then untouched). */
static long long getitems_run(b2_ws* w, const b2_hdr* h, int codec, const uint8_t* d_src, const uint8_t* d_chunk,
                              int count, int has_left, int nr, long long total, void* dest, int dest_dev,
                              const GatherRange* tab, const long long* at_b, int contiguous) {
  GatherArgs ga;
  const int* status = NULL;
  long long result = -1;
  uint8_t* tmp = NULL;
  int r;
  memset(&ga, 0, sizeof ga);
  do {
    if (!d_src) {
      if (buf_ensure(&w->out, (size_t)count * (size_t)h->blocksize + 64)) break;
      if (launch_decode_blocks(w, h, codec, d_chunk, 0, count, (const int*)w->bstarts.p, has_left, (uint8_t*)w->out.p)) break;
      d_src = (const uint8_t*)w->out.p;
      status = w->d_result + B2_R_STATUS_OUT;
    }
    ga.src = d_src; ga.dst = dest_dev ? (uint8_t*)dest : (uint8_t*)w->slots.p; ga.ranges = (const GatherRange*)w->segs.p;
    ga.nranges = nr; ga.total = total; ga.status = status;
    if (b2_launch_gather(&ga, w->stream)) { ws_reset_counters(w); break; }
    if (b2_copy_d2h(w->h_result + B2_R_STATUS_OUT, w->d_result + B2_R_STATUS_OUT, 4, w->stream) || b2_stream_sync(w->stream)) {
      ws_reset_counters(w);
      break;
    }
    if (status && w->h_result[B2_R_STATUS_OUT] < 0) { result = w->h_result[B2_R_STATUS_OUT]; break; }
    if (!dest_dev) {
      if (contiguous) {
        if (d2h_any(w, (uint8_t*)dest + at_b[0], w->slots.p, (size_t)total)) break;
      } else {                                                             /* scattered (frame pieces) */
        if (!(tmp = (uint8_t*)malloc((size_t)total))) break;
        if (d2h_any(w, tmp, w->slots.p, (size_t)total)) break;
        for (r = 0; r < nr; r++) memcpy((uint8_t*)dest + at_b[r], tmp + tab[r].pos, (size_t)(tab[r + 1].pos - tab[r].pos));
      }
    }
    result = total;
  } while (0);
  free(tmp);
  return result;
}

/* The host plan: `n` ranges of one chunk, in host memory; range r goes to dest + dsts[r] (back to back in request order
 * when dsts is NULL).  The header and every range are validated before anything is launched or written.  Returns the
 * bytes written, or blosc_getitem's code. */
static long long getitems_chunk(const void* src, long long max_cbytes, int n, const int* starts, const int* nitems,
                                const long long* dsts, void* dest) {
  b2_hdr h;
  int src_dev, dest_dev, codec = 0, rc, r, nr = 0, contiguous = 1;
  long long total = 0, result = -1;
  b2_ws* w = NULL;
  GatherRange* tab = NULL;       /* [nr + 1] non-empty ranges; src: offset in the gather's source, set once that is known */
  long long* lo_b = NULL;        /* [2n]: first byte of each listed range inside the chunk, then its dest offset */
  long long* at_b;
  b2_iv* iv = NULL;
  int* blocks = NULL;
  uint8_t* tmp = NULL;

  if (n <= 0) return 0;
  src_dev = b2_ptr_is_device(src);
  rc = getitem_header(src, src_dev, max_cbytes, &h, &codec);
  if (rc) return rc;
  tab = (GatherRange*)malloc(sizeof(GatherRange) * ((size_t)n + 1));
  lo_b = (long long*)malloc(2 * sizeof(long long) * (size_t)n);
  if (!tab || !lo_b) { free(tab); free(lo_b); return -1; }
  at_b = lo_b + n;
  for (r = 0; r < n; r++) {
    long long b_lo, b_hi;
    const long long at = dsts ? dsts[r] : total;
    if (getitem_range(&h, starts[r], nitems[r], &b_lo, &b_hi)) { free(tab); free(lo_b); return -1; }
    if (b_hi <= b_lo) continue;                                            /* empty: 0 bytes, as blosc_getitem */
    tab[nr].src = b_lo; tab[nr].dst = at; tab[nr].pos = total;
    lo_b[nr] = b_lo; at_b[nr] = at;
    contiguous &= at - tab[0].dst == total;
    total += b_hi - b_lo;
    nr++;
  }
  tab[nr].src = tab[nr].dst = 0; tab[nr].pos = total;
  if (nr == 0) { free(tab); free(lo_b); return 0; }
  dest_dev = b2_ptr_is_device(dest);

  if ((h.flags & BLOSC_MEMCPYED) && (nr == 1 || (!src_dev && !dest_dev))) {  /* :1678-1683, one copy per range */
    for (r = 0, rc = 0; r < nr && !rc; r++)
      rc = copy_some((uint8_t*)dest + tab[r].dst, dest_dev, (const uint8_t*)src + 16 + tab[r].src, src_dev,
                     (size_t)(tab[r + 1].pos - tab[r].pos));
    free(tab); free(lo_b);
    return rc ? -1 : total;
  }

  w = ws_acquire();
  if (!w) { free(tab); free(lo_b); return -1; }
  do {
    const uint8_t* d_src = NULL;
    const uint8_t* d_chunk = NULL;
    int count = 0, has_left = 0;
    if (h.flags & BLOSC_MEMCPYED) {
      if (src_dev) d_src = (const uint8_t*)src + 16;                       /* ranges read the payload in place */
      else {                                                               /* the ranges, packed, cross PCIe once */
        if (!(tmp = (uint8_t*)malloc((size_t)total))) break;
        for (r = 0; r < nr; r++) {
          memcpy(tmp + tab[r].pos, (const uint8_t*)src + 16 + tab[r].src, (size_t)(tab[r + 1].pos - tab[r].pos));
          tab[r].src = tab[r].pos;
        }
        if (buf_ensure(&w->in, (size_t)total + 64) || h2d_any(w, w->in.p, tmp, (size_t)total)) break;
        d_src = (const uint8_t*)w->in.p;
      }
      if (upload_ranges(w, tab, nr, total, dest_dev)) break;
    } else {
      /* the touched blocks: one interval of block numbers per range, merged, then listed in ascending order */
      const int bs = h.blocksize;
      int nv, k;
      if (!(iv = (b2_iv*)malloc(sizeof(b2_iv) * (size_t)nr))) break;
      for (r = 0; r < nr; r++) {
        iv[r].lo = lo_b[r] / bs;
        iv[r].hi = (lo_b[r] + (tab[r + 1].pos - tab[r].pos) - 1) / bs + 1;
      }
      nv = merge_ivs(iv, nr);
      for (k = 0; k < nv; k++) count += (int)(iv[k].hi - iv[k].lo);
      if (!(blocks = (int*)malloc(sizeof(int) * (size_t)count))) break;
      for (k = 0, count = 0; k < nv; k++) {
        long long b;
        for (b = iv[k].lo; b < iv[k].hi; b++) blocks[count++] = (int)b;
      }
      if (src_dev) d_chunk = (const uint8_t*)src;
      else {
        if (stage_blocks(w, &h, (const uint8_t*)src, blocks, count)) break;
        d_chunk = (const uint8_t*)w->in.p;
      }
      if (nr == 1) {                               /* one range: its run of blocks decodes with no list and no gather */
        if (buf_ensure(&w->out, (size_t)count * (size_t)bs + 64)) break;
        rc = decode_blocks(w, &h, codec, d_chunk, blocks[0], count, (uint8_t*)w->out.p);
        if (rc < 0) { result = rc; break; }                                /* :1689-1692 returns blosc_d's code */
        if (copy_any((uint8_t*)dest + tab[0].dst, dest_dev, (const uint8_t*)w->out.p + (lo_b[0] - (long long)blocks[0] * bs),
                     1, (size_t)total, w->stream)) break;
        result = total;
        break;
      }
      for (r = 0; r < nr; r++) {                                           /* range r -> its span of the scratch */
        const long long first = lo_b[r] / bs;
        int lo = 0, hi = count - 1;
        while (lo < hi) { const int m = (lo + hi + 1) / 2; if (blocks[m] <= first) lo = m; else hi = m - 1; }
        tab[r].src = (long long)lo * bs + (lo_b[r] - first * bs);
      }
      if (buf_ensure(&w->bstarts, sizeof(int) * (size_t)count + 64)) break;
      if (b2_copy_h2d(w->bstarts.p, blocks, sizeof(int) * (size_t)count, w->stream)) break;
      if (upload_ranges(w, tab, nr, total, dest_dev)) break;      /* before the decode: a pageable copy would wait for it */
      has_left = h.leftover > 0 && blocks[count - 1] == h.nblocks - 1;
    }
    result = getitems_run(w, &h, codec, d_src, d_chunk, count, has_left, nr, total, dest, dest_dev, tab, at_b, contiguous);
  } while (0);
  ws_release(w);
  free(tab); free(lo_b); free(iv); free(blocks); free(tmp);
  return result;
}

int blosc_getitem(const void* src, int start, int nitems, void* dest) {                 /* blosc.c:1574-1703 */
  return (int)getitems_chunk(src, -1, 1, &start, &nitems, NULL, dest);
}

/* Stage the payload of a memcpyed host chunk that the listed blocks cover, block j of the list at j * blocksize of
 * w->in; runs of consecutive blocks are copied as one. */
static int stage_memcpyed_blocks(b2_ws* w, const b2_hdr* h, const uint8_t* hs, const int* blocks, int count) {
  const long long bs = h->blocksize;
  int i = 0, j;
  if (buf_ensure(&w->in, (size_t)count * (size_t)bs + 64)) return -1;
  while (i < count) {
    long long end;
    for (j = i + 1; j < count && blocks[j] == blocks[j - 1] + 1; j++) {}
    end = ((long long)blocks[j - 1] + 1) * bs;
    if (end > h->nbytes) end = h->nbytes;
    if (h2d_any(w, (uint8_t*)w->in.p + i * bs, hs + 16 + blocks[i] * bs, (size_t)(end - blocks[i] * bs))) return -1;
    i = j;
  }
  return 0;
}

#define B2_R_PLAN 8   /* h_result words 8..13 receive the GPU plan's record (GetitemsPlan) */
#define B2_AL(x) (((x) + 15) & ~(size_t)15)

/* The GPU plan (dev_chunk.cuh plan_*_kernel), for range lists of which at least one is in device memory (a host one is
 * uploaded).  It builds the gather table in w->segs and the touched-block list in w->bstarts, both as the host plan
 * would (the table keeps empty ranges, which copy nothing), and the host reads back one small record.  A failing range
 * is reported by getitem_range on that range alone, so the code and the message are the host plan's.  A host chunk
 * also has the block list read back, to stage only the touched blocks. */
static long long getitems_gpu(const void* src, int src_dev, const b2_hdr* h, int codec, int n, const int* starts,
                              int starts_dev, const int* nitems, int nitems_dev, void* dest) {
  const int dest_dev = b2_ptr_is_device(dest);
  const int memcpyed = (h->flags & BLOSC_MEMCPYED) != 0, in_place = memcpyed && src_dev;
  const size_t tb = ((size_t)h->nblocks + PLAN_TILE - 1) / PLAN_TILE, tr = ((size_t)n + PLAN_TILE - 1) / PLAN_TILE;
  /* one scratch: the record, the tickets, the tile flags and the difference array, all zeroed; then the tiles' values,
   * the range lengths, the block slots and an uploaded host list */
  const size_t o_tk = 32, o_flag = 64, o_cover = B2_AL(o_flag + 4 * (2 * tb + tr));
  const size_t zeroed = B2_AL(o_cover + 4 * ((size_t)h->nblocks + 1));
  const size_t o_vals = zeroed, o_len = B2_AL(o_vals + 4 * 4 * tb + 8 * 2 * tr);
  const size_t o_slot = B2_AL(o_len + 8 * (size_t)n), o_up = B2_AL(o_slot + 4 * (size_t)h->nblocks);
  const size_t need = o_up + 4 * (size_t)n;
  const long long at0 = 0;
  long long result = -1;
  int* hblocks = NULL;
  b2_ws* w = ws_acquire();
  if (!w) return -1;
  do {
    PlanArgs pa;
    GetitemsPlan rec;
    uint8_t* base;
    const uint8_t* d_src = NULL;
    const uint8_t* d_chunk = NULL;
    int k;
    if (buf_ensure(&w->plan, need) || buf_ensure(&w->segs, sizeof(GatherRange) * ((size_t)n + 1) + 64)) break;
    if (!in_place && buf_ensure(&w->bstarts, 4 * (size_t)h->nblocks + 64)) break;
    base = (uint8_t*)w->plan.p;
    memset(&pa, 0, sizeof pa);
    pa.starts = starts; pa.nitems = nitems;
    if (!starts_dev || !nitems_dev) {                                      /* the host list joins the device one */
      if (h2d_any(w, base + o_up, starts_dev ? (const void*)nitems : (const void*)starts, 4 * (size_t)n)) break;
      if (starts_dev) pa.nitems = (const int*)(base + o_up); else pa.starts = (const int*)(base + o_up);
    }
    if (b2_memset_dev(base, 0, zeroed, w->stream) || b2_memset_dev(base, 0xff, 4, w->stream)) break;
    pa.nranges = n; pa.typesize = h->typesize; pa.blocksize = h->blocksize; pa.nblocks = h->nblocks;
    pa.leftover = h->leftover > 0; pa.nbytes = h->nbytes; pa.in_place = in_place;
    pa.len = (long long*)(base + o_len); pa.cover = (int*)(base + o_cover); pa.slot = (int*)(base + o_slot);
    pa.blocks = (int*)w->bstarts.p; pa.ranges = (GatherRange*)w->segs.p; pa.rec = (GetitemsPlan*)base;
    for (k = 0; k < 3; k++) {
      const size_t tiles = k < 2 ? tb : tr;
      const size_t flags_at = o_flag + 4 * (k < 2 ? k * tb : 2 * tb);
      const size_t vals_at = o_vals + (k < 2 ? 2 * 4 * k * tb : 4 * 4 * tb), width = k < 2 ? 4 : 8;
      pa.scan[k].ticket = (unsigned*)(base + o_tk) + k;
      pa.scan[k].flag = (unsigned*)(base + flags_at);
      pa.scan[k].agg = base + vals_at;
      pa.scan[k].inc = base + vals_at + width * tiles;
    }
    if (b2_launch_plan(&pa, w->stream)) break;
    if (b2_copy_d2h(w->h_result + B2_R_PLAN, base, sizeof rec, w->stream) || b2_stream_sync(w->stream)) break;
    memcpy(&rec, w->h_result + B2_R_PLAN, sizeof rec);
    if (rec.bad != 0xffffffffu) {                                          /* blosc_getitem's verdict on that range */
      int s, c;
      long long lo, hi;
      if (copy_any(&s, 0, starts + rec.bad, starts_dev, 4, w->stream) ||
          copy_any(&c, 0, nitems + rec.bad, nitems_dev, 4, w->stream)) break;
      getitem_range(h, s, c, &lo, &hi);
      break;
    }
    if (rec.total == 0) { result = 0; break; }
    if (!dest_dev && buf_ensure(&w->slots, (size_t)rec.total + 64)) break;
    if (in_place) d_src = (const uint8_t*)src + 16;
    else if (src_dev) d_chunk = (const uint8_t*)src;
    else {                                                                 /* stage the touched blocks only */
      if (!(hblocks = (int*)malloc(4 * (size_t)rec.nlisted))) break;
      if (d2h_any(w, hblocks, w->bstarts.p, 4 * (size_t)rec.nlisted)) break;
      if (memcpyed) {
        if (stage_memcpyed_blocks(w, h, (const uint8_t*)src, hblocks, rec.nlisted)) break;
        d_src = (const uint8_t*)w->in.p;
      } else {
        if (stage_blocks(w, h, (const uint8_t*)src, hblocks, rec.nlisted)) break;
        d_chunk = (const uint8_t*)w->in.p;
      }
    }
    result = getitems_run(w, h, codec, d_src, d_chunk, rec.nlisted, rec.has_left, n, rec.total, dest, dest_dev, NULL,
                          &at0, 1);
  } while (0);
  ws_release(w);
  free(hblocks);
  return result;
}

long long blosc_b200_getitems(const void* src, int nranges, const int* starts, const int* nitems, void* dest) {
  b2_hdr h;
  int starts_dev, nitems_dev, src_dev, dev, codec = 0, rc;
  if (nranges <= 0) return 0;
  starts_dev = b2_ptr_is_device(starts); nitems_dev = b2_ptr_is_device(nitems);
  if (!starts_dev && !nitems_dev) return getitems_chunk(src, -1, nranges, starts, nitems, NULL, dest);
  /* device lists: on the device the call runs on, that of src or dest when either is device memory */
  src_dev = b2_ptr_is_device(src);
  dev = src_dev ? b2_ptr_device(src) : b2_ptr_is_device(dest) ? b2_ptr_device(dest) : b2_get_device();
  if ((starts_dev && b2_ptr_device(starts) != dev) || (nitems_dev && b2_ptr_device(nitems) != dev)) {
    fprintf(stderr, "blosc_b200: starts / nitems are not on device %d, where the call runs\n", dev);
    return -1;
  }
  rc = getitem_header(src, src_dev, -1, &h, &codec);
  if (rc) return rc;
  return getitems_gpu(src, src_dev, &h, codec, nranges, starts, starts_dev, nitems, nitems_dev, dest);
}

/* ------------------------------------------------------------------------- */
/* frames: buffers larger than one chunk (SURVEY.md section 8, row f3)           */
/* ------------------------------------------------------------------------- */
/* A Blosc-1 chunk holds at most INT_MAX-16 bytes (blosc.h:40) and a single call leaves most of
 * the GPU idle (DESIGN.md section 5), so large buffers are cut into independent chunks that
 * are compressed by a few host threads at once, each on its own workspace and stream: chunk
 * i+1's PCIe transfer and filter overlap chunk i's codec kernels.  The container is a minimal
 * index in front of ordinary chunks, every one of which the reference library can decode:
 *
 *   0   "B2FR"            magic
 *   4   u8 version (1), 3 reserved bytes (0)
 *   8   u64 nbytes        uncompressed size of the whole frame
 *   16  u64 cbytes        size of the frame itself
 *   24  u32 chunksize     uncompressed bytes per chunk (the last one may be shorter)
 *   28  u32 nchunks
 *   32  u64 offset[nchunks]   from the start of the frame
 *   ..  the chunks, back to back, in order
 */
#define B2_FRAME_HDR 32
#define B2_FRAME_DEFAULT_CHUNK ((size_t)256 << 20)
#define B2_FRAME_MAX_WORKERS 8

struct b2_frame_job {
  pthread_mutex_t mu;
  pthread_cond_t cv;
  int next, commit, failed, err, nchunks, dev, dest_dev, workers;
  /* compression */
  int clevel, doshuffle, nthreads;
  size_t typesize, blocksize, chunksize, nbytes, destsize, cursor;
  const char* compressor;
  const uint8_t* src;
  uint8_t* dest;
  uint64_t* offsets;
  /* decompression */
  const uint8_t* frame;
};

static void wr_u64(uint8_t* p, uint64_t v) { int i; for (i = 0; i < 8; i++) p[i] = (uint8_t)(v >> (8 * i)); }
static uint64_t rd_u64(const uint8_t* p) { uint64_t v = 0; int i; for (i = 0; i < 8; i++) v |= (uint64_t)p[i] << (8 * i); return v; }
static void wr_u32(uint8_t* p, uint32_t v) { wr_i32(p, (int32_t)v); }
static uint32_t rd_u32(const uint8_t* p) { return (uint32_t)rd_i32(p); }

static int frame_workers(int nchunks) {
  const char* e = getenv("BLOSC_B200_FRAME_WORKERS");
  int n = e ? atoi(e) : 4;
  if (n < 1) n = 1;
  if (n > B2_FRAME_MAX_WORKERS) n = B2_FRAME_MAX_WORKERS;
  return n < nchunks ? n : nchunks;
}

/* Ordered commit: chunk `index` gets the bytes right after chunk index-1.  Returns NULL (and
 * marks the job failed) when the frame does not fit; cbytes < 0 gives up the turn after an error. */
static void* frame_place(b2_place* pl, int32_t cbytes) {
  b2_frame_job* j = pl->job;
  void* where = NULL;
  pthread_mutex_lock(&j->mu);
  while (j->commit != pl->index) pthread_cond_wait(&j->cv, &j->mu);
  if (cbytes >= 0 && !j->failed && j->cursor + (size_t)cbytes <= j->destsize) {
    j->offsets[pl->index] = j->cursor;
    where = j->dest + j->cursor;
    j->cursor += (size_t)cbytes;
  } else j->failed = 1;
  pl->placed = 1;
  j->commit++;
  pthread_cond_broadcast(&j->cv);
  pthread_mutex_unlock(&j->mu);
  return where;
}

static int frame_take(b2_frame_job* j, int* failed) {
  int i;
  pthread_mutex_lock(&j->mu);
  i = j->next < j->nchunks ? j->next++ : -1;
  *failed = j->failed;
  pthread_mutex_unlock(&j->mu);
  return i;
}

static void frame_fail(b2_frame_job* j, int rc) {
  pthread_mutex_lock(&j->mu);
  j->failed = 1;
  if (rc < 0 && !j->err) j->err = rc;
  pthread_mutex_unlock(&j->mu);
}

static void* frame_compress_worker(void* arg) {
  b2_frame_job* j = (b2_frame_job*)arg;
  int i, failed;
  b2_set_device(j->dev);
  while ((i = frame_take(j, &failed)) >= 0) {
    b2_place pl;
    const size_t off = (size_t)i * j->chunksize;
    const size_t n = j->nbytes - off < j->chunksize ? j->nbytes - off : j->chunksize;
    int rc = -1;
    pl.job = j; pl.index = i; pl.placed = 0; pl.many = j->workers > 1;
    if (!failed)
      rc = compress_impl(j->clevel, j->doshuffle, j->typesize, n, j->src + off, NULL, n + BLOSC_MAX_OVERHEAD,
                         j->compressor, j->blocksize, j->nthreads, &pl, j->dest_dev);
    if (!pl.placed) frame_place(&pl, -1);
    if (rc <= 0 && !failed) frame_fail(j, rc);
  }
  return NULL;
}

static void* frame_decompress_worker(void* arg) {
  b2_frame_job* j = (b2_frame_job*)arg;
  int i, failed;
  b2_set_device(j->dev);
  while ((i = frame_take(j, &failed)) >= 0) {
    const size_t off = (size_t)i * j->chunksize;
    const size_t n = j->nbytes - off < j->chunksize ? j->nbytes - off : j->chunksize;
    int rc;
    if (failed) continue;
    rc = decompress_impl(j->frame + j->offsets[i], j->dest + off, n, j->nthreads,
                         (long long)(j->offsets[i + 1] - j->offsets[i]), (long long)n);
    if (rc != (int)n) frame_fail(j, -1);
  }
  return NULL;
}

static int frame_run(b2_frame_job* j, void* (*fn)(void*)) {
  pthread_t th[B2_FRAME_MAX_WORKERS];
  int k, started = 0;
  pthread_mutex_init(&j->mu, NULL);
  pthread_cond_init(&j->cv, NULL);
  j->dev = b2_get_device();
  for (k = 1; k < j->workers; k++) {
    if (pthread_create(&th[started], NULL, fn, j) != 0) break;
    started++;
  }
  fn(j);                                   /* the calling thread is worker 0 */
  for (k = 0; k < started; k++) pthread_join(th[k], NULL);
  pthread_cond_destroy(&j->cv);
  pthread_mutex_destroy(&j->mu);
  return j->failed ? -1 : 0;
}

static size_t frame_chunksize(size_t chunksize, size_t typesize) {
  if (chunksize == 0) chunksize = B2_FRAME_DEFAULT_CHUNK;
  if (chunksize > BLOSC_MAX_BUFFERSIZE) chunksize = BLOSC_MAX_BUFFERSIZE;
  if (typesize > 1 && typesize <= BLOSC_MAX_TYPESIZE && chunksize >= typesize) chunksize -= chunksize % typesize;
  return chunksize;
}

size_t blosc_b200_frame_bound(size_t nbytes, size_t typesize, size_t chunksize) {
  size_t nchunks;
  chunksize = frame_chunksize(chunksize, typesize);
  nchunks = (nbytes + chunksize - 1) / chunksize;
  return B2_FRAME_HDR + nchunks * (8 + BLOSC_MAX_OVERHEAD) + nbytes;
}

long long blosc_b200_frame_compress(int clevel, int doshuffle, size_t typesize, size_t nbytes, const void* src,
                                    void* dest, size_t destsize, const char* compressor, size_t blocksize,
                                    size_t chunksize, int numinternalthreads) {
  b2_frame_job j;
  uint8_t* index;
  size_t nchunks, index_bytes;
  int i, rc, dest_dev;

  if (clevel < 0 || clevel > 9) return -10;                       /* same codes as the chunk API */
  if (doshuffle != 0 && doshuffle != 1 && doshuffle != 2) return -10;
  if (typesize == 0) return -10;
  if (blosc_compname_to_compcode(compressor) < 0) return -5;
  chunksize = frame_chunksize(chunksize, typesize);
  nchunks = (nbytes + chunksize - 1) / chunksize;
  if (nchunks > 0x7fffffff / 2) return -1;
  index_bytes = B2_FRAME_HDR + nchunks * 8;
  if (destsize < index_bytes) return 0;
  if (!backend_ready()) return -1;
  dest_dev = b2_ptr_is_device(dest);

  memset(&j, 0, sizeof j);
  j.nchunks = (int)nchunks; j.workers = frame_workers((int)nchunks); j.dest_dev = dest_dev;
  j.clevel = clevel; j.doshuffle = doshuffle; j.nthreads = numinternalthreads;
  j.typesize = typesize; j.blocksize = blocksize; j.chunksize = chunksize; j.nbytes = nbytes;
  j.destsize = destsize; j.cursor = index_bytes; j.compressor = compressor;
  j.src = (const uint8_t*)src; j.dest = (uint8_t*)dest;
  j.offsets = (uint64_t*)calloc(nchunks ? nchunks : 1, sizeof(uint64_t));
  index = (uint8_t*)malloc(index_bytes);
  if (!j.offsets || !index) { free(j.offsets); free(index); return -1; }
  rc = nchunks ? frame_run(&j, frame_compress_worker) : 0;
  if (rc == 0) {
    memcpy(index, "B2FR", 4); index[4] = 1; index[5] = index[6] = index[7] = 0;
    wr_u64(index + 8, (uint64_t)nbytes); wr_u64(index + 16, (uint64_t)j.cursor);
    wr_u32(index + 24, (uint32_t)chunksize); wr_u32(index + 28, (uint32_t)nchunks);
    for (i = 0; i < (int)nchunks; i++) wr_u64(index + B2_FRAME_HDR + 8 * (size_t)i, j.offsets[i]);
    rc = copy_some(dest, dest_dev, index, 0, index_bytes);
  }
  free(j.offsets); free(index);
  if (rc) return j.err ? j.err : (j.failed ? 0 : -1);            /* 0: does not fit in destsize, as blosc_compress */
  return (long long)j.cursor;
}

/* reads and validates the index; *offsets is malloc'ed (nchunks+1 entries, the last one = cbytes) */
static int frame_open(const void* frame, size_t framesize, size_t* nbytes, size_t* chunksize, size_t* nchunks,
                      uint64_t** offsets) {
  uint8_t hb[B2_FRAME_HDR];
  uint8_t* raw;
  uint64_t* off;
  uint64_t cbytes;
  size_t n, k;
  const int dev = b2_ptr_is_device(frame);
  int rc = -1;
  if (framesize < B2_FRAME_HDR || copy_some(hb, 0, frame, dev, B2_FRAME_HDR)) return -1;
  do {
    if (memcmp(hb, "B2FR", 4) != 0 || hb[4] != 1) break;
    *nbytes = (size_t)rd_u64(hb + 8); cbytes = rd_u64(hb + 16);
    *chunksize = rd_u32(hb + 24); n = rd_u32(hb + 28);
    if (cbytes > framesize || cbytes < B2_FRAME_HDR + 8 * (uint64_t)n) break;
    if (*nbytes > 0 && (*chunksize == 0 || *chunksize > BLOSC_MAX_BUFFERSIZE)) break;
    if (n != (*nbytes ? (*nbytes + *chunksize - 1) / *chunksize : 0)) break;
    raw = (uint8_t*)malloc(8 * n + 8);
    off = (uint64_t*)malloc(8 * (n + 1));
    if (!raw || !off) { free(raw); free(off); break; }
    if (copy_some(raw, 0, (const uint8_t*)frame + B2_FRAME_HDR, dev, 8 * n)) { free(raw); free(off); break; }
    for (k = 0; k < n; k++) off[k] = rd_u64(raw + 8 * k);
    off[n] = cbytes;
    free(raw);
    rc = 0;
    for (k = 0; k < n; k++)                /* chunks in order, at least a header each, inside the frame */
      if (off[k] < B2_FRAME_HDR + 8 * (uint64_t)n || off[k + 1] < off[k] + BLOSC_MAX_OVERHEAD || off[k + 1] > cbytes) rc = -1;
    if (rc) { free(off); break; }
    *nchunks = n; *offsets = off;
  } while (0);
  return rc;
}

int blosc_b200_frame_info(const void* frame, size_t framesize, size_t* nbytes, size_t* cbytes, size_t* chunksize,
                          size_t* nchunks) {
  size_t nb = 0, cs = 0, nc = 0;
  uint64_t* off = NULL;
  if (!backend_ready()) return -1;
  if (frame_open(frame, framesize, &nb, &cs, &nc, &off)) return -1;
  if (nbytes) *nbytes = nb;
  if (cbytes) *cbytes = (size_t)off[nc];
  if (chunksize) *chunksize = cs;
  if (nchunks) *nchunks = nc;
  free(off);
  return 0;
}

long long blosc_b200_frame_chunk(const void* frame, size_t framesize, size_t i, size_t* chunk_cbytes) {
  size_t nb = 0, cs = 0, nc = 0;
  uint64_t* off = NULL;
  long long r;
  if (!backend_ready()) return -1;
  if (frame_open(frame, framesize, &nb, &cs, &nc, &off)) return -1;
  if (i >= nc) { free(off); return -1; }
  if (chunk_cbytes) *chunk_cbytes = (size_t)(off[i + 1] - off[i]);
  r = (long long)off[i];
  free(off);
  return r;
}

long long blosc_b200_frame_decompress(const void* frame, size_t framesize, void* dest, size_t destsize,
                                      int numinternalthreads) {
  b2_frame_job j;
  size_t nb = 0, cs = 0, nc = 0;
  uint64_t* off = NULL;
  int rc;
  if (!backend_ready()) return -1;
  if (frame_open(frame, framesize, &nb, &cs, &nc, &off)) return -1;
  if (nb > destsize) { free(off); return -1; }
  memset(&j, 0, sizeof j);
  j.nchunks = (int)nc; j.workers = frame_workers((int)nc); j.nthreads = numinternalthreads;
  j.chunksize = cs; j.nbytes = nb; j.frame = (const uint8_t*)frame; j.dest = (uint8_t*)dest; j.offsets = off;
  rc = nc ? frame_run(&j, frame_decompress_worker) : 0;
  free(off);
  return rc ? -1 : (long long)nb;
}

/* One piece of a frame range: the part that falls in one chunk */
typedef struct { size_t chunk, order; int start, nitems; long long dst; } b2_piece;

static int cmp_piece(const void* a, const void* b) {
  const b2_piece *x = (const b2_piece*)a, *y = (const b2_piece*)b;
  if (x->chunk != y->chunk) return x->chunk < y->chunk ? -1 : 1;
  return x->order < y->order ? -1 : x->order > y->order;
}

/* Every range is checked against the frame's items before anything is read; then the ranges are cut at chunk
 * boundaries and each touched chunk, in ascending order, runs the chunk plan once, each piece landing at its own dest
 * offset. */
static long long frame_getitems_host(const void* frame, size_t framesize, size_t nranges, const size_t* starts,
                                     const size_t* nitems, void* dest) {
  size_t nb = 0, cs = 0, nc = 0, ts = 0, ipc, r, npieces = 0, i, j;
  uint64_t* off = NULL;
  uint8_t hb[16];
  b2_piece* pieces = NULL;
  long long result = -1, at = 0;
  if (frame_open(frame, framesize, &nb, &cs, &nc, &off)) return -1;
  do {
    if (nc == 0) {
      for (r = 0; r < nranges && nitems[r] == 0; r++) {}
      result = r == nranges ? 0 : -1;
      break;
    }
    if (copy_some(hb, 0, (const uint8_t*)frame + off[0], b2_ptr_is_device(frame), 16)) break;
    ts = hb[3];
    if (ts == 0 || cs % ts) break;
    ipc = cs / ts;                                     /* items per chunk */
    for (r = 0; r < nranges; r++) {
      if (starts[r] > nb / ts || nitems[r] > nb / ts - starts[r]) { fprintf(stderr, "`start`+`nitems` out of bounds"); break; }
      npieces += nitems[r] ? (starts[r] + nitems[r] - 1) / ipc - starts[r] / ipc + 1 : 0;
    }
    if (r < nranges) break;
    if (npieces == 0) { result = 0; break; }
    if (!(pieces = (b2_piece*)malloc(sizeof(b2_piece) * npieces))) break;
    for (r = 0, npieces = 0; r < nranges; r++) {
      size_t done = 0;
      while (done < nitems[r]) {
        const size_t c = (starts[r] + done) / ipc, first = (starts[r] + done) % ipc;
        const size_t take = nitems[r] - done < ipc - first ? nitems[r] - done : ipc - first;
        pieces[npieces].chunk = c; pieces[npieces].order = npieces;
        pieces[npieces].start = (int)first; pieces[npieces].nitems = (int)take;
        pieces[npieces].dst = at + (long long)(done * ts);
        npieces++;
        done += take;
      }
      at += (long long)(nitems[r] * ts);
    }
    qsort(pieces, npieces, sizeof *pieces, cmp_piece);
    result = 0;
    for (i = 0; i < npieces; i = j) {
      int* st;
      long long* dsts;
      long long want = 0, rc;
      size_t k;
      for (j = i; j < npieces && pieces[j].chunk == pieces[i].chunk; j++) want += (long long)pieces[j].nitems * (long long)ts;
      st = (int*)malloc(2 * sizeof(int) * (j - i));
      dsts = (long long*)malloc(sizeof(long long) * (j - i));
      if (!st || !dsts) { free(st); free(dsts); result = -1; break; }
      for (k = i; k < j; k++) { st[k - i] = pieces[k].start; st[j - i + k - i] = pieces[k].nitems; dsts[k - i] = pieces[k].dst; }
      rc = getitems_chunk((const uint8_t*)frame + off[pieces[i].chunk], (long long)(off[pieces[i].chunk + 1] - off[pieces[i].chunk]),
                          (int)(j - i), st, st + (j - i), dsts, dest);
      free(st); free(dsts);
      if (rc != want) { result = rc < 0 ? rc : -1; break; }
      result += rc;
    }
  } while (0);
  free(pieces); free(off);
  return result;
}

long long blosc_b200_frame_getitem(const void* frame, size_t framesize, size_t start, size_t nitems, void* dest) {
  if (!backend_ready()) return -1;
  return frame_getitems_host(frame, framesize, 1, &start, &nitems, dest);
}

/* Range lists in device memory are copied to the host (one copy each), and the frame is planned there */
long long blosc_b200_frame_getitems(const void* frame, size_t framesize, size_t nranges, const size_t* starts,
                                    const size_t* nitems, void* dest) {
  size_t* h = NULL;
  long long result = -1;
  int starts_dev, nitems_dev;
  if (nranges == 0) return 0;
  if (!backend_ready()) return -1;
  starts_dev = b2_ptr_is_device(starts); nitems_dev = b2_ptr_is_device(nitems);
  if (!starts_dev && !nitems_dev) return frame_getitems_host(frame, framesize, nranges, starts, nitems, dest);
  if (nranges > ((size_t)-1) / (2 * sizeof(size_t)) || !(h = (size_t*)malloc(2 * sizeof(size_t) * nranges))) return -1;
  if (!copy_some(h, 0, starts, starts_dev, sizeof(size_t) * nranges) &&
      !copy_some(h + nranges, 0, nitems, nitems_dev, sizeof(size_t) * nranges))
    result = frame_getitems_host(frame, framesize, nranges, h, h + nranges, dest);
  free(h);
  return result;
}

/* ------------------------------------------------------------------------- */
/* global-state front end                                                     */
/* ------------------------------------------------------------------------- */
void blosc_init(void) { g_initlib = 1; }                                    /* blosc.c:2223-2247 (no pool to create) */
void blosc_destroy(void) { if (g_initlib) { g_initlib = 0; blosc_free_resources(); } }   /* blosc.c:2249-2260 */
int blosc_get_nthreads(void) { return g_threads; }
int blosc_set_nthreads(int n) { int old = g_threads; if (!g_initlib) blosc_init(); g_threads = n; return old; }   /* blosc.c:1958-1975 */
const char* blosc_get_compressor(void) { const char* n; blosc_compcode_to_compname(g_compressor, &n); return n; }
int blosc_set_compressor(const char* compname) {                            /* blosc.c:2013-2023 */
  int code = blosc_compname_to_compcode(compname);
  g_compressor = code;
  if (!g_initlib) blosc_init();
  return code;
}
int blosc_get_blocksize(void) { return g_force_blocksize; }
void blosc_set_blocksize(size_t size) { g_force_blocksize = (int32_t)size; }
void blosc_set_splitmode(int mode) { g_splitmode = mode; }

int blosc_compress(int clevel, int doshuffle, size_t typesize, size_t nbytes, const void* src, void* dest,
                   size_t destsize) {                                      /* blosc.c:1311-1433 */
  const char* envvar;
  const char* compname;
  int result, nolock;
  if (!g_initlib) blosc_init();
  if ((envvar = getenv("BLOSC_CLEVEL")) != NULL) { long v = strtol(envvar, NULL, 10); if (v != EINVAL && v >= 0) clevel = (int)v; }
  if ((envvar = getenv("BLOSC_SHUFFLE")) != NULL) {
    if (strcmp(envvar, "NOSHUFFLE") == 0) doshuffle = BLOSC_NOSHUFFLE;
    if (strcmp(envvar, "SHUFFLE") == 0) doshuffle = BLOSC_SHUFFLE;
    if (strcmp(envvar, "BITSHUFFLE") == 0) doshuffle = BLOSC_BITSHUFFLE;
  }
  if ((envvar = getenv("BLOSC_TYPESIZE")) != NULL) { long v = strtol(envvar, NULL, 10); if (v != EINVAL && v > 0) typesize = (size_t)(int)v; }
  if ((envvar = getenv("BLOSC_COMPRESSOR")) != NULL) { result = blosc_set_compressor(envvar); if (result < 0) return result; }
  if ((envvar = getenv("BLOSC_BLOCKSIZE")) != NULL) { long v = strtol(envvar, NULL, 10); if (v != EINVAL && v > 0) blosc_set_blocksize((size_t)v); }
  if ((envvar = getenv("BLOSC_NTHREADS")) != NULL) { long v = strtol(envvar, NULL, 10); if (v != EINVAL && v > 0) { result = blosc_set_nthreads((int)v); if (result < 0) return result; } }
  if ((envvar = getenv("BLOSC_SPLITMODE")) != NULL) {
    if (strcmp(envvar, "FORWARD_COMPAT") == 0) blosc_set_splitmode(BLOSC_FORWARD_COMPAT_SPLIT);
    else if (strcmp(envvar, "AUTO") == 0) blosc_set_splitmode(BLOSC_AUTO_SPLIT);
    else if (strcmp(envvar, "ALWAYS") == 0) blosc_set_splitmode(BLOSC_ALWAYS_SPLIT);
    else if (strcmp(envvar, "NEVER") == 0) blosc_set_splitmode(BLOSC_NEVER_SPLIT);
    else { fprintf(stderr, "BLOSC_SPLITMODE environment variable '%s' not recognized\n", envvar); return -1; }
  }
  nolock = getenv("BLOSC_NOLOCK") != NULL;
  blosc_compcode_to_compname(g_compressor, &compname);
  if (compname == NULL) compname = "(null)";
  /* the global path serialises callers on one mutex (blosc.c:1410); BLOSC_NOLOCK skips it (:1400-1408) */
  if (!nolock) pthread_mutex_lock(&g_global_mutex);
  result = blosc_compress_ctx(clevel, doshuffle, typesize, nbytes, src, dest, destsize, compname,
                              (size_t)g_force_blocksize, g_threads);
  if (!nolock) pthread_mutex_unlock(&g_global_mutex);
  return result;
}

int blosc_decompress(const void* src, void* dest, size_t destsize) {        /* blosc.c:1537-1572 */
  const char* envvar;
  int result, nolock;
  if (!g_initlib) blosc_init();
  if ((envvar = getenv("BLOSC_NTHREADS")) != NULL) { long v = strtol(envvar, NULL, 10); if (v != EINVAL && v > 0) { result = blosc_set_nthreads((int)v); if (result < 0) return result; } }
  nolock = getenv("BLOSC_NOLOCK") != NULL;
  if (!nolock) pthread_mutex_lock(&g_global_mutex);
  result = blosc_decompress_ctx(src, dest, destsize, g_threads);
  if (!nolock) pthread_mutex_unlock(&g_global_mutex);
  return result;
}

/* ------------------------------------------------------------------------- */
/* blosc_b200 extensions                                                     */
/* ------------------------------------------------------------------------- */
int blosc_b200_filter(int mode, size_t typesize, size_t blocksize, const void* src, void* dest) {
  b2_ws* w;
  FilterArgs fa;
  int src_dev, dest_dev, rc = -1;
  if (mode < 0 || mode > 3 || typesize == 0 || blocksize > (size_t)INT_MAX) return -1;
  if (blocksize == 0) return 0;
  src_dev = b2_ptr_is_device(src); dest_dev = b2_ptr_is_device(dest);
  w = ws_acquire();
  if (!w) return -1;
  do {
    const uint8_t* d_src = (const uint8_t*)src;
    uint8_t* d_dst = (uint8_t*)dest;
    if (!src_dev) {
      if (buf_ensure(&w->in, blocksize + 64)) break;
      if (b2_copy_h2d(w->in.p, src, blocksize, w->stream)) break;
      d_src = (const uint8_t*)w->in.p;
    }
    if (!dest_dev) { if (buf_ensure(&w->out, blocksize + 64)) break; d_dst = (uint8_t*)w->out.p; }
    fa.src = d_src; fa.dst = d_dst; fa.nbytes = (long long)blocksize; fa.blocksize = (int)blocksize;
    fa.typesize = (int)typesize; fa.mode = mode;
    if (b2_launch_filter(&fa, w->stream)) break;
    if (!dest_dev && b2_copy_d2h(dest, d_dst, blocksize, w->stream)) break;
    if (b2_stream_sync(w->stream)) break;
    rc = 0;
  } while (0);
  ws_release(w);
  return rc;
}

int blosc_b200_set_device(int dev) { return backend_ready() ? b2_set_device(dev) : -1; }
void blosc_b200_set_profiling(int on) { b2_prof_enable(on); }
void blosc_b200_prof_reset(void) { b2_prof_reset(); }
int blosc_b200_prof_get(int kind, double* ms_total, long long* launches) { return b2_prof_get(kind, ms_total, launches); }
long long blosc_b200_launch_count(void) { return b2_launch_count(); }

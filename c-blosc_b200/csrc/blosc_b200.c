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
#include <limits.h>
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
  b2_buf fplan, fpieces, fstage;   /* frame getitems planned on the GPU: its scratch, the piece lists and a host dest's
                                    * staging, live while the chunk plan uses the buffers above */
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

/* the device scratch of a slot; its stream, result words and bounce slices stay */
static void ws_free_bufs(b2_ws* w) {
  buf_free(&w->in); buf_free(&w->filt); buf_free(&w->slots); buf_free(&w->out);
  buf_free(&w->csizes); buf_free(&w->needs); buf_free(&w->bstarts);
  buf_free(&w->prev); buf_free(&w->segs); buf_free(&w->ptail); buf_free(&w->plan);
  buf_free(&w->fplan); buf_free(&w->fpieces); buf_free(&w->fstage);
}

/* Everything a slot owns; the caller holds the slot (in_use) and the slot's device need not be current
 * (device and page-locked allocations are freed by address) */
static void ws_teardown(b2_ws* w) {
  int k;
  ws_free_bufs(w);
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
 * device is rebuilt for the caller's device when no matching or unused slot is left.  wait 0: NULL at once instead of
 * waiting (a helper thread of a call that already holds a slot, which must not wait for the slot it holds). */
static b2_ws* ws_acquire_if(int wait) {
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
    if (!wait) break;
    pthread_cond_wait(&g_ws_cv, &g_ws_mutex);
  }
  pthread_mutex_unlock(&g_ws_mutex);
  if (!w) return NULL;
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

static b2_ws* ws_acquire(void) { return ws_acquire_if(1); }

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
    ws_free_bufs(w);
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

/* Where a read writes n bytes: dest itself when it is device memory, else `stage`, which the caller copies to dest once
 * at the end (d2h_any), so that a failed read leaves dest untouched.  NULL when the staging buffer cannot be had. */
static uint8_t* stage_dest(b2_buf* stage, void* dest, int dest_dev, size_t n) {
  if (dest_dev) return (uint8_t*)dest;
  return buf_ensure(stage, n + 64) ? NULL : (uint8_t*)stage->p;
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

/* header + raw payload from device memory, inside a held workspace (no second one is taken) */
static int emit_memcpyed_ws(b2_ws* w, const uint8_t* hdr, const void* d_src, void* dest, int dest_dev, int32_t nbytes) {
  if (copy_any(dest, dest_dev, hdr, 0, 16, w->stream)) return -1;
  if (dest_dev ? copy_any((uint8_t*)dest + 16, 1, d_src, 1, (size_t)nbytes, w->stream)
               : d2h_any(w, (uint8_t*)dest + 16, d_src, (size_t)nbytes))
    return -1;
  return nbytes + 16;
}

/* A chunk of a grid being written (blosc_b200_grid_compress) whose input compress_impl packs out of a device array into
 * its own workspace: `pack` (dst and diff unset) and, for an edge chunk, `pad` (total > 0; dst unset), the fill over the
 * whole chunk that goes first.  skip: the pack compares with the fill pattern, and a chunk that holds nothing else is
 * `skipped`, with nothing written. */
typedef struct {
  GridPackArgs pack;
  PlacedGatherArgs pad;
  int skip, skipped;
} b2_pack;

/* The chunk's input made in w->in (room for it ensured) on w's stream; with skip, one read-back and sync of the
 * compare flag */
static int grid_pack(b2_ws* w, b2_pack* pk) {
  pk->pack.dst = (uint8_t*)w->in.p;
  pk->pack.diff = pk->skip ? w->d_result + B2_R_DIFF : NULL;
  if (pk->pad.total > 0) {
    pk->pad.dst = (uint8_t*)w->in.p;
    if (b2_launch_placed_fill(&pk->pad, w->stream)) return -1;
  }
  if (pk->skip && b2_memset_dev(pk->pack.diff, 0, 4, w->stream)) return -1;
  if (b2_launch_grid_pack(&pk->pack, w->stream)) return -1;
  if (pk->skip) {
    if (b2_copy_d2h(w->h_result + B2_R_DIFF, pk->pack.diff, 4, w->stream) || b2_stream_sync(w->stream)) return -1;
    pk->skipped = !w->h_result[B2_R_DIFF];
  }
  return 0;
}

/* ------------------------------------------------------------------------- */
/* compression                                                                */
/* ------------------------------------------------------------------------- */
/* pk NULL: the input is `src`.  Otherwise the input is packed into the workspace (grid_pack) and src is unused; every
 * exit, the MEMCPYED ones included, is then served from the packed bytes while the workspace is held. */
static int compress_impl(int clevel, int doshuffle, size_t typesize, size_t nbytes, const void* src, void* dest,
                         size_t destsize, const char* compressor, size_t blocksize, int numinternalthreads,
                         b2_place* pl, int pl_dest_dev, b2_pack* pk) {
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

  src_dev = pk ? 1 : (nb > 0) ? b2_ptr_is_device(src) : 0;
  dest_dev = pl ? pl_dest_dev : b2_ptr_is_device(dest);

  /* blosc_compress_context, blosc.c:1250-1279 */
  if ((flags & BLOSC_MEMCPYED) && nb + BLOSC_MAX_OVERHEAD > dsz) return 0;
  if (check_threads(numinternalthreads, nb, bs) < 0) return -1;
  if ((flags & BLOSC_MEMCPYED) && !pk) {
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
    if (pk) {                                  /* the input packed in place of the staging copy below */
      launched = 1;
      if (buf_ensure(&w->in, (size_t)nb + 64) || grid_pack(w, pk)) break;
      src = w->in.p;
      if (pk->skipped) { result = 0; break; }
      if (flags & BLOSC_MEMCPYED) { result = -2; break; }
    }
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
        if (recs == &w->in && pk) recs = &w->plan;         /* w->in holds the packed input the redo below reads */
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
  if (result == -2 && pk) {                  /* MEMCPYED, from the packed bytes before another call may reuse w->in */
    flags |= BLOSC_MEMCPYED;
    make_header(hdr, 1, flags, ts, nb, bs, nb + 16);
    result = pl && !(dest = frame_place(pl, nb + 16)) ? 0 : emit_memcpyed_ws(w, hdr, w->in.p, dest, dest_dev, nb);
  }
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
                       numinternalthreads, NULL, 0, NULL);
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

/* Wait for the launches so far and read their decode verdict: 0, blosc_d's negative code, or -1 when the copy or the
 * sync fails (the counters are reset then).  status NULL: nothing was decoded, and the word, possibly stale, is not
 * looked at. */
static int read_verdict(b2_ws* w, const int* status) {
  if (b2_copy_d2h(w->h_result + B2_R_STATUS_OUT, w->d_result + B2_R_STATUS_OUT, 4, w->stream) || b2_stream_sync(w->stream)) {
    ws_reset_counters(w);
    return -1;
  }
  return status && w->h_result[B2_R_STATUS_OUT] < 0 ? w->h_result[B2_R_STATUS_OUT] : 0;
}

/* Decode blocks [first, first+count) of a chunk that is already on the device into `d_out`
 * (device), which represents buffer offsets [first*blocksize, ...).  Shared by decompress and a one-range read. */
static int decode_blocks(b2_ws* w, const b2_hdr* h, int codec, const uint8_t* d_chunk, int first, int count,
                         uint8_t* d_out) {
  const int has_left = h->leftover > 0 && first + count == h->nblocks;
  if (launch_decode_blocks(w, h, codec, d_chunk, first, count, NULL, has_left, d_out)) return -1;
  return read_verdict(w, w->d_result + B2_R_STATUS_OUT);
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

/* the chunk-header checks of blosc_getitem (blosc.c:1574-1631), with its return codes; 0 when the chunk is readable.
 * A caller that holds a workspace passes it for the header's copy (NULL: one is taken when src is device memory). */
static int getitem_header(b2_ws* w, const void* src, int src_dev, long long max_cbytes, b2_hdr* h, int* codec) {
  uint8_t hb[16];
  int rc;
  if (w ? copy_any(hb, 0, src, src_dev, 16, w->stream) : copy_some(hb, 0, src, src_dev, 16)) return -1;
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

/* The gather's source for the touched blocks of a checked chunk, listed in ascending order in w->bstarts (has_left: the
 * last is the short last block).  A memcpyed device chunk is read in place; a host chunk has the list read back and its
 * listed blocks staged; a compressed chunk's are then decoded into the compact scratch w->out, and *status is the
 * verdict the gather must check (else NULL). */
static int touched_source(b2_ws* w, const void* src, int src_dev, const b2_hdr* h, int codec, int count, int has_left,
                          const uint8_t** d_src, const int** status) {
  const int memcpyed = (h->flags & BLOSC_MEMCPYED) != 0;
  const uint8_t* d_chunk = (const uint8_t*)src;
  int* hblocks = NULL;
  int rc = -1;
  *status = NULL;
  if (memcpyed && src_dev) { *d_src = d_chunk + 16; return 0; }
  do {
    if (!src_dev) {
      if (!(hblocks = (int*)malloc(4 * (size_t)count))) break;
      if (d2h_any(w, hblocks, w->bstarts.p, 4 * (size_t)count)) break;
      if (memcpyed ? stage_memcpyed_blocks(w, h, (const uint8_t*)src, hblocks, count)
                   : stage_blocks(w, h, (const uint8_t*)src, hblocks, count))
        break;
      d_chunk = (const uint8_t*)w->in.p;
    }
    if (memcpyed) *d_src = d_chunk;
    else {
      if (buf_ensure(&w->out, (size_t)count * (size_t)h->blocksize + 64)) break;
      if (launch_decode_blocks(w, h, codec, d_chunk, 0, count, (const int*)w->bstarts.p, has_left, (uint8_t*)w->out.p))
        break;
      *d_src = (const uint8_t*)w->out.p;
      *status = w->d_result + B2_R_STATUS_OUT;
    }
    rc = 0;
  } while (0);
  free(hblocks);
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

/* The execution tail of getitems, shared by its host plan and its GPU plan: the gather of `nr` ranges from d_src
 * (status: the verdict it checks, or NULL; see touched_source), the verdict, and a host dest's copy out.  On entry the
 * gather table (nr + 1 entries; dst = pos when dest is host memory) is in w->segs, and w->slots has room for `total`
 * bytes when dest is host memory.  A host dest then receives the ranges from w->slots: all of them at dest + at_b[0]
 * when tab is NULL, else range r at dest + at_b[r] (tab: the table on the host).  Returns total, or blosc_d's code when
 * a stream fails to decode (dest is then untouched). */
static long long getitems_run(b2_ws* w, const uint8_t* d_src, const int* status, int nr, long long total, void* dest,
                              int dest_dev, const GatherRange* tab, const long long* at_b) {
  GatherArgs ga;
  long long result = -1;
  uint8_t* tmp = NULL;
  int r, rc;
  memset(&ga, 0, sizeof ga);
  do {
    ga.src = d_src; ga.dst = dest_dev ? (uint8_t*)dest : (uint8_t*)w->slots.p; ga.ranges = (const GatherRange*)w->segs.p;
    ga.nranges = nr; ga.total = total; ga.status = status;
    if (b2_launch_gather(&ga, w->stream)) { ws_reset_counters(w); break; }
    if ((rc = read_verdict(w, status)) < 0) { result = rc; break; }
    if (!dest_dev) {
      if (!tab) {
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
  rc = getitem_header(NULL, src, src_dev, max_cbytes, &h, &codec);
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
    const int* status = NULL;
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
      const uint8_t* d_chunk = (const uint8_t*)src;
      int nv, k, count = 0;
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
      /* a host chunk is staged before the uploads below: after them, 4096 ranges of a pinned host chunk read 15 % slower
       * on an H100 (700 W) */
      if (!src_dev) {
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
      if (touched_source(w, d_chunk, 1, &h, codec, count, h.leftover > 0 && blocks[count - 1] == h.nblocks - 1, &d_src,
                         &status))
        break;
    }
    result = getitems_run(w, d_src, status, nr, total, dest, dest_dev, contiguous ? NULL : tab, at_b);
  } while (0);
  ws_release(w);
  free(tab); free(lo_b); free(iv); free(blocks); free(tmp);
  return result;
}

int blosc_getitem(const void* src, int start, int nitems, void* dest) {                 /* blosc.c:1574-1703 */
  return (int)getitems_chunk(src, -1, 1, &start, &nitems, NULL, dest);
}

#define B2_R_PLAN 8   /* h_result words 8..15 receive a GPU plan's record (GetitemsPlan, FramePlan) */
#define B2_AL(x) (((x) + 15) & ~(size_t)15)

/* Wait for a GPU plan and read the first n bytes of its record, at d_rec, into *rec */
static int read_plan(b2_ws* w, const void* d_rec, void* rec, size_t n) {
  if (b2_copy_d2h(w->h_result + B2_R_PLAN, d_rec, n, w->stream) || b2_stream_sync(w->stream)) return -1;
  memcpy(rec, w->h_result + B2_R_PLAN, n);
  return 0;
}

/* The tile state of one scan of `tiles` tiles: its ticket and flags (both zeroed by the caller), then the tiles'
 * aggregates and inclusive prefixes of `width` bytes each, back to back from `vals` */
static PlanScan plan_scan(uint8_t* ticket, uint8_t* flags, uint8_t* vals, size_t width, size_t tiles) {
  PlanScan s;
  s.ticket = (unsigned*)ticket; s.flag = (unsigned*)flags; s.agg = vals; s.inc = vals + width * tiles;
  return s;
}

/* The scratch of a chunk's GPU plan in w->plan, for n ranges (0: a box), and the fields of *pa that describe the chunk
 * or point into it: the record, the tickets, the tile flags and the difference array, all zeroed; then the tiles'
 * values, the range lengths and the block slots; the block list in w->bstarts unless in_place.  Returns the room for
 * one uploaded host list of n ints, or NULL. */
static uint8_t* plan_scratch(b2_ws* w, const b2_hdr* h, int n, int in_place, PlanArgs* pa) {
  const size_t tb = ((size_t)h->nblocks + PLAN_TILE - 1) / PLAN_TILE, tr = ((size_t)n + PLAN_TILE - 1) / PLAN_TILE;
  const size_t o_tk = 32, o_flag = 64, o_cover = B2_AL(o_flag + 4 * (2 * tb + tr));
  const size_t zeroed = B2_AL(o_cover + 4 * ((size_t)h->nblocks + 1));
  const size_t o_vals = zeroed, o_len = B2_AL(o_vals + 4 * 4 * tb + 8 * 2 * tr);
  const size_t o_slot = B2_AL(o_len + 8 * (size_t)n), o_up = B2_AL(o_slot + 4 * (size_t)h->nblocks);
  uint8_t* base;
  if (buf_ensure(&w->plan, o_up + 4 * (size_t)n)) return NULL;
  if (!in_place && buf_ensure(&w->bstarts, 4 * (size_t)h->nblocks + 64)) return NULL;
  base = (uint8_t*)w->plan.p;
  if (b2_memset_dev(base, 0, zeroed, w->stream)) return NULL;
  memset(pa, 0, sizeof *pa);
  pa->typesize = h->typesize; pa->blocksize = h->blocksize; pa->nblocks = h->nblocks;
  pa->leftover = h->leftover > 0; pa->nbytes = h->nbytes; pa->in_place = in_place;
  pa->len = (long long*)(base + o_len); pa->cover = (int*)(base + o_cover); pa->slot = (int*)(base + o_slot);
  pa->blocks = (int*)w->bstarts.p; pa->rec = (GetitemsPlan*)base;
  pa->scan[PLAN_COVER] = plan_scan(base + o_tk, base + o_flag, base + o_vals, 4, tb);
  pa->scan[PLAN_SLOT] = plan_scan(base + o_tk + 4, base + o_flag + 4 * tb, base + o_vals + 8 * tb, 4, tb);
  pa->scan[PLAN_POS] = plan_scan(base + o_tk + 8, base + o_flag + 8 * tb, base + o_vals + 16 * tb, 8, tr);
  return base + o_up;
}

/* A range list as a GPU plan reads it: the list itself when it is in device memory, else its copy in `room` (NULL when
 * the upload fails).  At most one of a call's two lists is in host memory, so one room serves both. */
static const void* dev_list(b2_ws* w, const void* list, int list_dev, size_t bytes, void* room) {
  if (list_dev) return list;
  return h2d_any(w, room, list, bytes) ? NULL : room;
}

/* The GPU plan (dev_chunk.cuh plan_*_kernel), for range lists of which at least one is in device memory (a host one is
 * uploaded), on the caller's workspace.  It builds the gather table in w->segs and the touched-block list in
 * w->bstarts, both as the host plan would (the table keeps empty ranges, which copy nothing), and the host reads back
 * one small record.  A failing range is reported by getitem_range on that range alone, so the code and the message
 * are the host plan's.  dsts NULL: the ranges land back to back in dest; else range r lands at dest + dsts[r] (device
 * lists, device dest: frame pieces). */
static long long getitems_gpu(b2_ws* w, const void* src, int src_dev, const b2_hdr* h, int codec, int n,
                              const int* starts, int starts_dev, const int* nitems, int nitems_dev,
                              const long long* dsts, void* dest, int dest_dev) {
  const long long at0 = 0;
  PlanArgs pa;
  GetitemsPlan rec;
  const uint8_t* d_src;
  const int* status;
  uint8_t* up = plan_scratch(w, h, n, (h->flags & BLOSC_MEMCPYED) && src_dev, &pa);
  if (!up || buf_ensure(&w->segs, sizeof(GatherRange) * ((size_t)n + 1) + 64)) return -1;
  if (!(pa.starts = (const int*)dev_list(w, starts, starts_dev, 4 * (size_t)n, up)) ||
      !(pa.nitems = (const int*)dev_list(w, nitems, nitems_dev, 4 * (size_t)n, up)))
    return -1;
  if (b2_memset_dev(pa.rec, 0xff, 4, w->stream)) return -1;
  pa.nranges = n; pa.ranges = (GatherRange*)w->segs.p; pa.dsts = dsts;
  if (b2_launch_plan(&pa, w->stream) || read_plan(w, pa.rec, &rec, sizeof rec)) return -1;
  if (rec.bad != 0xffffffffu) {                                            /* blosc_getitem's verdict on that range */
    int s, c;
    long long lo, hi;
    if (!copy_any(&s, 0, starts + rec.bad, starts_dev, 4, w->stream) &&
        !copy_any(&c, 0, nitems + rec.bad, nitems_dev, 4, w->stream))
      getitem_range(h, s, c, &lo, &hi);
    return -1;
  }
  if (rec.total == 0) return 0;
  if (!dest_dev && buf_ensure(&w->slots, (size_t)rec.total + 64)) return -1;
  if (touched_source(w, src, src_dev, h, codec, rec.nlisted, rec.has_left, &d_src, &status)) return -1;
  return getitems_run(w, d_src, status, n, rec.total, dest, dest_dev, NULL, &at0);
}

long long blosc_b200_getitems(const void* src, int nranges, const int* starts, const int* nitems, void* dest) {
  b2_hdr h;
  b2_ws* w;
  long long result;
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
  rc = getitem_header(NULL, src, src_dev, -1, &h, &codec);
  if (rc) return rc;
  if (!(w = ws_acquire())) return -1;
  result = getitems_gpu(w, src, src_dev, &h, codec, nranges, starts, starts_dev, nitems, nitems_dev, NULL, dest,
                        b2_ptr_is_device(dest));
  ws_release(w);
  return result;
}

/* ------------------------------------------------------------------------- */
/* boxes of an N-d array (blosc_b200_getslice, blosc_b200_frame_getslice)     */
/* ------------------------------------------------------------------------- */
/* A box needs no list of its runs: the blocks it touches and the source of every output byte follow from the box
 * itself (B2Box, b2_args.h).  A chunk's part of a box is planned by box_touch_kernel and the PLAN_SLOT scan, its
 * touched blocks are decoded and unfiltered into the compact scratch as getitems decodes them, and box_gather_kernel
 * writes it: a fixed number of launches, one record read-back and one status sync, whatever the number of runs. */

/* The checks that need no chunk: ndim, the shape and its product (*nitems), the box inside the shape.  -1 with a
 * message when one fails. */
static int box_geometry(int ndim, const int64_t* shape, const int64_t* start, const int64_t* stop, long long* nitems) {
  long long prod = 1;
  int k, zero = 0;
  if (ndim < 1 || ndim > B2_BOX_MAXDIM) {
    fprintf(stderr, "blosc_b200: ndim %d is not in 1..%d\n", ndim, B2_BOX_MAXDIM);
    return -1;
  }
  for (k = 0; k < ndim; k++) {
    if (shape[k] < 0) { fprintf(stderr, "blosc_b200: shape[%d] = %lld is negative\n", k, (long long)shape[k]); return -1; }
    zero |= shape[k] == 0;
  }
  for (k = 0; k < ndim && !zero; k++) {
    if (prod > LLONG_MAX / shape[k]) { fprintf(stderr, "blosc_b200: the product of the shape overflows int64\n"); return -1; }
    prod *= shape[k];
  }
  for (k = 0; k < ndim; k++)
    if (start[k] < 0 || start[k] > stop[k] || stop[k] > shape[k]) {
      fprintf(stderr, "blosc_b200: box [%lld, %lld) of dimension %d is not inside [0, %lld)\n", (long long)start[k],
              (long long)stop[k], k, (long long)shape[k]);
      return -1;
    }
  *nitems = zero ? 0 : prod;
  return 0;
}

/* the array's items times the typesize against the bytes that hold it; -1 with a message when they differ */
static int box_nbytes(long long nitems, long long typesize, unsigned long long nbytes) {
  if (nbytes % (unsigned long long)typesize || nbytes / (unsigned long long)typesize != (unsigned long long)nitems) {
    fprintf(stderr, "blosc_b200: %lld items of %lld bytes are not the %llu bytes of the data\n", nitems, typesize, nbytes);
    return -1;
  }
  return 0;
}

static int box_empty(int ndim, const int64_t* start, const int64_t* stop) {
  int k;
  for (k = 0; k < ndim; k++) if (start[k] == stop[k]) return 1;
  return 0;
}

/* Every step >= 1 (step == NULL: all ones); -1 with a message naming the first dimension whose step is not */
static int box_steps(int ndim, const int64_t* step) {
  int k;
  for (k = 0; step && k < ndim; k++)
    if (step[k] < 1) {
      fprintf(stderr, "blosc_b200: step[%d] = %lld is not >= 1\n", k, (long long)step[k]);
      return -1;
    }
  return 0;
}

/* The canonical box of a non-empty, checked one with steps (NULL: all ones), normalised in this order: each stop
 * becomes the last selected coordinate + 1; a dimension that selects one coordinate gets step 1; every dimension that
 * the box covers whole with step 1 is merged into the one before it when that one's step is 1 too (merged into a
 * stepped dimension, the selection would not be an arithmetic progression), so the innermost run is as long as it can
 * be.  The innermost run is the last extent, or 1 item when the last step is > 1.  A box whose steps are all 1 is
 * then exactly the step-less box, and `stepped` is 0. */
static void box_build(int ndim, const int64_t* shape, const int64_t* start, const int64_t* stop, const int64_t* step,
                      long long nitems, B2Box* b) {
  long long sh[B2_BOX_MAXDIM];
  int k, n = 0;
  memset(b, 0, sizeof *b);
  for (k = 0; k < ndim; k++) {
    const long long t = step ? step[k] : 1, e = (stop[k] - start[k] - 1) / t + 1;   /* e >= 1: no overflow */
    const long long last = start[k] + (e - 1) * t, u = e == 1 ? 1 : t;
    if (n > 0 && u == 1 && b->step[n - 1] == 1 && start[k] == 0 && last + 1 == shape[k]) {
      sh[n - 1] *= shape[k]; b->start[n - 1] *= shape[k]; b->stop[n - 1] *= shape[k];
    } else {
      sh[n] = shape[k]; b->start[n] = start[k]; b->stop[n] = last + 1; b->step[n] = u;
      b->stepped |= u > 1;
      n++;
    }
  }
  b->ndim = n;
  for (k = 0; k < n; k++) b->ext[k] = (b->stop[k] - b->start[k] - 1) / b->step[k] + 1;
  b->stride[n - 1] = 1; b->inner[n - 1] = 1;
  for (k = n - 2; k >= 0; k--) {
    b->stride[k] = b->stride[k + 1] * sh[k + 1];
    b->inner[k] = b->inner[k + 1] * b->ext[k + 1];
  }
  b->run = b->step[n - 1] == 1 ? b->ext[n - 1] : 1;
  b->count = b->inner[0] * b->ext[0];
  b->nitems = nitems;
}

/* One chunk's part of a box: the chunk (header h, checked) holds the array's flat items [window, window + nbytes /
 * typesize); the box items among them land, in C order, at d_dst (device memory).  Returns the bytes written, blosc_d's
 * code when a touched block fails to decode (nothing is written then), or -1. */
static long long getslice_chunk(b2_ws* w, const void* src, int src_dev, const b2_hdr* h, int codec, const B2Box* box,
                                long long window, uint8_t* d_dst) {
  const long long ts = h->typesize, p0 = b2_box_rank(box, window, box->stepped);
  const long long total = (b2_box_rank(box, window + h->nbytes / ts, box->stepped) - p0) * ts;
  GetitemsPlan rec = {0};
  BoxGatherArgs ga;
  int rc;
  if (total == 0) return 0;
  memset(&ga, 0, sizeof ga);
  ga.box = *box; ga.window = window; ga.p0 = p0; ga.total = total;
  ga.typesize = h->typesize; ga.blocksize = h->blocksize; ga.dst = d_dst;
  if (!((h->flags & BLOSC_MEMCPYED) && src_dev)) {            /* a memcpyed device chunk is read in place: no plan */
    BoxPlanArgs bp;
    bp.box = *box; bp.window = window;
    if (!plan_scratch(w, h, 0, 0, &bp.plan) || b2_launch_box_plan(&bp, w->stream) ||
        read_plan(w, bp.plan.rec, &rec, sizeof rec))
      return -1;
    ga.slot = bp.plan.slot;
  }
  if (touched_source(w, src, src_dev, h, codec, rec.nlisted, rec.has_left, &ga.src, &ga.status)) return -1;
  if (b2_launch_box_gather(&ga, w->stream)) { ws_reset_counters(w); return -1; }
  rc = read_verdict(w, ga.status);
  return rc < 0 ? rc : total;
}

long long blosc_b200_getslice_step(const void* src, int ndim, const int64_t* shape, const int64_t* start,
                                   const int64_t* stop, const int64_t* step, void* dest) {
  b2_hdr h;
  B2Box box;
  b2_ws* w;
  uint8_t* d_dst;
  long long nitems = 0, result = -1;
  int src_dev, dest_dev, codec = 0, rc;
  if (box_geometry(ndim, shape, start, stop, &nitems) || box_steps(ndim, step)) return -1;
  src_dev = b2_ptr_is_device(src);
  rc = getitem_header(NULL, src, src_dev, -1, &h, &codec);
  if (rc) return rc;
  if (box_nbytes(nitems, h.typesize, (unsigned long long)h.nbytes)) return -1;
  if (box_empty(ndim, start, stop)) return 0;
  box_build(ndim, shape, start, stop, step, nitems, &box);
  dest_dev = b2_ptr_is_device(dest);
  if (!(w = ws_acquire())) return -1;
  if ((d_dst = stage_dest(&w->slots, dest, dest_dev, (size_t)(box.count * h.typesize)))) {
    result = getslice_chunk(w, src, src_dev, &h, codec, &box, 0, d_dst);
    if (result > 0 && !dest_dev && d2h_any(w, dest, d_dst, (size_t)result)) result = -1;
  }
  ws_release(w);
  return result;
}

long long blosc_b200_getslice(const void* src, int ndim, const int64_t* shape, const int64_t* start,
                              const int64_t* stop, void* dest) {
  return blosc_b200_getslice_step(src, ndim, shape, start, stop, NULL, dest);
}

/* The checks of getslices that need no data: box_geometry on the box [0, extent), the count of boxes, and corners in
 * device memory on the device the call runs on (that of data or dest when either is device memory, as for getitems).
 * -1 with a message when one fails. */
static const int64_t g_box_origin[B2_BOX_MAXDIM] = {0};

static int boxes_geometry(int ndim, const int64_t* shape, const int64_t* extent, long long nboxes, const void* data,
                          const void* dest, const int64_t* starts, long long* nitems) {
  int dev;
  if (box_geometry(ndim, shape, g_box_origin, extent, nitems)) return -1;
  if (nboxes < 0) { fprintf(stderr, "blosc_b200: nboxes = %lld is negative\n", nboxes); return -1; }
  if (nboxes == 0 || !b2_ptr_is_device(starts)) return 0;
  dev = b2_ptr_is_device(data) ? b2_ptr_device(data) : b2_ptr_is_device(dest) ? b2_ptr_device(dest) : b2_get_device();
  if (b2_ptr_device(starts) != dev) {
    fprintf(stderr, "blosc_b200: starts are not on device %d, where the call runs\n", dev);
    return -1;
  }
  return 0;
}

/* The sizes of a batch of nboxes boxes of `count` items: -1 with a message when its output bytes, or the corners,
 * offsets and parts its plan keeps (8 * (ndim + 3) bytes a box at most), overflow int64 */
static int boxes_nbytes(long long nboxes, int ndim, long long count, long long typesize) {
  if (nboxes > LLONG_MAX / (8 * (ndim + 3)) || (count > 0 && nboxes > LLONG_MAX / (count * typesize))) {
    fprintf(stderr, "blosc_b200: %lld boxes of %lld bytes overflow int64\n", nboxes, count * typesize);
    return -1;
  }
  return 0;
}

/* The origin box of a batch (box_build at corner 0) and the check's arguments that follow from the geometry */
static void boxes_build(int ndim, const int64_t* shape, const int64_t* extent, long long nitems, long long nboxes,
                        B2Box* box, BoxCheckArgs* ck) {
  int k;
  box_build(ndim, shape, g_box_origin, extent, NULL, nitems, box);
  memset(ck, 0, sizeof *ck);
  ck->box = *box; ck->nboxes = nboxes; ck->ndim = ndim;
  ck->span = b2_box_unrank(box, box->count - 1, 0) + 1;
  ck->stride[ndim - 1] = 1;
  for (k = ndim - 2; k >= 0; k--) ck->stride[k] = ck->stride[k + 1] * shape[k + 1];
  for (k = 0; k < ndim; k++) ck->hi[k] = shape[k] - extent[k];
}

/* The check's scratch in w->fplan, which the chunk plans leave alone: for a frame (nchunks > 0), the first failing box
 * (all ones) and the touched flags of its chunks (zeroed); then the boxes' offsets, for a frame each box's part of the
 * chunk being read (*part), and the caller's corners (uploaded when they are in host memory).  Fills ck's pointers but
 * for a chunk's ck->bad, which the chunk plan's record holds.  Returns 0, or -1. */
static int boxes_scratch(b2_ws* w, const int64_t* starts, long long nchunks, BoxCheckArgs* ck, long long** part) {
  const size_t o_off = nchunks ? B2_AL(16 + 4 * (size_t)nchunks) : 0, o_part = B2_AL(o_off + 8 * (size_t)ck->nboxes);
  const size_t o_up = o_part + (nchunks ? 16 * (size_t)ck->nboxes : 0), up = 8 * (size_t)ck->ndim * (size_t)ck->nboxes;
  uint8_t* base;
  if (buf_ensure(&w->fplan, o_up + up)) return -1;
  base = (uint8_t*)w->fplan.p;
  if (nchunks) {
    if (b2_memset_dev(base, 0, o_off, w->stream) || b2_memset_dev(base, 0xff, 8, w->stream)) return -1;
    ck->bad = (unsigned long long*)base; ck->touched = (int*)(base + 16); ck->nchunks = nchunks;
  }
  ck->off = (long long*)(base + o_off);
  *part = nchunks ? (long long*)(base + o_part) : NULL;
  ck->starts = (const long long*)dev_list(w, starts, b2_ptr_is_device(starts), up, base + o_up);
  return ck->starts ? 0 : -1;
}

/* A failing corner: box i of the check's corners (device memory) is read back, and the message names the box, the
 * first dimension whose coordinate fails and the interval it must lie in.  Returns -1. */
static int box_bad_corner(b2_ws* w, const BoxCheckArgs* ck, unsigned long long i) {
  long long c[B2_BOX_MAXDIM];
  int k;
  if (copy_any(c, 0, ck->starts + i * (unsigned long long)ck->ndim, 1, 8 * (size_t)ck->ndim, w->stream)) return -1;
  for (k = 0; k < ck->ndim; k++)
    if (c[k] < 0 || c[k] > ck->hi[k]) {
      fprintf(stderr, "blosc_b200: box %llu starts at %lld in dimension %d, not in [0, %lld]\n", i, c[k], k, ck->hi[k]);
      break;
    }
  return -1;
}

/* One chunk's part of a batch: the chunk (header h, checked) holds the array's flat items [window, window + nbytes /
 * typesize); the boxes at the offsets ck->off land at d_dst (device memory), box i at i * count * typesize, total bytes
 * in all; with part (room for two words a box: a frame), only each box's part in the chunk.  check: launch ck's corner
 * check first, its verdict read back with the plan's record (a chunk call).  Returns total, blosc_d's code when a
 * touched block fails to decode (nothing is written then), or -1. */
static long long boxes_read(b2_ws* w, const void* src, int src_dev, const b2_hdr* h, int codec, BoxCheckArgs* ck,
                            int check, long long window, long long* part, long long total, uint8_t* d_dst) {
  const int in_place = (h->flags & BLOSC_MEMCPYED) && src_dev;   /* a memcpyed device chunk is read in place */
  GetitemsPlan rec = {0};
  BoxesPlanArgs bp;
  BoxesGatherArgs ga;
  int rc;
  memset(&ga, 0, sizeof ga);
  ga.box = ck->box; ga.off = ck->off; ga.part = part; ga.window = window;
  ga.total = total; ga.typesize = h->typesize; ga.blocksize = h->blocksize; ga.dst = d_dst;
  bp.box = ck->box; bp.off = ck->off; bp.nboxes = ck->nboxes; bp.span = ck->span; bp.window = window;
  bp.part = part; bp.in_place = in_place; bp.pad = 0;
  bp.per_box = (ck->span * h->typesize + h->blocksize - 1) / h->blocksize + 1;   /* the blocks one box can touch */
  if (bp.per_box > h->nblocks) bp.per_box = h->nblocks;
  if (bp.per_box > LLONG_MAX / ck->nboxes) {
    fprintf(stderr, "blosc_b200: %lld boxes of %lld blocks each are too many to plan\n", ck->nboxes, bp.per_box);
    return -1;
  }
  if (!in_place || check || part) {
    if (!plan_scratch(w, h, 0, 0, &bp.plan)) return -1;
    if (check) {
      ck->bad = &bp.plan.rec->bad_box;
      if (b2_memset_dev(ck->bad, 0xff, 8, w->stream) || b2_launch_box_check(ck, w->stream)) return -1;
    }
    if (((!in_place || part) && b2_launch_boxes_plan(&bp, w->stream)) || read_plan(w, bp.plan.rec, &rec, sizeof rec))
      return -1;
    if (check && rec.bad_box != ~0ull) return box_bad_corner(w, ck, rec.bad_box);
    if (!in_place) ga.slot = bp.plan.slot;
  }
  if (touched_source(w, src, src_dev, h, codec, rec.nlisted, rec.has_left, &ga.src, &ga.status)) return -1;
  if (b2_launch_boxes_gather(&ga, w->stream)) { ws_reset_counters(w); return -1; }
  rc = read_verdict(w, ga.status);
  return rc < 0 ? rc : total;
}

long long blosc_b200_getslices(const void* src, int ndim, const int64_t* shape, const int64_t* extent,
                               long long nboxes, const int64_t* starts, void* dest) {
  b2_hdr h;
  B2Box box;
  BoxCheckArgs ck;
  b2_ws* w;
  uint8_t* d_dst;
  long long nitems = 0, nbytes, result = -1, *part = NULL;
  int src_dev, dest_dev, codec = 0, rc;
  if (boxes_geometry(ndim, shape, extent, nboxes, src, dest, starts, &nitems)) return -1;
  src_dev = b2_ptr_is_device(src);
  rc = getitem_header(NULL, src, src_dev, -1, &h, &codec);
  if (rc) return rc;
  if (box_nbytes(nitems, h.typesize, (unsigned long long)h.nbytes)) return -1;
  if (nboxes == 0 || box_empty(ndim, g_box_origin, extent)) return 0;
  boxes_build(ndim, shape, extent, nitems, nboxes, &box, &ck);
  if (boxes_nbytes(nboxes, ndim, box.count, h.typesize)) return -1;
  nbytes = nboxes * box.count * h.typesize;
  dest_dev = b2_ptr_is_device(dest);
  if (!(w = ws_acquire())) return -1;
  if ((d_dst = stage_dest(&w->slots, dest, dest_dev, (size_t)nbytes)) && !boxes_scratch(w, starts, 0, &ck, &part)) {
    result = boxes_read(w, src, src_dev, &h, codec, &ck, 1, 0, NULL, nbytes, d_dst);
    if (result > 0 && !dest_dev && d2h_any(w, dest, d_dst, (size_t)result)) result = -1;
  }
  ws_release(w);
  return result;
}

/* ------------------------------------------------------------------------- */
/* orthogonal index selections (blosc_b200_getoindex, _frame_getoindex)       */
/* ------------------------------------------------------------------------- */
/* numpy's a[np.ix_(...)]: some dimensions select a list of coordinates, the others a slice.  The selection (B2OSel,
 * b2_args.h) holds the lists as device pointers, so neither the plan nor the gather keeps per-run state:
 * oindex_touch_kernel checks the entries and marks the touched blocks in one launch, the PLAN_SLOT scan lists them,
 * they are decoded as for a box, and oindex_gather_kernel writes the output.  A frame runs the check once over all its
 * chunks, which also flags the touched ones. */

/* whether some dimension is a list (ndim already checked) */
static int osel_any(int ndim, const int64_t* const* index) {
  int k;
  for (k = 0; index && k < ndim; k++) if (index[k]) return 1;
  return 0;
}

/* The checks of an index selection that need no data, with getslice_step's messages on the slice dimensions: its
 * slices with the list dimensions made whole (st, sp, t), the array's items, the output's items, and device lists on
 * the device the call runs on (that of data or dest when either is device memory).  -1 with a message when one fails. */
static int osel_geometry(int ndim, const int64_t* shape, const int64_t* start, const int64_t* stop, const int64_t* step,
                         const int64_t* const* index, const int64_t* nindex, const void* data, const void* dest,
                         int64_t* st, int64_t* sp, int64_t* t, long long* nitems, long long* count) {
  long long prod = 1;
  int k, dev, zero = 0;
  for (k = 0; k < ndim; k++) {
    st[k] = index[k] ? 0 : start[k]; sp[k] = index[k] ? shape[k] : stop[k]; t[k] = index[k] || !step ? 1 : step[k];
  }
  if (box_geometry(ndim, shape, st, sp, nitems) || box_steps(ndim, t)) return -1;
  for (k = 0; k < ndim; k++) {
    const long long n = index[k] ? nindex[k] : st[k] == sp[k] ? 0 : (sp[k] - st[k] - 1) / t[k] + 1;
    if (n < 0) { fprintf(stderr, "blosc_b200: nindex[%d] = %lld is negative\n", k, n); return -1; }
    zero |= n == 0;
    if (!zero && ((index[k] && n > (1LL << 56)) || prod > LLONG_MAX / n)) {   /* the check's key holds 56 bits */
      fprintf(stderr, "blosc_b200: the selection's item count overflows int64\n");
      return -1;
    }
    if (!zero) prod *= n;
  }
  *count = zero ? 0 : prod;
  dev = b2_ptr_is_device(data) ? b2_ptr_device(data) : b2_ptr_is_device(dest) ? b2_ptr_device(dest) : b2_get_device();
  for (k = 0; k < ndim; k++)
    if (index[k] && b2_ptr_is_device(index[k]) && b2_ptr_device(index[k]) != dev) {
      fprintf(stderr, "blosc_b200: index[%d] is not on device %d, where the call runs\n", k, dev);
      return -1;
    }
  return 0;
}

/* the output's bytes: -1 with a message when they overflow int64 */
static int osel_nbytes(long long count, long long typesize) {
  if (count > LLONG_MAX / typesize) {
    fprintf(stderr, "blosc_b200: the selection's %lld items of %lld bytes overflow int64\n", count, typesize);
    return -1;
  }
  return 0;
}

/* The selection of a checked, non-empty one: the lists as the kernels read them, in device memory (host lists are
 * uploaded into w->segs, one copy each), and the slice dimensions merged as box_build merges them, a list never.
 * Returns 0, or -1 when an upload fails. */
static int osel_build(b2_ws* w, int ndim, const int64_t* shape, const int64_t* st, const int64_t* sp, const int64_t* t,
                      const int64_t* const* index, const int64_t* nindex, B2OSel* s) {
  long long sh[B2_BOX_MAXDIM], up = 0, at = 0;
  int k, n = 0;
  memset(s, 0, sizeof *s);
  for (k = 0; k < ndim; k++) if (index[k] && !b2_ptr_is_device(index[k])) up += nindex[k];
  if (up && buf_ensure(&w->segs, 8 * (size_t)up + 64)) return -1;
  for (k = 0; k < ndim; k++) {
    if (index[k]) {
      const long long* l = (const long long*)index[k];
      if (!b2_ptr_is_device(l)) {
        l = (const long long*)w->segs.p + at;
        if (h2d_any(w, (void*)l, index[k], 8 * (size_t)nindex[k])) return -1;
        at += nindex[k];
      }
      sh[n] = shape[k]; s->list[n] = l; s->ext[n] = nindex[k]; s->step[n] = 1; s->kdim[n] = k;
      s->lbase[n] = s->nentries; s->nentries += nindex[k];
      n++;
    } else {
      const long long e = (sp[k] - st[k] - 1) / t[k] + 1, u = e == 1 ? 1 : t[k];
      if (n > 0 && !s->list[n - 1] && s->step[n - 1] == 1 && u == 1 && st[k] == 0 && e == shape[k]) {
        sh[n - 1] *= shape[k]; s->start[n - 1] *= shape[k]; s->ext[n - 1] *= shape[k];
      } else {
        sh[n] = shape[k]; s->start[n] = st[k]; s->step[n] = u; s->ext[n] = e;
        n++;
      }
    }
  }
  s->ndim = n;
  s->stride[n - 1] = 1;
  for (k = n - 2; k >= 0; k--) s->stride[k] = s->stride[k + 1] * sh[k + 1];
  s->count = 1;
  for (k = 0; k < n; k++) { s->shape[k] = sh[k]; s->count *= s->ext[k]; }
  s->run = !s->list[n - 1] && s->step[n - 1] == 1 ? s->ext[n - 1] : 1;
  s->slab = s->count / s->ext[0];
  s->nruns = s->count / s->run;
  return 0;
}

/* A bad list entry, from the check's key (the caller's dimension << 56 | position): the entry is read back from the
 * device list and named.  Returns -1. */
static int osel_bad_entry(b2_ws* w, const B2OSel* s, unsigned long long key) {
  const int kd = (int)(key >> 56);
  const long long q = (long long)(key & ((1ull << 56) - 1));
  long long c = 0;
  int k;
  for (k = 0; k < s->ndim; k++)
    if (s->list[k] && s->kdim[k] == kd && !copy_any(&c, 0, s->list[k] + q, 1, 8, w->stream))
      fprintf(stderr, "blosc_b200: index[%d][%lld] = %lld is not in [0, %lld)\n", kd, q, c, s->shape[k]);
  return -1;
}

/* One chunk's part of a selection: the chunk (header h, checked) holds the array's flat items [window, window + nbytes
 * / typesize), and the output bytes [g0, g1) are written at d_dst + byte (device memory).  A chunk call (frame 0)
 * checks the list entries with the touch, and a memcpyed device chunk is then read in place after the check alone; a
 * frame's chunk (frame 1, checked already) writes only the items inside it.  Returns 0, blosc_d's code when a touched
 * block fails to decode (nothing is written then), or -1. */
static int oindex_chunk(b2_ws* w, const void* src, int src_dev, const b2_hdr* h, int codec, const B2OSel* sel, int frame,
                        long long window, long long g0, long long g1, uint8_t* d_dst) {
  const int in_place = (h->flags & BLOSC_MEMCPYED) && src_dev;
  GetitemsPlan rec = {0};
  OIndexGatherArgs ga;
  int rc;
  memset(&ga, 0, sizeof ga);
  ga.sel = *sel; ga.window = window; ga.wend = window + h->nbytes / h->typesize; ga.g0 = g0; ga.g1 = g1;
  ga.typesize = h->typesize; ga.blocksize = h->blocksize; ga.clip = frame; ga.dst = d_dst;
  if (!in_place || !frame) {
    OIndexPlanArgs pa;
    memset(&pa, 0, sizeof pa);
    pa.sel = *sel; pa.window = window; pa.check = !frame;
    if (!in_place) { pa.r0 = g0 / (sel->run * h->typesize); pa.r1 = g1 / (sel->run * h->typesize); }
    if (!plan_scratch(w, h, 0, 0, &pa.plan)) return -1;
    pa.bad = &pa.plan.rec->bad_box;
    if (b2_memset_dev(pa.bad, 0xff, 8, w->stream) || b2_launch_oindex_plan(&pa, w->stream) ||
        read_plan(w, pa.plan.rec, &rec, sizeof rec))
      return -1;
    if (rec.bad_box != ~0ull) return osel_bad_entry(w, sel, rec.bad_box);
    if (!in_place) ga.slot = pa.plan.slot;
  }
  if (touched_source(w, src, src_dev, h, codec, rec.nlisted, rec.has_left, &ga.src, &ga.status)) return -1;
  if (b2_launch_oindex_gather(&ga, w->stream)) { ws_reset_counters(w); return -1; }
  rc = read_verdict(w, ga.status);
  return rc < 0 ? rc : 0;
}

long long blosc_b200_getoindex(const void* src, int ndim, const int64_t* shape, const int64_t* start,
                               const int64_t* stop, const int64_t* step, const int64_t* const* index,
                               const int64_t* nindex, void* dest) {
  int64_t st[B2_BOX_MAXDIM], sp[B2_BOX_MAXDIM], t[B2_BOX_MAXDIM];
  b2_hdr h;
  B2OSel sel;
  b2_ws* w;
  uint8_t* d_dst;
  long long nitems = 0, count = 0, result = -1;
  int src_dev, dest_dev, codec = 0, rc;
  if (ndim < 1 || ndim > B2_BOX_MAXDIM || !osel_any(ndim, index))      /* no list: getslice_step (which checks ndim) */
    return blosc_b200_getslice_step(src, ndim, shape, start, stop, step, dest);
  if (osel_geometry(ndim, shape, start, stop, step, index, nindex, src, dest, st, sp, t, &nitems, &count)) return -1;
  src_dev = b2_ptr_is_device(src);
  rc = getitem_header(NULL, src, src_dev, -1, &h, &codec);
  if (rc) return rc;
  if (box_nbytes(nitems, h.typesize, (unsigned long long)h.nbytes) || osel_nbytes(count, h.typesize)) return -1;
  if (count == 0) return 0;
  dest_dev = b2_ptr_is_device(dest);
  if (!(w = ws_acquire())) return -1;
  if ((d_dst = stage_dest(&w->slots, dest, dest_dev, (size_t)(count * h.typesize))) &&
      !osel_build(w, ndim, shape, st, sp, t, index, nindex, &sel) &&
      (result = oindex_chunk(w, src, src_dev, &h, codec, &sel, 0, 0, 0, count * h.typesize, d_dst)) == 0) {
    result = count * h.typesize;
    if (!dest_dev && d2h_any(w, dest, d_dst, (size_t)result)) result = -1;
  }
  ws_release(w);
  return result;
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
  /* a chunk grid (blosc_b200_grid_compress): src is the array */
  int ndim, src_dev, skip_fill;
  long long itemsize, nitems, chunk_items;
  int64_t shape[B2_BOX_MAXDIM], chunkshape[B2_BOX_MAXDIM];
  const uint8_t* fill;      /* the fill pattern where the pack reads it (device memory for a device src); NULL: zeros */
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
                         j->compressor, j->blocksize, j->nthreads, &pl, j->dest_dev, NULL);
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

/* An opened frame: its index, and (frame_open_items) the items its chunks hold */
typedef struct {
  size_t nbytes, chunksize, nchunks;
  uint64_t* off;            /* [nchunks + 1] chunk offsets, malloc'ed; off[nchunks] is the frame's cbytes */
  int dev;                  /* the frame is in device memory */
  size_t typesize, ipc;     /* chunk 0's typesize (1 in a frame with no chunk) and the items per chunk */
} b2_frame;

/* reads and validates the index into *f */
static int frame_open(const void* frame, size_t framesize, b2_frame* f) {
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
    f->nbytes = (size_t)rd_u64(hb + 8); cbytes = rd_u64(hb + 16);
    f->chunksize = rd_u32(hb + 24); n = rd_u32(hb + 28);
    if (cbytes > framesize || cbytes < B2_FRAME_HDR + 8 * (uint64_t)n) break;
    if (f->nbytes > 0 && (f->chunksize == 0 || f->chunksize > BLOSC_MAX_BUFFERSIZE)) break;
    if (n != (f->nbytes ? (f->nbytes + f->chunksize - 1) / f->chunksize : 0)) break;
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
    f->nchunks = n; f->off = off; f->dev = dev;
  } while (0);
  return rc;
}

/* frame_open, then the typesize of chunk 0 and the items per chunk.  -1 when the frame cannot be read, -2 when that
 * typesize (left in f->typesize) does not divide the chunksize; f->off is freed on a failure. */
static int frame_open_items(const void* frame, size_t framesize, b2_frame* f) {
  uint8_t hb[16];
  if (frame_open(frame, framesize, f)) return -1;
  f->typesize = 1;
  if (f->nchunks > 0) {
    if (copy_some(hb, 0, (const uint8_t*)frame + f->off[0], f->dev, 16)) { free(f->off); return -1; }
    f->typesize = hb[3];
    if (f->typesize == 0 || f->chunksize % f->typesize) { free(f->off); return -2; }
  }
  f->ipc = f->chunksize / f->typesize;
  return 0;
}

/* The header of chunk c of an opened frame, checked as blosc_getitem checks it, within the chunk's slot: 0,
 * getitem_header's code, or 1 when the chunk's typesize is not the frame's (its items would not fit in dest) */
static int frame_chunk_header(b2_ws* w, const void* frame, const b2_frame* f, size_t c, b2_hdr* h, int* codec) {
  const int rc = getitem_header(w, (const uint8_t*)frame + f->off[c], f->dev, (long long)(f->off[c + 1] - f->off[c]), h,
                                codec);
  if (rc) return rc;
  return (size_t)h->typesize != f->typesize;
}

int blosc_b200_frame_info(const void* frame, size_t framesize, size_t* nbytes, size_t* cbytes, size_t* chunksize,
                          size_t* nchunks) {
  b2_frame f;
  if (!backend_ready()) return -1;
  if (frame_open(frame, framesize, &f)) return -1;
  if (nbytes) *nbytes = f.nbytes;
  if (cbytes) *cbytes = (size_t)f.off[f.nchunks];
  if (chunksize) *chunksize = f.chunksize;
  if (nchunks) *nchunks = f.nchunks;
  free(f.off);
  return 0;
}

long long blosc_b200_frame_chunk(const void* frame, size_t framesize, size_t i, size_t* chunk_cbytes) {
  b2_frame f;
  long long r;
  if (!backend_ready()) return -1;
  if (frame_open(frame, framesize, &f)) return -1;
  if (i >= f.nchunks) { free(f.off); return -1; }
  if (chunk_cbytes) *chunk_cbytes = (size_t)(f.off[i + 1] - f.off[i]);
  r = (long long)f.off[i];
  free(f.off);
  return r;
}

long long blosc_b200_frame_decompress(const void* frame, size_t framesize, void* dest, size_t destsize,
                                      int numinternalthreads) {
  b2_frame_job j;
  b2_frame f;
  int rc;
  if (!backend_ready()) return -1;
  if (frame_open(frame, framesize, &f)) return -1;
  if (f.nbytes > destsize) { free(f.off); return -1; }
  memset(&j, 0, sizeof j);
  j.nchunks = (int)f.nchunks; j.workers = frame_workers((int)f.nchunks); j.nthreads = numinternalthreads;
  j.chunksize = f.chunksize; j.nbytes = f.nbytes; j.frame = (const uint8_t*)frame; j.dest = (uint8_t*)dest;
  j.offsets = f.off;
  rc = f.nchunks ? frame_run(&j, frame_decompress_worker) : 0;
  free(f.off);
  return rc ? -1 : (long long)f.nbytes;
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
  size_t r, npieces = 0, i, j;
  b2_frame f;
  b2_piece* pieces = NULL;
  long long result = -1, at = 0;
  if (frame_open_items(frame, framesize, &f)) return -1;
  do {
    const size_t ts = f.typesize, ipc = f.ipc;
    if (f.nchunks == 0) {
      for (r = 0; r < nranges && nitems[r] == 0; r++) {}
      result = r == nranges ? 0 : -1;
      break;
    }
    for (r = 0; r < nranges; r++) {
      if (b2_frame_range_bad(starts[r], nitems[r], f.nbytes / ts)) { fprintf(stderr, "`start`+`nitems` out of bounds"); break; }
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
      rc = getitems_chunk((const uint8_t*)frame + f.off[pieces[i].chunk],
                          (long long)(f.off[pieces[i].chunk + 1] - f.off[pieces[i].chunk]), (int)(j - i), st, st + (j - i),
                          dsts, dest);
      free(st); free(dsts);
      if (rc != want) { result = rc < 0 ? rc : -1; break; }
      result += rc;
    }
  } while (0);
  free(pieces); free(f.off);
  return result;
}

long long blosc_b200_frame_getitem(const void* frame, size_t framesize, size_t start, size_t nitems, void* dest) {
  if (!backend_ready()) return -1;
  return frame_getitems_host(frame, framesize, 1, &start, &nitems, dest);
}

/* The GPU plan of a frame (dev_chunk.cuh fplan_*_kernel), for range lists of which at least one is in device memory
 * (a host one is uploaded).  It checks every range as frame_getitems_host does, cuts the ranges into pieces and
 * gathers each chunk's pieces into a bucket of device piece lists; the host reads back one small record and then the
 * list of touched chunks.  Each touched chunk, in ascending order, then runs the chunk's GPU plan on its bucket, every
 * piece landing at its own dest offset: in dest itself when it is device memory, else in a device staging buffer that
 * is copied to dest at the end.  Neither the lists nor the pieces travel to the host. */
static long long frame_getitems_gpu(const void* frame, size_t framesize, size_t nranges, const size_t* starts,
                                    int starts_dev, const size_t* nitems, int nitems_dev, void* dest) {
  const int dest_dev = b2_ptr_is_device(dest);
  b2_frame f;
  FrameTouch* touched = NULL;
  long long result = -1;
  b2_ws* w;
  if (frame_open_items(frame, framesize, &f)) return -1;
  if (nranges > ((size_t)-1) / 64 || !(w = ws_acquire())) { free(f.off); return -1; }
  do {
    /* one scratch: the record, the tickets, the tile flags and the difference array over chunks, all zeroed; then the
     * tiles' values, the range offsets, the bucket cursors, the touched chunks and an uploaded host list */
    const size_t nc = f.nchunks, tr = (nranges + PLAN_TILE - 1) / PLAN_TILE, tc = (nc + PLAN_TILE - 1) / PLAN_TILE;
    const size_t tiles = tr + 3 * tc, o_tk = 32, o_flag = 64, o_count = B2_AL(o_flag + 4 * tiles);
    const size_t zeroed = B2_AL(o_count + 8 * (nc + 1)), o_vals = zeroed, o_dst = B2_AL(o_vals + 16 * tiles);
    const size_t o_cursor = B2_AL(o_dst + 8 * nranges), o_touch = B2_AL(o_cursor + 8 * nc);
    const size_t o_up = B2_AL(o_touch + sizeof(FrameTouch) * nc);
    FramePlanArgs fa;
    FramePlan rec;
    uint8_t* base;
    uint8_t* d_dest;
    long long sum = 0, t, done;
    int k;
    if (buf_ensure(&w->fplan, o_up + 8 * nranges)) break;
    base = (uint8_t*)w->fplan.p;
    memset(&fa, 0, sizeof fa);
    if (!(fa.starts = (const unsigned long long*)dev_list(w, starts, starts_dev, 8 * nranges, base + o_up)) ||
        !(fa.nitems = (const unsigned long long*)dev_list(w, nitems, nitems_dev, 8 * nranges, base + o_up)))
      break;
    if (nc == 0) fa.starts = NULL;              /* an empty frame: only the counts are looked at, as on the host */
    if (b2_memset_dev(base, 0, zeroed, w->stream) || b2_memset_dev(base, 0xff, 8, w->stream)) break;
    fa.nranges = (long long)nranges; fa.total_items = f.nbytes / f.typesize; fa.ipc = (long long)f.ipc;
    fa.typesize = (int)f.typesize; fa.nchunks = (long long)nc;
    fa.dst = (long long*)(base + o_dst); fa.count = (long long*)(base + o_count); fa.cursor = (long long*)(base + o_cursor);
    fa.touched = (FrameTouch*)(base + o_touch); fa.rec = (FramePlan*)base;
    for (k = 0; k < 4; k++) {                           /* FPLAN_DST over the ranges, the other three over the chunks */
      const size_t before = k == 0 ? 0 : tr + (size_t)(k - 1) * tc;
      fa.scan[k] = plan_scan(base + o_tk + 4 * k, base + o_flag + 4 * before, base + o_vals + 16 * before, 8,
                             k == 0 ? tr : tc);
    }
    if (b2_launch_fplan(&fa, w->stream) || read_plan(w, base, &rec, sizeof rec)) break;
    if (rec.bad != ~0ull) {                                                /* frame_getitems_host's verdict */
      if (nc > 0) fprintf(stderr, "`start`+`nitems` out of bounds");
      break;
    }
    if (rec.npieces == 0) { result = 0; break; }
    if (buf_ensure(&w->fpieces, 16 * (size_t)rec.npieces)) break;
    fa.pdst = (long long*)w->fpieces.p; fa.pstart = (int*)(fa.pdst + rec.npieces); fa.pnitems = fa.pstart + rec.npieces;
    if (b2_launch_fplan_scatter(&fa, w->stream)) break;
    if (!(touched = (FrameTouch*)malloc(sizeof(FrameTouch) * (size_t)rec.ntouched))) break;
    if (d2h_any(w, touched, base + o_touch, sizeof(FrameTouch) * (size_t)rec.ntouched)) break;
    if (!(d_dest = stage_dest(&w->fstage, dest, dest_dev, (size_t)rec.total))) break;
    for (t = 0; t < rec.ntouched; t++) {              /* the chunks in ascending order; the first failure decides */
      const FrameTouch ch = touched[t];
      b2_hdr h;
      int codec = 0, rc;
      long long got = 0;
      rc = frame_chunk_header(w, frame, &f, (size_t)ch.chunk, &h, &codec);
      if (rc) { if (rc < 0) result = rc; break; }
      for (done = 0; done < ch.count; done += INT_MAX) {     /* the chunk plan counts its ranges in int */
        const int n = ch.count - done < INT_MAX ? (int)(ch.count - done) : INT_MAX;
        const long long at = ch.base + done;
        got = getitems_gpu(w, (const uint8_t*)frame + f.off[ch.chunk], f.dev, &h, codec, n, fa.pstart + at, 1,
                           fa.pnitems + at, 1, fa.pdst + at, d_dest, 1);
        if (got < 0) break;
        sum += got;
      }
      if (got < 0) { result = got; break; }
    }
    if (t < rec.ntouched || sum != rec.total) break;
    if (!dest_dev && d2h_any(w, dest, d_dest, (size_t)rec.total)) break;
    result = rec.total;
  } while (0);
  ws_release(w);
  free(touched); free(f.off);
  return result;
}

/* Range lists in device memory are planned on the GPU when they are on the device the call runs on: that of the frame
 * or of dest when either is device memory, else the current one.  Lists on another device are copied to the host (one
 * copy each), and the frame is planned there. */
long long blosc_b200_frame_getitems(const void* frame, size_t framesize, size_t nranges, const size_t* starts,
                                    const size_t* nitems, void* dest) {
  size_t* h = NULL;
  long long result = -1;
  int starts_dev, nitems_dev, dev;
  if (nranges == 0) return 0;
  if (!backend_ready()) return -1;
  starts_dev = b2_ptr_is_device(starts); nitems_dev = b2_ptr_is_device(nitems);
  if (!starts_dev && !nitems_dev) return frame_getitems_host(frame, framesize, nranges, starts, nitems, dest);
  dev = b2_ptr_is_device(frame) ? b2_ptr_device(frame) : b2_ptr_is_device(dest) ? b2_ptr_device(dest) : b2_get_device();
  if ((!starts_dev || b2_ptr_device(starts) == dev) && (!nitems_dev || b2_ptr_device(nitems) == dev))
    return frame_getitems_gpu(frame, framesize, nranges, starts, starts_dev, nitems, nitems_dev, dest);
  if (nranges > ((size_t)-1) / (2 * sizeof(size_t)) || !(h = (size_t*)malloc(2 * sizeof(size_t) * nranges))) return -1;
  if (!copy_some(h, 0, starts, starts_dev, sizeof(size_t) * nranges) &&
      !copy_some(h + nranges, 0, nitems, nitems_dev, sizeof(size_t) * nranges))
    result = frame_getitems_host(frame, framesize, nranges, h, h + nranges, dest);
  free(h);
  return result;
}

/* A box of the array a frame holds, in items of chunk 0's typesize: the touched chunks and where each one's part lands
 * in dest follow from the box (b2_box_next, b2_box_rank on the chunks' item windows), and each touched chunk, in
 * ascending order, is read by the chunk path; the first failure decides the result.  A host dest is staged in device
 * memory and copied out once, so it is untouched on a failure. */
long long blosc_b200_frame_getslice_step(const void* frame, size_t framesize, int ndim, const int64_t* shape,
                                         const int64_t* start, const int64_t* stop, const int64_t* step, void* dest) {
  size_t c;
  b2_frame f;
  long long nitems = 0, ts, ipc, sum = 0, got = 0, result = -1;
  int dest_dev, rc;
  B2Box box;
  b2_ws* w;
  uint8_t* d_dst;
  if (!backend_ready()) return -1;
  if (box_geometry(ndim, shape, start, stop, &nitems) || box_steps(ndim, step)) return -1;
  rc = frame_open_items(frame, framesize, &f);
  if (rc == -2)
    fprintf(stderr, "blosc_b200: chunk 0's typesize %lld does not divide the frame's chunksize\n", (long long)f.typesize);
  if (rc) return -1;
  ts = (long long)f.typesize; ipc = (long long)f.ipc;
  dest_dev = b2_ptr_is_device(dest);
  if (box_nbytes(nitems, ts, (unsigned long long)f.nbytes)) { free(f.off); return -1; }
  if (box_empty(ndim, start, stop)) { free(f.off); return 0; }
  box_build(ndim, shape, start, stop, step, nitems, &box);
  if (!(w = ws_acquire())) { free(f.off); return -1; }
  do {
    if (!(d_dst = stage_dest(&w->fstage, dest, dest_dev, (size_t)(box.count * ts)))) break;
    for (c = 0; c < f.nchunks; c++) {
      const long long w0 = (long long)c * ipc, w1 = w0 + ipc < nitems ? w0 + ipc : nitems;
      b2_hdr h;
      int codec = 0;
      if (b2_box_next(&box, w0, box.stepped) >= w1) continue;             /* no box item in this chunk */
      got = frame_chunk_header(w, frame, &f, c, &h, &codec);
      if (got < 0) break;
      if (got || h.nbytes != (w1 - w0) * ts) {
        fprintf(stderr, "blosc_b200: chunk %zu holds %d items of %d bytes, not the frame's %lld of %lld\n", c,
                h.nbytes / h.typesize, h.typesize, w1 - w0, ts);
        got = -1;
        break;
      }
      got = getslice_chunk(w, (const uint8_t*)frame + f.off[c], f.dev, &h, codec, &box, w0,
                           d_dst + b2_box_rank(&box, w0, box.stepped) * ts);
      if (got < 0) break;
      sum += got;
    }
    if (c < f.nchunks) { result = got; break; }
    if (sum != box.count * ts) break;
    if (!dest_dev && d2h_any(w, dest, d_dst, (size_t)sum)) break;
    result = sum;
  } while (0);
  ws_release(w);
  free(f.off);
  return result;
}

long long blosc_b200_frame_getslice(const void* frame, size_t framesize, int ndim, const int64_t* shape,
                                    const int64_t* start, const int64_t* stop, void* dest) {
  return blosc_b200_frame_getslice_step(frame, framesize, ndim, shape, start, stop, NULL, dest);
}

/* Boxes of the array a frame holds: one corner check over all of them, which also flags the chunks that hold an item
 * of some box, read back with one sync; then each flagged chunk, in ascending order, reads its part of every box by
 * the chunk path, clipped to the chunk, and the first failure decides the result.  A host dest is staged in device
 * memory and copied out once. */
long long blosc_b200_frame_getslices(const void* frame, size_t framesize, int ndim, const int64_t* shape,
                                     const int64_t* extent, long long nboxes, const int64_t* starts, void* dest) {
  size_t c;
  b2_frame f;
  long long nitems = 0, ts, ipc, nbytes, got = 0, result = -1;
  int dest_dev, rc;
  B2Box box;
  BoxCheckArgs ck;
  b2_ws* w;
  uint8_t *d_dst, *head = NULL;
  long long* part = NULL;
  if (!backend_ready()) return -1;
  if (boxes_geometry(ndim, shape, extent, nboxes, frame, dest, starts, &nitems)) return -1;
  rc = frame_open_items(frame, framesize, &f);
  if (rc == -2)
    fprintf(stderr, "blosc_b200: chunk 0's typesize %lld does not divide the frame's chunksize\n", (long long)f.typesize);
  if (rc) return -1;
  ts = (long long)f.typesize; ipc = (long long)f.ipc;
  dest_dev = b2_ptr_is_device(dest);
  if (box_nbytes(nitems, ts, (unsigned long long)f.nbytes)) { free(f.off); return -1; }
  if (nboxes == 0 || box_empty(ndim, g_box_origin, extent)) { free(f.off); return 0; }
  boxes_build(ndim, shape, extent, nitems, nboxes, &box, &ck);
  if (boxes_nbytes(nboxes, ndim, box.count, ts)) { free(f.off); return -1; }
  nbytes = nboxes * box.count * ts;
  ck.ipc = ipc;
  if (!(w = ws_acquire())) { free(f.off); return -1; }
  do {
    if (!(d_dst = stage_dest(&w->fstage, dest, dest_dev, (size_t)nbytes))) break;
    if (boxes_scratch(w, starts, (long long)f.nchunks, &ck, &part) || b2_launch_box_check(&ck, w->stream)) break;
    if (!(head = (uint8_t*)malloc(16 + 4 * f.nchunks)) || d2h_any(w, head, ck.bad, 16 + 4 * f.nchunks)) break;
    if (*(unsigned long long*)head != ~0ull) { box_bad_corner(w, &ck, *(unsigned long long*)head); break; }
    for (c = 0; c < f.nchunks; c++) {
      const long long w0 = (long long)c * ipc, w1 = w0 + ipc < nitems ? w0 + ipc : nitems;
      b2_hdr h;
      int codec = 0;
      if (!((int*)(head + 16))[c]) continue;                               /* no box item in this chunk */
      got = frame_chunk_header(w, frame, &f, c, &h, &codec);
      if (got < 0) break;
      if (got || h.nbytes != (w1 - w0) * ts) {
        fprintf(stderr, "blosc_b200: chunk %zu holds %d items of %d bytes, not the frame's %lld of %lld\n", c,
                h.nbytes / h.typesize, h.typesize, w1 - w0, ts);
        got = -1;
        break;
      }
      got = boxes_read(w, (const uint8_t*)frame + f.off[c], f.dev, &h, codec, &ck, 0, w0, part, nbytes, d_dst);
      if (got < 0) break;
    }
    if (c < f.nchunks) { result = got; break; }
    if (!dest_dev && d2h_any(w, dest, d_dst, (size_t)nbytes)) break;
    result = nbytes;
  } while (0);
  ws_release(w);
  free(head);
  free(f.off);
  return result;
}

/* The output bytes [*g0, *g1) that a frame chunk of items [w0, w1) can write: those of the positions of dimension 0
 * whose coordinate's rows meet the chunk.  A slice's coordinates ascend, so they are one interval; a list's are not,
 * and the gather then walks all of them, skipping the positions that miss the chunk. */
static void osel_slabs(const B2OSel* s, long long w0, long long w1, long long ts, long long* g0, long long* g1) {
  long long jlo = 0, jhi = s->ext[0];
  if (!s->list[0]) {                     /* rows [clo, chi) meet the chunk */
    const long long clo = w0 / s->stride[0], chi = (w1 + s->stride[0] - 1) / s->stride[0];
    jlo = clo <= s->start[0] ? 0 : (clo - s->start[0] + s->step[0] - 1) / s->step[0];
    jhi = chi <= s->start[0] ? 0 : (chi - s->start[0] + s->step[0] - 1) / s->step[0];
    if (jhi > s->ext[0]) jhi = s->ext[0];
    if (jlo > jhi) jlo = jhi;
  }
  *g0 = jlo * s->slab * ts; *g1 = jhi * s->slab * ts;
}

/* An index selection of the array a frame holds, in items of chunk 0's typesize: one launch checks the list entries
 * and flags the chunks that hold a selected item, read back with one sync; then each flagged chunk, in ascending
 * order, writes the selected items it holds by the chunk path, and the first failure decides the result.  A host dest
 * is staged in device memory and copied out once. */
long long blosc_b200_frame_getoindex(const void* frame, size_t framesize, int ndim, const int64_t* shape,
                                     const int64_t* start, const int64_t* stop, const int64_t* step,
                                     const int64_t* const* index, const int64_t* nindex, void* dest) {
  int64_t st[B2_BOX_MAXDIM], sp[B2_BOX_MAXDIM], t[B2_BOX_MAXDIM];
  size_t c;
  b2_frame f;
  long long nitems = 0, count = 0, ts, ipc, nbytes, got = 0, result = -1;
  int dest_dev, rc;
  B2OSel sel;
  b2_ws* w;
  uint8_t *d_dst, *head = NULL;
  if (ndim < 1 || ndim > B2_BOX_MAXDIM || !osel_any(ndim, index))
    return blosc_b200_frame_getslice_step(frame, framesize, ndim, shape, start, stop, step, dest);
  if (!backend_ready()) return -1;
  if (osel_geometry(ndim, shape, start, stop, step, index, nindex, frame, dest, st, sp, t, &nitems, &count)) return -1;
  rc = frame_open_items(frame, framesize, &f);
  if (rc == -2)
    fprintf(stderr, "blosc_b200: chunk 0's typesize %lld does not divide the frame's chunksize\n", (long long)f.typesize);
  if (rc) return -1;
  ts = (long long)f.typesize; ipc = (long long)f.ipc;
  dest_dev = b2_ptr_is_device(dest);
  if (box_nbytes(nitems, ts, (unsigned long long)f.nbytes) || osel_nbytes(count, ts)) { free(f.off); return -1; }
  if (count == 0) { free(f.off); return 0; }
  nbytes = count * ts;
  if (!(w = ws_acquire())) { free(f.off); return -1; }
  do {
    OIndexPlanArgs fa;
    if (!(d_dst = stage_dest(&w->fstage, dest, dest_dev, (size_t)nbytes))) break;
    if (osel_build(w, ndim, shape, st, sp, t, index, nindex, &sel)) break;
    /* the scratch in w->fplan, which the chunk plans leave alone: the first bad entry (all ones), then the chunks' flags
     * (zeroed) */
    if (buf_ensure(&w->fplan, 16 + 4 * f.nchunks) || b2_memset_dev(w->fplan.p, 0, 16 + 4 * f.nchunks, w->stream) ||
        b2_memset_dev(w->fplan.p, 0xff, 8, w->stream))
      break;
    memset(&fa, 0, sizeof fa);
    fa.sel = sel; fa.check = 1; fa.r1 = sel.nruns; fa.ipc = ipc;
    fa.bad = (unsigned long long*)w->fplan.p; fa.touched = (int*)((uint8_t*)w->fplan.p + 16);
    if (b2_launch_oindex_plan(&fa, w->stream)) break;
    if (!(head = (uint8_t*)malloc(16 + 4 * f.nchunks)) || d2h_any(w, head, w->fplan.p, 16 + 4 * f.nchunks)) break;
    if (*(unsigned long long*)head != ~0ull) { osel_bad_entry(w, &sel, *(unsigned long long*)head); break; }
    for (c = 0; c < f.nchunks; c++) {
      const long long w0 = (long long)c * ipc, w1 = w0 + ipc < nitems ? w0 + ipc : nitems;
      long long g0, g1;
      b2_hdr h;
      int codec = 0;
      if (!((int*)(head + 16))[c]) continue;                               /* no selected item in this chunk */
      got = frame_chunk_header(w, frame, &f, c, &h, &codec);
      if (got < 0) break;
      if (got || h.nbytes != (w1 - w0) * ts) {
        fprintf(stderr, "blosc_b200: chunk %zu holds %d items of %d bytes, not the frame's %lld of %lld\n", c,
                h.nbytes / h.typesize, h.typesize, w1 - w0, ts);
        got = -1;
        break;
      }
      osel_slabs(&sel, w0, w1, ts, &g0, &g1);
      got = oindex_chunk(w, (const uint8_t*)frame + f.off[c], f.dev, &h, codec, &sel, 1, w0, g0, g1, d_dst);
      if (got < 0) break;
    }
    if (c < f.nchunks) { result = got; break; }
    if (!dest_dev && d2h_any(w, dest, d_dst, (size_t)nbytes)) break;
    result = nbytes;
  } while (0);
  ws_release(w);
  free(head);
  free(f.off);
  return result;
}

/* ------------------------------------------------------------------------- */
/* boxes of arrays stored as a grid of chunks (blosc_b200_grid_getslice)      */
/* ------------------------------------------------------------------------- */
/* zarr v2, the HDF5 blosc filter and PyTables store an N-d array as a regular grid of equally shaped chunks, each one
 * Blosc-1 buffer holding its sub-array in C order (edge chunks at full shape, their padding never read).  The chunks a
 * selection touches follow from the geometry alone: per dimension, the chunk indices that hold a selected coordinate,
 * and their product in C order.  A touched chunk's part is two boxes with the same extents (PlacedGatherArgs): one in
 * the chunk's coordinates, which plans and decodes the chunk as getslice_step does, and one in the output's, where the
 * placed gather writes the part directly.  A missing chunk is one placed fill.  Touched chunks are taken in ascending
 * order by up to BLOSC_B200_FRAME_WORKERS threads, each with its own workspace and stream; the parts are disjoint in
 * dest, so they are written without ordering. */
typedef struct {
  pthread_mutex_t mu;
  int ndim, dev, failed, err;
  long long next, ntouched, failed_at;     /* the next touched chunk to take; the lowest failing one */
  const int64_t *chunkshape, *start, *step;
  int64_t shape[B2_BOX_MAXDIM], n[B2_BOX_MAXDIM];  /* the array's shape and the output's */
  long long itemsize, chunk_items, out_items;
  long long* list[B2_BOX_MAXDIM];          /* the chunk indices of dimension k that hold a selected coordinate */
  long long nlist[B2_BOX_MAXDIM];
  const void** src;                        /* [ntouched] the touched chunks' table entries, in grid C order */
  uint8_t* src_dev;                        /* [ntouched] which of them are device memory */
  const uint8_t* fill;                     /* the fill pattern in device memory, or NULL for zeros */
  uint8_t* d_dst;
} b2_grid_job;

/* The checks of grid_getslice that need no chunk: getslice_step's on the shape, the chunk shape, the item size and a
 * chunk's bytes (*chunk_items: the items of one chunk).  -1 with a message when one fails. */
static int grid_geometry(int ndim, const int64_t* shape, const int64_t* chunkshape, size_t itemsize,
                         const int64_t* start, const int64_t* stop, const int64_t* step, long long* chunk_items) {
  long long nitems = 0, items = 1;
  int k;
  if (box_geometry(ndim, shape, start, stop, &nitems) || box_steps(ndim, step)) return -1;
  if (itemsize < 1) { fprintf(stderr, "blosc_b200: itemsize is 0\n"); return -1; }
  for (k = 0; k < ndim; k++)
    if (chunkshape[k] < 1) {
      fprintf(stderr, "blosc_b200: chunkshape[%d] = %lld is not >= 1\n", k, (long long)chunkshape[k]);
      return -1;
    }
  for (k = 0; k < ndim && items <= BLOSC_MAX_BUFFERSIZE; k++)
    items = chunkshape[k] > BLOSC_MAX_BUFFERSIZE ? (long long)BLOSC_MAX_BUFFERSIZE + 1 : items * chunkshape[k];
  if (items > BLOSC_MAX_BUFFERSIZE || itemsize > (size_t)(BLOSC_MAX_BUFFERSIZE / items)) {
    fprintf(stderr, "blosc_b200: a chunk of the chunk shape and %zu-byte items is larger than %d bytes\n", itemsize,
            BLOSC_MAX_BUFFERSIZE);
    return -1;
  }
  *chunk_items = items;
  return 0;
}

/* The first selected coordinate of dimension k at or after `org` and below `lim`, or -1 when there is none */
static long long grid_first(const b2_grid_job* j, int k, long long org, long long lim) {
  const long long s = j->start[k], t = j->step[k], d = org - s;
  const long long q = d <= 0 ? 0 : d / t + (d % t != 0);
  return q < j->n[k] && s + q * t < lim ? s + q * t : -1;      /* q < n: s + q * t is a selected coordinate */
}

/* The per-dimension lists of touched chunk indices, ascending: the chunks of the selected coordinates, or the chunks of
 * the selection's span that hold one, whichever is fewer to walk.  Returns the number of touched chunks, or -1. */
static long long grid_lists(b2_grid_job* j) {
  long long total = 1;
  int k;
  for (k = 0; k < j->ndim; k++) {
    const long long cs = j->chunkshape[k], t = j->step[k], first = j->start[k], last = first + (j->n[k] - 1) * t;
    const long long c0 = first / cs, c1 = last / cs;
    long long i, c, m = 0;
    if (!(j->list[k] = (long long*)malloc(8 * (size_t)(j->n[k] < c1 - c0 + 1 ? j->n[k] : c1 - c0 + 1)))) return -1;
    if (j->n[k] < c1 - c0 + 1) {
      for (i = 0; i < j->n[k]; i++)
        if (m == 0 || j->list[k][m - 1] != (first + i * t) / cs) j->list[k][m++] = (first + i * t) / cs;
    } else {
      for (c = c0; c <= c1; c++) {
        const long long org = c * cs, lim = cs < j->shape[k] - org ? org + cs : j->shape[k];
        if (grid_first(j, k, org, lim) >= 0) j->list[k][m++] = c;
      }
    }
    j->nlist[k] = m;
    total *= m;                          /* at most the grid's chunks, which the caller's table holds */
  }
  return total;
}

/* The grid coordinates of touched chunk `t` (its position in C order of the lists' product), and its index in the
 * chunk table */
static long long grid_coords(const b2_grid_job* j, long long t, long long* c) {
  long long g = 0, gs = 1;
  int k;
  for (k = j->ndim - 1; k >= 0; k--) {
    c[k] = j->list[k][t % j->nlist[k]];
    t /= j->nlist[k];
    g += c[k] * gs;
    gs *= (j->shape[k] - 1) / j->chunkshape[k] + 1;
  }
  return g;
}

/* The part of the chunk at grid coordinates c, as the box in the chunk's coordinates and the box in the output's */
static void grid_part(const b2_grid_job* j, const long long* c, B2Box* box, B2Box* out) {
  int64_t lst[B2_BOX_MAXDIM], lsp[B2_BOX_MAXDIM], ost[B2_BOX_MAXDIM], osp[B2_BOX_MAXDIM];
  int k;
  for (k = 0; k < j->ndim; k++) {
    const long long cs = j->chunkshape[k], t = j->step[k], org = c[k] * cs;
    const long long lim = cs < j->shape[k] - org ? org + cs : j->shape[k];
    const long long last = j->start[k] + (j->n[k] - 1) * t, hi = last < lim - 1 ? last : lim - 1;
    const long long f = grid_first(j, k, org, lim), l = f + (hi - f) / t * t;
    lst[k] = f - org; lsp[k] = l - org + 1;
    ost[k] = (f - j->start[k]) / t; osp[k] = ost[k] + (l - f) / t + 1;
  }
  box_build(j->ndim, j->chunkshape, lst, lsp, j->step, j->chunk_items, box);
  box_build(j->ndim, j->n, ost, osp, NULL, j->out_items, out);
}

static long long grid_take(b2_grid_job* j) {
  long long t;
  pthread_mutex_lock(&j->mu);
  t = !j->failed && j->next < j->ntouched ? j->next++ : -1;
  pthread_mutex_unlock(&j->mu);
  return t;
}

/* Touched chunk t failed with rc: the lowest failing chunk decides the result.  Chunks are taken in ascending order,
 * so every chunk below t was taken already and finishes; none above it is taken from now on. */
static void grid_fail(b2_grid_job* j, long long t, int rc) {
  pthread_mutex_lock(&j->mu);
  if (t < j->failed_at) { j->failed_at = t; j->err = rc; }
  j->failed = 1;
  pthread_mutex_unlock(&j->mu);
}

/* Touched chunk t, present at grid coordinates c: its header checked with blosc_getitem's codes and its bytes against
 * the chunk shape, its touched blocks planned at the caller's item size (the header's typesize only unshuffles) and
 * decoded, and its part gathered into place.  Returns 0, blosc_getitem's or blosc_d's code, or -1. */
static int grid_chunk(const b2_grid_job* j, b2_ws* w, long long t, const long long* c, const B2Box* box,
                      const B2Box* out) {
  const void* src = j->src[t];
  const int src_dev = j->src_dev[t];
  GetitemsPlan rec = {0};
  PlacedGatherArgs ga;
  b2_hdr h;
  int codec = 0, rc, k;
  if ((rc = getitem_header(w, src, src_dev, -1, &h, &codec))) return rc;
  if ((long long)h.nbytes != j->chunk_items * j->itemsize) {
    char at[B2_BOX_MAXDIM * 24];
    size_t o = 0;
    for (k = 0; k < j->ndim; k++) o += (size_t)snprintf(at + o, sizeof at - o, k ? ", %lld" : "%lld", c[k]);
    fprintf(stderr, "blosc_b200: chunk (%s) holds %d bytes, not the %lld of its shape\n", at, h.nbytes,
            j->chunk_items * j->itemsize);
    return -1;
  }
  memset(&ga, 0, sizeof ga);
  ga.box = *box; ga.out = *out; ga.run = box->run < out->run ? box->run : out->run;
  ga.total = out->count * j->itemsize; ga.itemsize = j->itemsize; ga.blocksize = h.blocksize; ga.dst = j->d_dst;
  if (!((h.flags & BLOSC_MEMCPYED) && src_dev)) {            /* a memcpyed device chunk is read in place: no plan */
    BoxPlanArgs bp;
    bp.box = *box; bp.window = 0;
    if (!plan_scratch(w, &h, 0, 0, &bp.plan)) return -1;
    bp.plan.typesize = (int)j->itemsize;
    if (b2_launch_box_plan(&bp, w->stream) || read_plan(w, bp.plan.rec, &rec, sizeof rec)) return -1;
    ga.slot = bp.plan.slot;
  }
  if (touched_source(w, src, src_dev, &h, codec, rec.nlisted, rec.has_left, &ga.src, &ga.status)) return -1;
  if (b2_launch_placed_gather(&ga, w->stream)) { ws_reset_counters(w); return -1; }
  return read_verdict(w, ga.status);
}

/* A worker: takes touched chunks until none is left or one has failed.  A missing chunk is one fill launch, with no
 * sync; the worker's stream is drained once at the end. */
static void grid_work(b2_grid_job* j, b2_ws* w) {
  long long t, c[B2_BOX_MAXDIM];
  B2Box box, out;
  while ((t = grid_take(j)) >= 0) {
    int rc = 0;
    grid_coords(j, t, c);
    grid_part(j, c, &box, &out);
    if (j->src[t]) rc = grid_chunk(j, w, t, c, &box, &out);
    else {
      PlacedGatherArgs fa;
      memset(&fa, 0, sizeof fa);
      fa.out = out; fa.run = out.run; fa.total = out.count * j->itemsize; fa.itemsize = j->itemsize;
      fa.fill = j->fill; fa.dst = j->d_dst;
      if (b2_launch_placed_fill(&fa, w->stream)) rc = -1;
    }
    if (rc < 0) grid_fail(j, t, rc);
  }
  if (b2_stream_sync(w->stream)) grid_fail(j, j->ntouched, -1);
}

/* A worker thread beside the caller's: on the call's device, with a workspace of its own when one is free (else the
 * other workers take its share) */
static void* grid_helper(void* arg) {
  b2_grid_job* j = (b2_grid_job*)arg;
  b2_ws* w;
  b2_set_device(j->dev);
  if (!(w = ws_acquire_if(0))) return NULL;
  grid_work(j, w);
  ws_release(w);
  return NULL;
}

long long blosc_b200_grid_getslice(int ndim, const int64_t* shape, const int64_t* chunkshape, size_t itemsize,
                                   const void* const* chunks, const void* fill, const int64_t* start,
                                   const int64_t* stop, const int64_t* step, void* dest) {
  static const int64_t ones[B2_BOX_MAXDIM] = {1, 1, 1, 1, 1, 1, 1, 1};
  pthread_t th[B2_FRAME_MAX_WORKERS];
  b2_grid_job j;
  b2_ws* w = NULL;
  long long t, c[B2_BOX_MAXDIM], chunk_items = 0, nbytes = 0, result = -1;
  int k, dest_dev, dev, old_dev = 0, started = 0, missing = 0, workers;
  if (grid_geometry(ndim, shape, chunkshape, itemsize, start, stop, step, &chunk_items)) return -1;
  if (box_empty(ndim, start, stop)) return 0;
  memset(&j, 0, sizeof j);
  j.chunk_items = chunk_items; j.ndim = ndim; j.chunkshape = chunkshape; j.start = start; j.step = step ? step : ones;
  j.itemsize = (long long)itemsize; j.out_items = 1;
  for (k = 0; k < ndim; k++) {
    j.shape[k] = shape[k];
    j.n[k] = (stop[k] - start[k] - 1) / j.step[k] + 1;
    j.out_items *= j.n[k];                 /* at most the array's items */
  }
  if (j.out_items > LLONG_MAX / j.itemsize) {
    fprintf(stderr, "blosc_b200: the output of %lld items of %zu bytes overflows int64\n", j.out_items, itemsize);
    return -1;
  }
  nbytes = j.out_items * j.itemsize;
  if (!chunks) { fprintf(stderr, "blosc_b200: chunks is NULL\n"); return -1; }
  do {
    if ((j.ntouched = grid_lists(&j)) < 0) break;
    j.src = (const void**)malloc(sizeof(void*) * (size_t)j.ntouched);
    j.src_dev = (uint8_t*)malloc((size_t)j.ntouched);
    if (!j.src || !j.src_dev) break;
    for (t = 0; t < j.ntouched; t++) {                 /* the table entries of touched chunks, and no other */
      j.src[t] = chunks[grid_coords(&j, t, c)];
      j.src_dev[t] = j.src[t] && b2_ptr_is_device(j.src[t]);
      missing |= !j.src[t];
    }
    /* the call runs on dest's device, else on the first device chunk's, else on the current one */
    dest_dev = b2_ptr_is_device(dest);
    dev = dest_dev ? b2_ptr_device(dest) : -1;
    for (t = 0; t < j.ntouched && dev < 0; t++) if (j.src_dev[t]) dev = b2_ptr_device(j.src[t]);
    if (dev < 0) dev = b2_get_device();
    for (t = 0; t < j.ntouched; t++)
      if (j.src_dev[t] && b2_ptr_device(j.src[t]) != dev) break;
    if (t < j.ntouched) {
      fprintf(stderr, "blosc_b200: chunk %lld of the table is on device %d, not on device %d where the call runs\n",
              grid_coords(&j, t, c), b2_ptr_device(j.src[t]), dev);
      break;
    }
    if (!backend_ready()) break;
    old_dev = b2_get_device();
    if (dev != old_dev && b2_set_device(dev)) break;
    if ((w = ws_acquire())) {
      do {
        if (!(j.d_dst = stage_dest(&w->fstage, dest, dest_dev, (size_t)nbytes))) break;
        if (missing && fill) {
          if (buf_ensure(&w->fplan, itemsize) || copy_any(w->fplan.p, 1, fill, b2_ptr_is_device(fill), itemsize, w->stream))
            break;
          j.fill = (const uint8_t*)w->fplan.p;
        }
        pthread_mutex_init(&j.mu, NULL);
        j.dev = dev; j.failed_at = LLONG_MAX;
        workers = frame_workers(j.ntouched < B2_FRAME_MAX_WORKERS ? (int)j.ntouched : B2_FRAME_MAX_WORKERS);
        for (k = 1; k < workers; k++) {
          if (pthread_create(&th[started], NULL, grid_helper, &j) != 0) break;
          started++;
        }
        grid_work(&j, w);                              /* the calling thread is a worker too */
        for (k = 0; k < started; k++) pthread_join(th[k], NULL);
        pthread_mutex_destroy(&j.mu);
        if (j.failed) { result = j.err; break; }
        if (!dest_dev && d2h_any(w, dest, j.d_dst, (size_t)nbytes)) break;
        result = nbytes;
      } while (0);
      ws_release(w);
    }
    if (dev != old_dev) b2_set_device(old_dev);
  } while (0);
  for (k = 0; k < ndim; k++) free(j.list[k]);
  free(j.src); free(j.src_dev);
  return result;
}

/* ------------------------------------------------------------------------- */
/* writing arrays as a grid of chunks (blosc_b200_grid_compress)              */
/* ------------------------------------------------------------------------- */
/* The write side of the grid above: every chunk of the array's grid is compressed by the frame's machinery -- workers
 * from BLOSC_B200_FRAME_WORKERS take chunks in order, each through compress_impl on its own workspace and stream, and
 * frame_place lays them out back to back in grid C order whatever the worker count.  A chunk's input is its sub-array
 * at full chunk shape: two step-1 boxes with the same extents, one in the array's coordinates and one in the chunk's.
 * From a device array, compress_impl packs it into its workspace with grid_pack_kernel (after one placed_fill_kernel
 * over an edge chunk), so the array is never copied whole; from a host array, the worker gathers it run by run into
 * a pinned buffer of its own, which compress_impl stages as any host input. */

size_t blosc_b200_grid_bound(int ndim, const int64_t* shape, const int64_t* chunkshape, size_t itemsize) {
  size_t n = 1, items = 1;
  int k;
  if (ndim < 1 || ndim > B2_BOX_MAXDIM || itemsize < 1) return 0;
  for (k = 0; k < ndim; k++) {
    size_t g;
    if (shape[k] < 0 || chunkshape[k] < 1) return 0;
    g = (size_t)(shape[k] / chunkshape[k] + (shape[k] % chunkshape[k] != 0));
    if ((g && n > SIZE_MAX / g) || items > SIZE_MAX / (size_t)chunkshape[k]) return 0;
    n *= g;
    items *= (size_t)chunkshape[k];
  }
  if (items > (SIZE_MAX - BLOSC_MAX_OVERHEAD) / itemsize) return 0;
  items = items * itemsize + BLOSC_MAX_OVERHEAD;
  return n && items > SIZE_MAX / n ? 0 : n * items;
}

/* Chunk g of the grid: its sub-array as the box in the array's coordinates and the box in the chunk's.  Returns 1 for
 * an edge chunk, which holds padding. */
static int grid_chunk_boxes(const b2_frame_job* j, long long g, B2Box* box, B2Box* out) {
  int64_t org[B2_BOX_MAXDIM], lim[B2_BOX_MAXDIM], ext[B2_BOX_MAXDIM];
  int k, edge = 0;
  for (k = j->ndim - 1; k >= 0; k--) {
    const long long cs = j->chunkshape[k], n = (j->shape[k] - 1) / cs + 1;
    org[k] = g % n * cs;
    lim[k] = cs < j->shape[k] - org[k] ? org[k] + cs : j->shape[k];
    ext[k] = lim[k] - org[k];
    edge |= ext[k] < cs;
    g /= n;
  }
  box_build(j->ndim, j->shape, org, lim, NULL, j->nitems, box);
  box_build(j->ndim, j->chunkshape, g_box_origin, ext, NULL, j->chunk_items, out);
  return edge;
}

/* n bytes of whole items, each the itemsize-byte pattern fill (NULL: zeros) */
static void pattern_fill(uint8_t* p, size_t n, const uint8_t* fill, size_t ts) {
  size_t have = ts < n ? ts : n;
  if (!fill) { memset(p, 0, n); return; }
  memcpy(p, fill, have);
  for (; have < n; have *= 2) memcpy(p + have, p, have < n - have ? have : n - have);
}

/* n bytes of whole items all equal to the pattern fill (NULL: zeros) */
static int pattern_equal(const uint8_t* p, size_t n, const uint8_t* fill, size_t ts) {
  size_t x;
  uint8_t d = 0;
  if (!fill) { for (x = 0; x < n; x++) d |= p[x]; return d == 0; }
  for (x = 0; x < n; x += ts) if (memcmp(p + x, fill, ts)) return 0;
  return 1;
}

/* A host array: chunk a's sub-array gathered run by run into `host`, over the fill pattern in an edge chunk.  Returns
 * 1 when skip_fill is asked and every gathered byte is the fill pattern (the chunk is then not written), else 0. */
static int grid_gather_host(const b2_frame_job* j, const GridPackArgs* a, int edge, uint8_t* host) {
  const long long ts = j->itemsize, runb = a->run * ts;
  long long q;
  int same = j->skip_fill;
  if (edge) pattern_fill(host, (size_t)(j->chunk_items * ts), j->fill, (size_t)ts);
  for (q = 0; q < a->box.count; q += a->run) {
    const uint8_t* from = j->src + b2_box_unrank(&a->box, q, 0) * ts;
    memcpy(host + b2_box_unrank(&a->out, q, 0) * ts, from, (size_t)runb);
    if (same) same = pattern_equal(from, (size_t)runb, j->fill, (size_t)ts);
  }
  return same;
}

static void* grid_compress_worker(void* arg) {
  b2_frame_job* j = (b2_frame_job*)arg;
  const long long cb = j->chunk_items * j->itemsize;
  const int64_t items = j->chunk_items;
  B2Box whole;                               /* the whole chunk, which an edge chunk's fill covers */
  uint8_t* host = NULL;
  int i, failed;
  b2_set_device(j->dev);
  box_build(1, &items, g_box_origin, &items, NULL, items, &whole);
  if (!j->src_dev) {
    void* p = NULL;
    if (b2_pinned_alloc(&p, (size_t)cb) == 0) host = (uint8_t*)p;
  }
  while ((i = frame_take(j, &failed)) >= 0) {
    b2_place pl;
    b2_pack pk;
    int rc = -1, edge;
    pl.job = j; pl.index = i; pl.placed = 0; pl.many = j->workers > 1;
    memset(&pk, 0, sizeof pk);
    if (!failed && (j->src_dev || host)) {
      edge = grid_chunk_boxes(j, i, &pk.pack.box, &pk.pack.out);
      pk.pack.run = pk.pack.box.run < pk.pack.out.run ? pk.pack.box.run : pk.pack.out.run;
      pk.pack.total = pk.pack.box.count * j->itemsize; pk.pack.itemsize = j->itemsize;
      pk.pack.src = j->src; pk.pack.fill = j->fill;
      pk.skip = j->skip_fill;
      if (j->src_dev) {
        if (edge) {
          pk.pad.out = whole; pk.pad.run = whole.run; pk.pad.total = cb; pk.pad.itemsize = j->itemsize;
          pk.pad.fill = j->fill;
        }
        rc = compress_impl(j->clevel, j->doshuffle, j->typesize, (size_t)cb, NULL, NULL, (size_t)cb + BLOSC_MAX_OVERHEAD,
                           j->compressor, j->blocksize, j->nthreads, &pl, j->dest_dev, &pk);
      } else if (!(pk.skipped = grid_gather_host(j, &pk.pack, edge, host)))
        rc = compress_impl(j->clevel, j->doshuffle, j->typesize, (size_t)cb, host, NULL, (size_t)cb + BLOSC_MAX_OVERHEAD,
                           j->compressor, j->blocksize, j->nthreads, &pl, j->dest_dev, NULL);
      if (pk.skipped) {                      /* its turn in the ordered commit, with no bytes: not "does not fit" */
        frame_place(&pl, 0);
        rc = 1;
      }
    }
    if (!pl.placed) frame_place(&pl, -1);
    if (rc <= 0 && !failed) frame_fail(j, rc);
  }
  if (host) b2_pinned_free(host);
  return NULL;
}

long long blosc_b200_grid_compress(int clevel, int doshuffle, size_t typesize, const char* compressor, size_t blocksize,
                                   int numinternalthreads, int ndim, const int64_t* shape, const int64_t* chunkshape,
                                   size_t itemsize, const void* src, const void* fill, int skip_fill, void* dest,
                                   size_t destsize, int64_t* offsets) {
  b2_frame_job j;
  void* d_fill = NULL;
  long long chunk_items = 0, nchunks = 1, nitems = 1;
  int k, rc, src_dev, dest_dev, dev, old_dev;
  if (clevel < 0 || clevel > 9) return -10;                       /* the chunk API's codes */
  if (doshuffle != 0 && doshuffle != 1 && doshuffle != 2) return -10;
  if (typesize == 0) return -10;
  if (!compressor || blosc_compname_to_compcode(compressor) < 0) return -5;
  if (grid_geometry(ndim, shape, chunkshape, itemsize, g_box_origin, shape, NULL, &chunk_items)) return -1;
  for (k = 0; k < ndim; k++) {
    const long long g = shape[k] / chunkshape[k] + (shape[k] % chunkshape[k] != 0);
    nitems *= shape[k];                                           /* box_geometry checked the product */
    if (g == 0) nchunks = 0;
    else if (nchunks > 0) nchunks = nchunks > (INT_MAX / 2) / g ? (long long)INT_MAX : nchunks * g;
  }
  if (nchunks > INT_MAX / 2) {
    fprintf(stderr, "blosc_b200: the grid has more than %d chunks\n", INT_MAX / 2);
    return -1;
  }
  if (nchunks == 0) {
    if (offsets) offsets[0] = 0;
    return 0;
  }
  if (!src || !offsets) { fprintf(stderr, "blosc_b200: %s is NULL\n", src ? "offsets" : "src"); return -1; }
  /* the call runs on dest's device when dest is device memory, else on src's, else on the current one */
  src_dev = b2_ptr_is_device(src);
  dest_dev = b2_ptr_is_device(dest);
  dev = dest_dev ? b2_ptr_device(dest) : src_dev ? b2_ptr_device(src) : b2_get_device();
  if (src_dev && b2_ptr_device(src) != dev) {
    fprintf(stderr, "blosc_b200: src is on device %d, not on device %d where the call runs\n", b2_ptr_device(src), dev);
    return -1;
  }
  if (!backend_ready()) return -1;
  old_dev = b2_get_device();
  if (dev != old_dev && b2_set_device(dev)) return -1;
  memset(&j, 0, sizeof j);
  j.nchunks = (int)nchunks; j.workers = frame_workers((int)nchunks); j.dest_dev = dest_dev;
  j.clevel = clevel; j.doshuffle = doshuffle; j.nthreads = numinternalthreads;
  j.typesize = typesize; j.blocksize = blocksize; j.compressor = compressor;
  j.destsize = destsize; j.cursor = 0; j.src = (const uint8_t*)src; j.dest = (uint8_t*)dest;
  j.offsets = (uint64_t*)offsets;
  j.ndim = ndim; j.src_dev = src_dev; j.skip_fill = skip_fill != 0;
  j.itemsize = (long long)itemsize; j.nitems = nitems; j.chunk_items = chunk_items;
  for (k = 0; k < ndim; k++) { j.shape[k] = shape[k]; j.chunkshape[k] = chunkshape[k]; }
  j.fill = (const uint8_t*)fill;
  rc = 0;
  if (src_dev && fill) {                     /* the pack reads the pattern on the device */
    if (b2_dev_alloc(&d_fill, itemsize) || copy_some(d_fill, 1, fill, 0, itemsize)) rc = -1;
    j.fill = (const uint8_t*)d_fill;
  }
  if (rc == 0) rc = frame_run(&j, grid_compress_worker);
  else j.err = -1;
  if (d_fill) b2_dev_free(d_fill);
  if (dev != old_dev) b2_set_device(old_dev);
  if (rc) return j.err ? j.err : (j.failed ? 0 : -1);            /* 0: does not fit in destsize, as frame_compress */
  offsets[nchunks] = (int64_t)j.cursor;
  return (long long)j.cursor;
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

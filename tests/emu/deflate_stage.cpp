/*
 * deflate_stage.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * The DEFLATE entropy stage (dz_stream, csrc/dev_deflate.cuh) on its own, inside the lock-step SIMT emulator, for
 * tests/test_zlib_encode.py.  The test builds it into a small library of its own with simt_emu.cpp; the product
 * never includes this file.
 */
#include "simt_emu.h"

#include "../../c-blosc_b200/csrc/dev_deflate.cuh"

extern "C" {

/* one warp runs dz_stream on src[0, n) from sequence records the caller chose, in zse_parse_lane's format with
 * offsets <= 32768: rec[k * ZE_SEG_RECS + r] for segment k, cnt[k] records each.  Scratch of 2n bytes (the stream's
 * part of prev[]), out n bytes, FLEVEL 2.  Returns the zlib stream's size, or n for "stored". */
int emu_deflate_stream(const unsigned char* src, int n, const unsigned int* rec, const unsigned int* cnt, unsigned char* out) {
  int result = 0;
  DzSm* S = new DzSm;
  unsigned char* scratch = (unsigned char*)malloc(2 * (size_t)n + 8);
  simt::launch(simt::Dim3(1), simt::Dim3(32), 0, [&] {
    const int r = dz_stream(*S, src, n, rec, cnt, scratch, out, 2);
    if ((threadIdx.x & 31) == 11) result = r;
  });
  free(scratch);
  delete S;
  return result;
}

}  // extern "C"

/*
 * snappy_stage.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * The emulated library (backend_emu.cpp, included whole so that this file shares its translation unit and the
 * emulator-only counters of dev_snappy.cuh / dev_chunk.cuh), plus entry points that drive the snappy code on its own,
 * for tests/test_snappy.py.  The test links it with the host code (blosc_b200.c) and simt_emu.cpp into a library of
 * its own; the product never includes this file.
 */
#include "backend_emu.cpp"

extern "C" {

/* one stream through the decoder (one warp, LZ4D_SMEM of shared memory); returns cap or -1 */
int emu_snappy_decode(const unsigned char* src, int csize, unsigned char* dst, int cap) {
  int result = 0;
  g_sn_fail_line = 0;
  simt::launch(simt::Dim3(1), simt::Dim3(32), LZ4D_SMEM, [&] {
    const int r = snappy_decode_warp(src, csize, dst, cap, simt::g_dynsmem);
    if ((threadIdx.x & 31) == 21) result = r;
  });
  return result;
}
/* the decoder's first refusing line in the last call */
int emu_snappy_fail_line(void) { return g_sn_fail_line; }
/* the decoder's branch counters (SN_H_*), copied out and cleared */
int emu_snappy_hits(long long* h) { for (int i = 0; i < SN_NHIT; i++) { h[i] = g_sn_hit[i]; g_sn_hit[i] = 0; } return SN_NHIT; }

/* the stream writer alone (sn_stream) on records the caller chose in zse_parse_lane's format: rec[k * ZE_SEG_RECS + r]
 * for segment k, cnt[k] records each.  Scratch of 2n (+8) bytes as in senc_body, out n bytes.  Returns the stream
 * size, or n for "raw" (nothing written). */
int emu_snappy_stream(const unsigned char* src, int n, const unsigned int* rec, const unsigned int* cnt, unsigned char* out) {
  int result = 0;
  unsigned char* scratch = (unsigned char*)malloc(2 * (size_t)n + 8);
  simt::launch(simt::Dim3(1), simt::Dim3(32), 0, [&] {
    const int r = sn_stream(src, n, rec, cnt, scratch, out);
    if ((threadIdx.x & 31) == 5) result = r;
  });
  free(scratch);
  return result;
}

/* the next snappy compress calls copy their stream sizes, as the maxout rule finds them, to buf[0, cap) (NULL: off) */
void emu_snappy_presizes(int* buf, int cap) { g_sn_presizes = buf; g_sn_presizes_cap = cap; }

}  // extern "C"

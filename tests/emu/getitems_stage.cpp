/*
 * getitems_stage.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * The emulated library (backend_emu.cpp, included whole) with its decode launcher wrapped, so that tests/test_getitems.py
 * can see what each decode launch covered: how many streams, and how many listed blocks (DecodeArgs.blocks).  The test
 * links it with the host code (blosc_b200.c) and simt_emu.cpp into a library of its own; the product never includes
 * this file.
 */
#define b2_launch_decode emu_base_launch_decode
#include "backend_emu.cpp"
#undef b2_launch_decode

static int g_last_decode_streams = 0, g_last_decode_blocks = 0;

extern "C" {

int b2_launch_decode(const DecodeArgs* a, b2_stream_t s) {
  g_last_decode_streams = a->map.nstreams;
  g_last_decode_blocks = a->blocks ? a->map.nfull + (a->map.leftover ? 1 : 0) : 0;
  return emu_base_launch_decode(a, s);
}

/* streams and listed blocks of the most recent decode launch (0 blocks: a contiguous range, no list) */
int emu_last_decode_streams(void) { return g_last_decode_streams; }
int emu_last_decode_blocks(void) { return g_last_decode_blocks; }
/* launches of backend_emu.cpp's launchers plus those of the gather launcher (dev_chunk.cuh) */
long long emu_launches_with_gather(void) { return g_launches + g_emu_gather_launches; }

}  // extern "C"

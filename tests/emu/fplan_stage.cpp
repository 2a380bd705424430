/*
 * fplan_stage.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * The emulated library (backend_emu.cpp, included whole) with its decode launcher wrapped, so that
 * tests/test_frame_getitems_device.py can count what a frame read launches: decode launches, gather launches and plan
 * launches (the chunk plan's and the frame plan's, dev_chunk.cuh).  The test links it with the host code
 * (blosc_b200.c) and simt_emu.cpp into a library of its own; the product never includes this file.
 */
#define b2_launch_decode emu_base_launch_decode
#include "backend_emu.cpp"
#undef b2_launch_decode

static long long g_decode_launches = 0;

extern "C" {

int b2_launch_decode(const DecodeArgs* a, b2_stream_t s) {
  if (a->map.nstreams > 0) g_decode_launches++;
  return emu_base_launch_decode(a, s);
}

/* launches so far: [0] decode, [1] gather, [2] plan */
void emu_frame_launches(long long* c) { c[0] = g_decode_launches; c[1] = g_emu_gather_launches; c[2] = g_emu_plan_launches; }

}  // extern "C"

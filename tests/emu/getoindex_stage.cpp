/*
 * getoindex_stage.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * The getslice_step stage (getslice_step_stage.cpp, included whole: the launch counters, the decode launch's listed
 * blocks, the pointer shim and the box gather's kernel choice) with the index-selection gather launcher wrapped, so
 * that tests/test_getoindex.py can see which chunks of a frame were gathered (by their item window), and with the
 * device-to-host copies and the stream syncs counted.  The test links it with the host code (blosc_b200.c) and
 * simt_emu.cpp into a library of its own; the product never includes this file.
 */
#define b2_launch_oindex_gather emu_base_launch_oindex_gather
#define b2_copy_d2h emu_base_copy_d2h
#define b2_stream_sync emu_base_stream_sync
#include "getslice_step_stage.cpp"
#undef b2_launch_oindex_gather
#undef b2_copy_d2h
#undef b2_stream_sync

#define EMU_MAX_WINDOWS 256
static long long g_windows[EMU_MAX_WINDOWS];
static int g_nwindows = 0, g_last_oindex_run = -1;
static long long g_d2h = 0, g_syncs = 0;

extern "C" {

int b2_launch_oindex_gather(const OIndexGatherArgs* a, b2_stream_t s) {
  if (g_nwindows < EMU_MAX_WINDOWS) g_windows[g_nwindows++] = a->clip ? a->window : -1;
  g_last_oindex_run = (int)a->sel.run;
  return emu_base_launch_oindex_gather(a, s);
}
int b2_copy_d2h(void* h, const void* d, size_t n, b2_stream_t s) { g_d2h++; return emu_base_copy_d2h(h, d, n, s); }
int b2_stream_sync(b2_stream_t s) { g_syncs++; return emu_base_stream_sync(s); }

/* the item windows of the index gathers since the last reset, in launch order (-1: a chunk call's, unclipped) */
void emu_oindex_reset(void) { g_nwindows = 0; g_last_oindex_run = -1; }
int emu_oindex_ngathers(void) { return g_nwindows; }
long long emu_oindex_window(int i) { return i < g_nwindows ? g_windows[i] : -2; }
/* the run, in items, of the most recent index gather (-1: none since the reset) */
int emu_oindex_last_run(void) { return g_last_oindex_run; }
/* device-to-host copies and stream syncs so far */
long long emu_d2h_copies(void) { return g_d2h; }
long long emu_syncs(void) { return g_syncs; }

}  // extern "C"

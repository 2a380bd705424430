/*
 * getslice_step_stage.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * The getslice stage (getslice_stage.cpp, included whole: the launch counters, the decode launch's listed blocks and
 * the pointer shim) with its box gather launcher wrapped, so that tests/test_getslice_step.py can see whether a box
 * read launched the stepped or the step-1 kernels, and the run length they gathered.  The test links it with
 * box_step_shim.c and simt_emu.cpp into a library of its own; the product never includes this file.
 */
#define b2_launch_box_gather emu_base_launch_box_gather
#include "getslice_stage.cpp"
#undef b2_launch_box_gather

static int g_last_box_stepped = -1;
static long long g_last_box_run = -1;

extern "C" {

int b2_launch_box_gather(const BoxGatherArgs* a, b2_stream_t s) {
  g_last_box_stepped = a->box.stepped;
  g_last_box_run = a->box.run;
  return emu_base_launch_box_gather(a, s);
}

/* the box of the most recent box gather launch: its stepped flag (-1 before any) and its run in items */
int emu_last_box_stepped(void) { return g_last_box_stepped; }
long long emu_last_box_run(void) { return g_last_box_run; }

}  // extern "C"

/*
 * getslice_stage.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * The getitems stage (getitems_stage.cpp, included whole: the decode launch's listed blocks and the pointer shim) with
 * one more counter, so that tests/test_getslice.py can count every launch of a box read: those of backend_emu.cpp's
 * launchers, the gather launches and the plan launches (dev_chunk.cuh).  The test links it with the host code
 * (blosc_b200.c) and simt_emu.cpp into a library of its own; the product never includes this file.
 */
#include "getitems_stage.cpp"

extern "C" long long emu_all_launches(void) { return g_launches + g_emu_gather_launches + g_emu_plan_launches; }

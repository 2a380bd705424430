/*
 * lz4t_window_stage.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * The emulated library (backend_emu.cpp, included whole) plus the counters of the LZ4 team walker's chained windows
 * (dev_lz4.cuh, LZ4T_W_*), so that tests/test_lz4_team_window.py can see how many sequences its streams' windows took
 * and what ended them.  The test links it with the host code (blosc_b200.c) and simt_emu.cpp into a library of its
 * own; the product never includes this file.
 */
#include "backend_emu.cpp"

extern "C" {

/* totals since the library was loaded; returns their number */
int emu_lz4t_window_counters(long long* c) { for (int i = 0; i < LZ4T_W_N; i++) c[i] = g_dbg_lz4t_w[i]; return LZ4T_W_N; }

}  // extern "C"

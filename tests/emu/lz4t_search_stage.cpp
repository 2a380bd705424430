/*
 * lz4t_search_stage.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * The emulated library (backend_emu.cpp, included whole) plus the branch counters of the LZ4 team walker's search after
 * a chained miss (dev_lz4.cuh, LZ4T_S_*), so that tests/test_lz4_team_search.py can see which branches its streams
 * reached.  The test links it with the host code (blosc_b200.c) and simt_emu.cpp into a library of its own; the
 * product never includes this file.
 */
#include "backend_emu.cpp"

extern "C" {

/* totals since the library was loaded; returns their number */
int emu_lz4t_search_counters(long long* c) { for (int i = 0; i < LZ4T_S_N; i++) c[i] = g_dbg_lz4t_s[i]; return LZ4T_S_N; }

}  // extern "C"

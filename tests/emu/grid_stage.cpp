/*
 * grid_stage.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * The emulated library (backend_emu.cpp, included whole) with the launchers and the pointer test wrapped, so that
 * tests/test_grid_getslice.py can count a grid read's launches by kind, see the block list of every decode launch, and
 * place any set of buffers in device memory.  It wraps the same hooks as getslice_stage.cpp, but keeps every decode's
 * list rather than the last one's count and tests a set of device buffers rather than two, so it includes the backend
 * itself.  The counters take a lock: a grid read launches from several threads.  The test links it with the host code
 * (blosc_b200.c) and simt_emu.cpp into a library of its own; the product never includes this file.
 */
#define b2_launch_decode emu_base_launch_decode
#define b2_launch_filter emu_base_launch_filter
#define b2_ptr_is_device emu_base_ptr_is_device
#define b2_launch_placed_fill emu_base_launch_placed_fill
#include "backend_emu.cpp"
#undef b2_launch_decode
#undef b2_launch_filter
#undef b2_ptr_is_device
#undef b2_launch_placed_fill

#include <mutex>
#include <set>
#include <vector>

static std::mutex g_grid_mu;
static std::set<const void*> g_dev_set;
static std::vector<std::vector<int>> g_decode_lists;
static long long g_decodes = 0, g_filters = 0, g_fills = 0;

extern "C" {

int b2_launch_decode(const DecodeArgs* a, b2_stream_t s) {
  {
    std::lock_guard<std::mutex> lk(g_grid_mu);
    const int n = a->map.nfull + (a->map.leftover ? 1 : 0);
    std::vector<int> list;
    for (int i = 0; i < n; i++) list.push_back(a->blocks ? a->blocks[i] : a->map.first_block + i);
    g_decode_lists.push_back(list);
    g_decodes++;
  }
  return emu_base_launch_decode(a, s);
}
int b2_launch_filter(const FilterArgs* a, b2_stream_t s) {
  { std::lock_guard<std::mutex> lk(g_grid_mu); g_filters++; }
  return emu_base_launch_filter(a, s);
}
int b2_launch_placed_fill(const PlacedGatherArgs* a, b2_stream_t s) {
  { std::lock_guard<std::mutex> lk(g_grid_mu); g_fills++; }
  return emu_base_launch_placed_fill(a, s);
}

/* these n addresses count as device memory (n = 0: none), on top of emu_set_all_device */
void emu_grid_set_device(const void* const* p, int n) {
  std::lock_guard<std::mutex> lk(g_grid_mu);
  g_dev_set.clear();
  for (int i = 0; i < n; i++) g_dev_set.insert(p[i]);
}
int b2_ptr_is_device(const void* p) {
  std::lock_guard<std::mutex> lk(g_grid_mu);
  return emu_base_ptr_is_device(p) || (p && g_dev_set.count(p));
}

/* launches since the last reset: c[0] decode, c[1] unfilter, c[2] plan, c[3] gather (the fills included), c[4] fill,
 * c[5] all of them */
void emu_grid_reset(void) {
  std::lock_guard<std::mutex> lk(g_grid_mu);
  g_decode_lists.clear();
  g_decodes = g_filters = g_fills = 0;
  g_emu_plan_launches = g_emu_gather_launches = 0;
  g_launches = 0;
}
void emu_grid_counts(long long* c) {
  std::lock_guard<std::mutex> lk(g_grid_mu);
  c[0] = g_decodes; c[1] = g_filters; c[2] = g_emu_plan_launches; c[3] = g_emu_gather_launches; c[4] = g_fills;
  c[5] = g_launches + g_emu_plan_launches + g_emu_gather_launches;
}
/* the blocks listed by decode launch i since the reset, ascending, into out (room for cap); returns their number, or
 * -1 when there is no launch i */
int emu_grid_decode_list(int i, int* out, int cap) {
  std::lock_guard<std::mutex> lk(g_grid_mu);
  if (i < 0 || i >= (int)g_decode_lists.size()) return -1;
  const std::vector<int>& l = g_decode_lists[(size_t)i];
  for (size_t k = 0; k < l.size() && (int)k < cap; k++) out[k] = l[k];
  return (int)l.size();
}

}  // extern "C"

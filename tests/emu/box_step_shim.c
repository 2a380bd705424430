/*
 * box_step_shim.c -- TEST INFRASTRUCTURE ONLY.
 *
 * The host code (blosc_b200.c, included whole) with its box normalisation and the three box functions exported, so
 * that tests/test_getslice_step.py can check box_build's B2Box and b2_box_next / b2_box_rank / b2_box_unrank against
 * brute force over every flat index.  The test compiles this file in place of blosc_b200.c into a library of its own
 * (with getslice_step_stage.cpp and simt_emu.cpp); the product never includes it.
 */
#include "../../c-blosc_b200/csrc/blosc_b200.c"

size_t emu_box_size(void) { return sizeof(B2Box); }

/* the checked, normalised box of a getslice_step call into *b: 0, 1 for an empty box, or -1 (with the call's message) */
int emu_box_build(int ndim, const int64_t* shape, const int64_t* start, const int64_t* stop, const int64_t* step,
                  B2Box* b) {
  long long nitems = 0;
  if (box_geometry(ndim, shape, start, stop, &nitems) || box_steps(ndim, step)) return -1;
  if (box_empty(ndim, start, stop)) return 1;
  box_build(ndim, shape, start, stop, step, nitems, b);
  return 0;
}

int emu_box_ndim(const B2Box* b) { return b->ndim; }
int emu_box_stepped(const B2Box* b) { return b->stepped; }
long long emu_box_run(const B2Box* b) { return b->run; }
long long emu_box_count(const B2Box* b) { return b->count; }
long long emu_box_next(const B2Box* b, long long x) { return b2_box_next(b, x, b->stepped); }
long long emu_box_rank(const B2Box* b, long long x) { return b2_box_rank(b, x, b->stepped); }
long long emu_box_unrank(const B2Box* b, long long p) { return b2_box_unrank(b, p, b->stepped); }

#!/usr/bin/env python
"""Workload for compute-sanitizer (memcheck / racecheck) on the LZ4 and BloscLZ decoders: every crafted stream of
tests/test_lz_decode_edges.py wrapped into a chunk -- unsplit single-stream blocks (decode_kernel) and typesize-4
blocks of four streams (decode_pair_kernel) -- in a device buffer of exactly its size, decoded into an exact-size
device buffer, so that a read past the input, a write past the output or a missing hand-off between the parser and
the copier shows.
  compute-sanitizer --tool memcheck python scripts/sanitize_lz_decode_edges.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import __graft_entry__ as g
import test_lz_decode_edges as ledges
pkg = g.load_package()
cases = 0
for _, ch, n in ledges.chunk_corpus():
    d_c = torch.from_numpy(np.frombuffer(ch, np.uint8).copy()).cuda()
    d_o = torch.empty(n, dtype=torch.uint8, device="cuda")
    pkg.decompress_ctx(d_c, d_o, n)
    cases += 1
torch.cuda.synchronize()
print("lz decode-edges sanitize workload ok, chunks", cases)

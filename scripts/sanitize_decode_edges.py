#!/usr/bin/env python
"""Workload for compute-sanitizer (memcheck) on the zstd and inflate decoders: every crafted, STRICT and damaged
zstd frame of tests/test_zstd_decode_edges.py and every crafted zlib stream of tests/test_zlib_decode_edges.py, each
wrapped into a chunk in a device buffer of exactly its size, decoded into an exact-size device buffer, so that a read
past the input or a write past the output shows.
  compute-sanitizer --tool memcheck python scripts/sanitize_decode_edges.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import __graft_entry__ as g
import test_zlib_decode_edges as iedges
import test_zstd_decode_edges as zedges
pkg = g.load_package()
cases = 0
chunks = [(ch, n) for _, ch, n, _ in zedges.chunk_corpus(damaged=True)] + [(ch, n) for _, ch, n in iedges.chunk_corpus()]
for ch, n in chunks:
    d_c = torch.from_numpy(np.frombuffer(ch, np.uint8).copy()).cuda()
    d_o = torch.empty(n, dtype=torch.uint8, device="cuda")
    pkg.decompress_ctx(d_c, d_o, n)
    cases += 1
torch.cuda.synchronize()
print("decode-edges sanitize workload ok, chunks", cases)

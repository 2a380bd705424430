#!/usr/bin/env python
"""Workload for compute-sanitizer (memcheck) on the one-warp LZ4 and BloscLZ encoders: every chunk of
tests/test_lz_encode_edges.py's corpus compressed from a device buffer that ends exactly at the source's last byte.
On the GPU the window loads (ldp_win12 / ldp_raw12) read aligned words up to 15 bytes past the position they start
at, where the emulator reads exactly 12 bytes, so a read past the input near a stream's end shows only here.
  compute-sanitizer --tool memcheck python scripts/sanitize_lz_encode_edges.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import __graft_entry__ as g
import test_lz_encode_edges as eedges
pkg = g.load_package()
cases = 0
for name, x, ts, shuf, comp, clevel, bs in eedges.chunk_corpus():
    d_x = torch.from_numpy(x.copy()).cuda()                     # exactly len(x) bytes
    d_out = torch.empty(len(x) + 16, dtype=torch.uint8, device="cuda")
    r = pkg.compress_ctx(clevel, shuf, ts, len(x), d_x, d_out, len(x) + 16, comp, bs)
    assert r > 0, (name, r)
    cases += 1
torch.cuda.synchronize()
print("lz encode-edges sanitize workload ok, chunks", cases)

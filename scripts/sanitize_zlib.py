#!/usr/bin/env python
"""Small workload for compute-sanitizer on the DEFLATE encoder (BLOSC_B200_ZLIB=1, csrc/dev_deflate.cuh): ragged sizes,
streams of several DEFLATE blocks (forced blocksize), split and unsplit chunks, raw and compressed streams, exact-size device buffers so that any
overrun shows."""
import os, sys
os.environ["BLOSC_B200_ZLIB"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
import __graft_entry__ as g
from datagen import gen
pkg = g.load_package()
for kind in ("bench", "text", "lowent", "mixed", "zeros", "rand"):
    for n in (100, 1000, 70001, 300001):
        src = gen(kind, n)
        d_src = torch.from_numpy(src).cuda()
        for ts, shuf, clevel, bs in ((4, 1, 5, 0), (1, 0, 9, 0), (8, 2, 1, 0), (3, 1, 5, 200000)):
            d_chunk = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
            cb = pkg.compress_ctx(clevel, shuf, ts, n, d_src, d_chunk, n + 16, "zlib", bs)
            assert cb > 0
            exact = d_chunk[:cb].clone()
            d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
            assert pkg.decompress_ctx(exact, d_out, n) == n and torch.equal(d_out, d_src)
print("zlib sanitize workload ok")

#!/usr/bin/env python
"""Small workload for compute-sanitizer on the snappy encoder and decoder (BLOSC_B200_SNAPPY=1, csrc/dev_snappy.cuh):
ragged sizes, split and unsplit chunks, raw and compressed streams, serial and pool maxout rules, the four snappy
goldens, exact-size device buffers so that any overrun shows."""
import os, sys
os.environ["BLOSC_B200_SNAPPY"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import glob
import numpy as np, torch
import __graft_entry__ as g
from datagen import gen
pkg = g.load_package()
for kind in ("bench", "text", "lowent", "mixed", "zeros", "rand"):
    for n in (100, 1000, 70001, 300001):
        src = gen(kind, n)
        d_src = torch.from_numpy(src).cuda()
        for ts, shuf, clevel, bs, nt in ((4, 1, 5, 0, 1), (1, 0, 9, 0, 4), (8, 2, 1, 0, 1), (3, 1, 5, 200000, 4)):
            d_chunk = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
            cb = pkg.compress_ctx(clevel, shuf, ts, n, d_src, d_chunk, n + 16, "snappy", bs, nt)
            assert cb > 0
            exact = d_chunk[:cb].clone()
            d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
            assert pkg.decompress_ctx(exact, d_out, n) == n and torch.equal(d_out, d_src)
want = torch.from_numpy(np.arange(1000000, dtype=np.int32).view(np.uint8).copy()).cuda()
for f in sorted(glob.glob(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "compat", "*-snappy.cdata"))):
    d_chunk = torch.from_numpy(np.fromfile(f, np.uint8)).cuda()
    d_out = torch.empty(4000000, dtype=torch.uint8, device="cuda")
    assert pkg.decompress_ctx(d_chunk, d_out, 4000000) == 4000000 and torch.equal(d_out, want)
print("snappy sanitize workload ok")

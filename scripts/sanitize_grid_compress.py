#!/usr/bin/env python
"""Small workload for compute-sanitizer memcheck: grid_compress of device arrays in exact-size device allocations,
edge chunks with and without a fill pattern, skip_fill, memcpyed chunks, device and host dest; each chunk checked
against compress_ctx of its padded sub-array."""
import itertools, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import __graft_entry__ as g
pkg = g.load_package()
for shape, cs, itemsize in (((300, 260), (64, 50), 4), ((37, 41, 29), (16, 16, 8), 2), ((5000,), (1024,), 8)):
    n = int(np.prod(shape)) * itemsize
    src = (torch.arange(n, device="cuda") // 24 % 200).to(torch.uint8)          # exactly n bytes
    src[: n // 5] = 0
    arr = src.view(*shape, itemsize)
    for fill, skip, clevel in ((None, False, 5), (bytes(range(1, itemsize + 1)), False, 5), (None, True, 5),
                               (None, False, 0)):
        bound = pkg.grid_bound(shape, cs, itemsize)
        for dest_dev in (True, False):
            dest = torch.empty(bound, dtype=torch.uint8, device="cuda" if dest_dev else "cpu")
            r, off = pkg.grid_compress(src, shape, cs, itemsize, clevel, 1, "lz4", dest, fill=fill, skip_fill=skip)
            assert r == off[-1] > 0
            pat = torch.zeros(itemsize, dtype=torch.uint8) if fill is None else torch.tensor(list(fill), dtype=torch.uint8)
            for i, co in enumerate(itertools.product(*(range(-(-s // c)) for s, c in zip(shape, cs)))):
                buf = pat.cuda().expand(tuple(cs) + (itemsize,)).contiguous()
                part = arr[tuple(slice(c * k, min((c + 1) * k, s)) for c, k, s in zip(co, cs, shape))]
                buf[tuple(slice(0, e) for e in part.shape[:-1])] = part
                if off[i + 1] == off[i]:
                    assert skip and bool((part == pat.cuda()).all())
                    continue
                d = torch.empty(buf.numel() + 16, dtype=torch.uint8, device="cuda")
                cb = pkg.compress_ctx(clevel, 1, itemsize, buf.numel(), buf, d, buf.numel() + 16, "lz4")
                assert cb == off[i + 1] - off[i] and torch.equal(d[:cb].cpu(), dest[off[i]:off[i + 1]].cpu())
torch.cuda.synchronize()
print("grid_compress memcheck workload ok")

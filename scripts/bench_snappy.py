#!/usr/bin/env python
"""bench_snappy.py -- the snappy encoder and decoder (BLOSC_B200_SNAPPY=1) on the cfg 2 data: one 256 MiB bench.c buffer,
shuffle, typesize 4, clevel 5, device resident.  Reports compress, decompress and compress+decompress GB/s, the ratio
next to this library's "lz4" and "lz4hc" ratios on the same call, the GPU's name and power limit (read in the same
run) and per-kernel CUDA-event times.  There is no CPU snappy baseline: the reference here is built without snappy.
Prints one JSON line.
    python scripts/bench_snappy.py [--steps K] [--warmup W]"""
import argparse
import json
import os
import sys
import time

sys.dont_write_bytecode = True
os.environ["BLOSC_B200_SNAPPY"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np
import torch

import __graft_entry__ as g

WORKLOAD = ("snappy", 1, 4, 5, 256 << 20)      # compressor, doshuffle, typesize, clevel, nbytes


def power_limit():
    """the board's power limit in watts, read with nvidia-smi (None where it cannot be read)"""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    comp, shuf, ts, clevel, nbytes = WORKLOAD
    pkg = g.load_package()
    i = np.arange(nbytes // 4, dtype=np.uint32)
    src = (((i << np.uint32(26)) ^ (i << np.uint32(18)) ^ (i << np.uint32(11)) ^ (i << np.uint32(3)) ^ i)
           & np.uint32((1 << 19) - 1)).view(np.uint8)
    d_src = torch.from_numpy(src.copy()).cuda()
    d_chunk = torch.zeros(nbytes + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    hc = pkg.compress_ctx(clevel, shuf, ts, nbytes, d_src, d_chunk, nbytes + 16, "lz4hc")
    l4 = pkg.compress_ctx(clevel, shuf, ts, nbytes, d_src, d_chunk, nbytes + 16, "lz4")
    for _ in range(max(1, args.warmup)):
        cb = pkg.compress_ctx(clevel, shuf, ts, nbytes, d_src, d_chunk, nbytes + 16, comp)
        nb = pkg.decompress_ctx(d_chunk, d_out, nbytes)
    assert cb > 0 and nb == nbytes and torch.equal(d_out, d_src), (cb, nb)
    pkg.set_profiling(True); pkg.prof_reset()
    torch.cuda.synchronize()
    tc = td = 0.0
    for _ in range(args.steps):
        t0 = time.perf_counter()
        cb = pkg.compress_ctx(clevel, shuf, ts, nbytes, d_src, d_chunk, nbytes + 16, comp)
        t1 = time.perf_counter()
        nb = pkg.decompress_ctx(d_chunk, d_out, nbytes)
        t2 = time.perf_counter()
        tc += t1 - t0; td += t2 - t1
    prof = pkg.prof_get(); pkg.set_profiling(False)
    assert cb > 0 and nb == nbytes and torch.equal(d_out, d_src)
    line = {"workload": "snappy-shuffle-ts4-cl5-256MiB", "gpu": torch.cuda.get_device_name(), "steps": args.steps,
            "compress_gbs": nbytes / (tc / args.steps) / 1e9, "decompress_gbs": nbytes / (td / args.steps) / 1e9,
            "value": 2 * nbytes / ((tc + td) / args.steps) / 1e9, "unit": "GB/s", "cbytes": cb, "ratio": nbytes / cb,
            "lz4_cbytes": l4, "lz4_ratio": nbytes / l4, "lz4hc_cbytes": hc, "lz4hc_ratio": nbytes / hc,
            "power_limit_w": power_limit(),
            "kernels_ms": {k: v[0] / v[1] for k, v in prof.items() if v[1]}}
    line["cpu_baseline"] = "none: the reference here is built without snappy"
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""lz4_cycles.py -- where the LZ4 team encoder's cycles go, per phase, on the headline workload
(bench.py: LZ4, shuffle, typesize 4, clevel 5, 256 MiB of bench.c data).

    python scripts/lz4_cycles.py [--lib variant.so] [-D FLAG ...]

Builds the library with -DB2_LZ4_CYCLES into a temporary directory (or takes an instrumented build
given with --lib), compresses the buffer in team mode (one warm-up call, then the measured one) and
prints, per split of a block, the streams' sequence counts and clock64() cycles, then the phase
breakdown of the hard streams (more than 1000 sequences) per sequence.  Phases (dev_lz4.cuh, LZ4C_*):
  start    chain start: publishing the walker's tile until the chain's first tiles are ready
  chain    the walker's own work in a chain (chain time minus its tile waits), including the first four probes
           of the search after a chained miss, which the walker takes from the verdicts
  fullwait the walker waiting for the ready word of a tile inside a chain
  reprobe  stale verdicts and post-match probes done by the scalar code
  search   the rest of a search the chain left (scalar probes, 32-wide rounds, catch-up)
  other    the rest of the call (emission of searched sequences, table init, last literals)
and, for the preparers, the cycles per tile from being allowed to prepare it to posting its ready word,
split into the load of the tile's own bytes (with hash and table read) and the candidate gather (with
compare); and the share of chained positions whose verdict was stale (its snap differed from the live
table), which the scalar code probes again; and the chained windows: sequences per window and what ended them
(a stale element, a valid miss, a valid LZ4T_LONG, the end of the stream, a full window, the next position
past the checked tiles)."""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# dev_lz4.cuh, enum LZ4C_*
TOTAL, START, SESSION, FULLWAIT, REPROBE, SEARCH, SESSIONS, SEQS, CHAIN_SEQS, PREP_BUSY, PREP_OWN, PREP_GATHER, \
    PREP_TILES, SMID, SUBP, STALE = range(16)
NCOL = 16
# the second enum: chained windows and what ended each
WINDOWS, W_STALE, W_MISS, W_LONG, W_END, W_CAP, W_TILE = range(NCOL, NCOL + 7)
NREC = NCOL + 7                                 # LZ4C_NREC: columns of a stream's record
MAXSTREAMS = 16384


def build(tmp, flags):
    import __graft_entry__ as g
    lib = os.path.join(tmp, "libblosc_b200_cycles.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run([nvcc, *g.NVCC_FLAGS, "-DB2_LZ4_CYCLES", *flags, os.path.join(g.CSRC, "backend_cuda.cu"),
                    os.path.join(g.CSRC, "blosc_b200.c"), "-o", lib], check=True)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="an instrumented build (-DB2_LZ4_CYCLES) to use instead of building one")
    ap.add_argument("-D", dest="defs", action="append", default=[], help="extra preprocessor definition for the build")
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="lz4_cycles_")
    os.environ["BLOSC_B200_LIB"] = args.lib or build(tmp, ["-D" + d for d in args.defs])
    os.environ["BLOSC_B200_LZ4_TEAM"] = "1"

    import numpy as np
    import torch

    import __graft_entry__ as g
    from bench import WORKLOADS, CFG2, bench_words
    pkg = g.load_package()
    pkg.lib.b2_lz4_cycles_read.restype = C.c_int
    pkg.lib.b2_lz4_cycles_read.argtypes = [C.c_void_p, C.c_int]

    comp, shuf, ts, clevel, nbytes = WORKLOADS[CFG2]
    d_src = torch.from_numpy(bench_words(nbytes, np).copy()).cuda()
    d_chunk = torch.zeros(nbytes + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(clevel, shuf, ts, nbytes, d_src, d_chunk, nbytes + 16, comp)
    pkg.set_profiling(True); pkg.prof_reset()
    cb = pkg.compress_ctx(clevel, shuf, ts, nbytes, d_src, d_chunk, nbytes + 16, comp)
    prof = pkg.prof_get(); pkg.set_profiling(False)
    rec = np.zeros((MAXSTREAMS, NREC), np.uint64)
    ns = pkg.lib.b2_lz4_cycles_read(rec.ctypes.data_as(C.c_void_p), MAXSTREAMS)
    props = torch.cuda.get_device_properties(0)
    print(f"{props.name}, {props.multi_processor_count} SMs; {CFG2}: cbytes {cb}; kernels (ms) "
          f"{ {k: round(v[0] / max(v[1], 1), 3) for k, v in prof.items() if v[1]} }")
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        print(f"power limit, max SM clock, SM clock: {q}")
    except (OSError, subprocess.SubprocessError):
        pass

    # a full block of a typesize-4 shuffle is 4 streams, one per byte-plane
    r = rec[:ns].astype(np.float64)
    used = r[:, TOTAL] > 0
    nsplits = 4
    print("split streams  seqs/stream  cycles/stream  cycles/seq")
    for sp in range(nsplits):
        m = used & (np.arange(ns) % nsplits == sp)
        if not m.any():
            continue
        seqs, tot = r[m, SEQS] + r[m, CHAIN_SEQS], r[m, TOTAL]
        print(f"{sp:5d} {m.sum():7d} {seqs.mean():12.0f} {tot.mean():14.0f} {tot.sum() / max(seqs.sum(), 1):11.1f}")

    hard = used & (r[:, SEQS] + r[:, CHAIN_SEQS] > 1000)
    if not hard.any():
        print("no hard streams")
        return
    h = r[hard]
    seqs = (h[:, SEQS] + h[:, CHAIN_SEQS]).sum()
    chain = h[:, SESSION] - h[:, FULLWAIT]
    other = h[:, TOTAL] - h[:, START] - h[:, SESSION] - h[:, REPROBE] - h[:, SEARCH]
    print(f"hard streams: {hard.sum()}, {seqs / hard.sum():.0f} sequences each ({h[:, CHAIN_SEQS].sum() / seqs:.1%} in a chain), "
          f"{h[:, SESSIONS].sum() / hard.sum():.0f} chains each; "
          f"{len(set(zip(h[:, SMID].astype(int), h[:, SUBP].astype(int))))} distinct (SM, sub-partition) walker slots, "
          f"{len(set(h[:, SMID].astype(int)))} SMs")
    print("walker phase   cycles/seq   share")
    tot = h[:, TOTAL].sum()
    for name, v in (("start", h[:, START].sum()), ("chain", chain.sum()), ("fullwait", h[:, FULLWAIT].sum()),
                    ("reprobe", h[:, REPROBE].sum()), ("search", h[:, SEARCH].sum()), ("other", other.sum()),
                    ("total", tot)):
        print(f"  {name:10s} {v / seqs:10.1f} {v / tot:7.1%}")
    tiles = h[:, PREP_TILES].sum()
    print(f"preparers: {tiles / hard.sum():.0f} tiles per stream; cycles per tile: allowed..ready {h[:, PREP_BUSY].sum() / tiles:.0f}, "
          f"own bytes {h[:, PREP_OWN].sum() / tiles:.0f}, gather {h[:, PREP_GATHER].sum() / tiles:.0f}")
    looked = h[:, CHAIN_SEQS].sum() + h[:, STALE].sum()
    print(f"stale verdicts re-probed: {h[:, STALE].sum() / hard.sum():.0f} per stream, "
          f"{h[:, STALE].sum() / seqs:.2%} of all sequences, {h[:, STALE].sum() / max(looked, 1):.2%} of chained lookups; "
          f"chain cycles per chained sequence {chain.sum() / max(h[:, CHAIN_SEQS].sum(), 1):.1f}")
    win = h[:, WINDOWS].sum()
    ends = ", ".join(f"{name} {h[:, k].sum() / max(win, 1):.1%}" for name, k in
                     (("stale", W_STALE), ("miss", W_MISS), ("long", W_LONG), ("end", W_END), ("full", W_CAP), ("tile", W_TILE)))
    print(f"windows: {win / hard.sum():.0f} per stream, {h[:, CHAIN_SEQS].sum() / max(win, 1):.2f} chained sequences per window; "
          f"ended by {ends}")


if __name__ == "__main__":
    main()

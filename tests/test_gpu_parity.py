"""GPU parity tests: the CUDA path, called through the C ABI of libblosc_b200.so, against
the oracle (bit-exact) on the same seeded inputs, against the compat golden chunks, and at
BASELINE.json's full sizes.  Mirrors the reference's own test strategy
(tests/test_compress_roundtrip.c, test_getitem.c, test_maxout.c, test_bitshuffle_leftovers.c,
test_shuffle_roundtrip_*.c, compat/CMakeLists.txt)."""
import glob
import os

import numpy as np
import pytest

from datagen import bench_words, ci, compress, decompress, gen, ptr, sz

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpu_compress(pkg, clevel, shuf, ts, src, destsize, comp, bs=0, nt=1):
    dest = np.full(destsize + 64, 0xAA, np.uint8)
    r = pkg.compress_ctx(clevel, shuf, ts, len(src), src, dest, destsize, comp, bs, nt)
    return r, dest


def _gpu_decompress(pkg, chunk, destsize):
    dest = np.zeros(destsize + 64, np.uint8)
    r = pkg.decompress_ctx(chunk, dest, destsize)
    return r, dest


# ---------------------------------------------------------------- filters
@pytest.mark.parametrize("ts", [1, 2, 3, 4, 5, 7, 8, 11, 16, 17, 32, 53])
def test_filters_match_oracle(pkg, orc, cuda, ts):
    """tests/test_shuffle_roundtrip_generic.csv shapes + cross-implementation equality
    (the reference pins SIMD == generic in test_shuffle_roundtrip_sse2.c)."""
    for n in [7, 192, 500, 1792, 8000, 100000, 702713, 131072, 1 << 20]:
        n_bytes = n * ts if n < 200000 else n
        src = gen("rand", n_bytes, seed=ts)
        for mode, fn in enumerate(["orc_shuffle", "orc_unshuffle", "orc_bitshuffle", "orc_bitunshuffle"]):
            if mode >= 2 and n_bytes < ts:
                continue
            want = np.zeros(n_bytes + 1, np.uint8)
            got = np.zeros(n_bytes + 1, np.uint8)
            getattr(orc, fn)(sz(ts), sz(n_bytes), ptr(src), ptr(want))
            assert pkg.filter_block(mode, ts, n_bytes, src, got) == 0
            assert (want == got).all(), (fn, ts, n_bytes)


def test_filters_device_pointers_and_misalignment(pkg, orc, cuda):
    torch = cuda
    n = 1 << 20
    host = gen("rand", n + 64, seed=5)
    dev = torch.from_numpy(host).cuda()
    for off in (0, 1, 3, 16):
        for ts in (4, 8):
            for mode, fn in enumerate(["orc_shuffle", "orc_unshuffle", "orc_bitshuffle", "orc_bitunshuffle"]):
                want = np.zeros(n, np.uint8)
                getattr(orc, fn)(sz(ts), sz(n), ptr(host[off:off + n]), ptr(want))
                out = torch.zeros(n + 64, dtype=torch.uint8, device="cuda")
                assert pkg.filter_block(mode, ts, n, dev[off:], out[off:]) == 0
                assert (out[off:off + n].cpu().numpy() == want).all(), (fn, ts, off)


# ---------------------------------------------------------------- compress / decompress
CASES = [(comp, ts, shuf, clevel)
         for comp in ("lz4", "blosclz")
         for ts in (1, 2, 4, 8, 16, 3, 32)
         for shuf in (0, 1, 2)
         for clevel in (1, 5, 9)]


@pytest.mark.parametrize("comp,ts,shuf,clevel", CASES)
def test_chunks_bit_identical_to_oracle(pkg, orc, cuda, comp, ts, shuf, clevel):
    """GPU chunk == oracle chunk byte for byte (the oracle itself is pinned to the reference),
    oracle decodes it, GPU decodes it."""
    for kind, n in (("bench", 4 << 20), ("i32", 1000000), ("text", 300001), ("mixed", 1 << 20), ("rand", 70000)):
        src = gen(kind, n, seed=clevel)
        want_n, want = compress(orc, "orc_compress_ctx", clevel, shuf, ts, src, n + 16, comp)
        got_n, got = _gpu_compress(pkg, clevel, shuf, ts, src, n + 16, comp)
        assert got_n == want_n, (kind, n, got_n, want_n)
        assert (got[:got_n] == want[:want_n]).all(), (kind, n)
        assert (got[got_n:] == 0xAA).all(), "wrote past the returned size"
        dn, out = _gpu_decompress(pkg, got, n)
        assert dn == n and (out[:n] == src).all()


@pytest.mark.parametrize("n", [0, 1, 7, 100, 127, 128, 129, 1000, 4096, 32767, 32768, 65536, 100000, 641091])
def test_small_and_ragged_sizes(pkg, orc, cuda, n):
    """tests/test_compress_roundtrip.csv sizes, test_compressor.c:232-260 (empty / <128 B ->
    MEMCPYED), test_bitshuffle_leftovers.c (641091 B, lz4, clevel 9, bitshuffle)."""
    for kind in ("bench", "rand"):
        src = gen(kind, n, seed=n)
        for comp, ts, shuf, clevel, bs in (("lz4", 4, 1, 5, 0), ("blosclz", 8, 2, 5, 0), ("lz4", 4, 2, 9, 0), ("lz4", 8, 2, 9, 0),
                                           ("blosclz", 3, 1, 5, 0), ("lz4", 4, 1, 5, 4096), ("blosclz", 4, 1, 5, 100), ("lz4", 2, 1, 0, 0)):
            want_n, want = compress(orc, "orc_compress_ctx", clevel, shuf, ts, src, n + 16, comp, bs)
            got_n, got = _gpu_compress(pkg, clevel, shuf, ts, src, n + 16, comp, bs)
            assert got_n == want_n and (got[:got_n] == want[:want_n]).all(), (kind, n, comp, ts, shuf, clevel, bs)
            dn, out = _gpu_decompress(pkg, got, n)
            assert dn == n and (out[:n] == src).all()


def test_baseline_cfg1_memcpyed_1mib(pkg, orc, cuda):
    """BASELINE.json configs[0]: 1 MiB, typesize 4, shuffle, clevel 0 -> a MEMCPYED chunk of nbytes+16 with blocksize 8192 and
    no filter applied (blosc.c:825-830), identical to the oracle's, from host and from device pointers."""
    torch = cuda
    n = 1 << 20
    src = gen("rand", n, seed=11)
    want_n, want = compress(orc, "orc_compress_ctx", 0, 1, 4, src, n + 16, "blosclz")
    got_n, got = _gpu_compress(pkg, 0, 1, 4, src, n + 16, "blosclz")
    assert got_n == want_n == n + 16 and (got[:got_n] == want[:want_n]).all()
    assert got[2] & 0x2 and int.from_bytes(bytes(got[8:12]), "little") == 8192 and (got[16:16 + n] == src).all()
    d_src = torch.from_numpy(src).cuda()
    d_chunk = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    assert pkg.compress_ctx(0, 1, 4, n, d_src, d_chunk, n + 16, "lz4") == n + 16
    d_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
    assert pkg.decompress_ctx(d_chunk, d_out, n) == n and torch.equal(d_out, d_src)
    dn, out = _gpu_decompress(pkg, got, n)
    assert dn == n and (out[:n] == src).all()


def test_maxout_semantics(pkg, cuda):
    """tests/test_maxout.c:26-143."""
    n = 1000 * 1000
    src = gen("rand", n, seed=1)
    assert _gpu_compress(pkg, 5, 1, 4, src, n + 16 - 1, "blosclz")[0] == 0
    assert _gpu_compress(pkg, 5, 1, 4, src, n + 16, "blosclz")[0] == n + 16
    r, chunk = _gpu_compress(pkg, 5, 1, 4, src, n + 16 + 1, "lz4")
    assert r == n + 16 and chunk[2] & 0x2
    dn, out = _gpu_decompress(pkg, chunk, n)
    assert dn == n and (out[:n] == src).all()
    assert _gpu_compress(pkg, 5, 1, 4, src, 15, "blosclz")[0] == 0
    assert _gpu_compress(pkg, 10, 1, 4, src, n + 16, "blosclz")[0] == -10
    assert _gpu_compress(pkg, 5, 3, 4, src, n + 16, "blosclz")[0] == -10
    assert _gpu_compress(pkg, 5, 1, 0, src, n + 16, "blosclz")[0] == -10
    assert _gpu_compress(pkg, 5, 1, 4, src, n + 16, "snappy")[0] == -5
    # nthreads is validated only where the reference takes its pool path (more than one block, blosc.c:910)
    assert _gpu_compress(pkg, 5, 1, 4, src, n + 16, "lz4", 0, 0)[0] == n + 16
    big = gen("rand", 4 << 20, seed=2)
    assert _gpu_compress(pkg, 5, 1, 4, big, len(big) + 16, "lz4", 0, 0)[0] == -1
    assert _gpu_compress(pkg, 5, 1, 4, big, len(big) + 16, "lz4", 0, 300)[0] == -1


def test_block_scan_of_more_than_65536_blocks(pkg, orc, cuda):
    """scan_kernel, launched for chunks of more than 65536 blocks: the oracle's return codes and chunks under the serial
    (nthreads 1) and the pool (nthreads 2) fit rules, with room to spare and with one byte too few."""
    n = 128 * 65536 + 4100
    src = gen("bench", n, seed=7)
    for comp, clevel in (("blosclz", 1), ("lz4", 5)):
        for nt in (1, 2):
            fit, _ = compress(orc, "orc_compress_ctx", clevel, 1, 4, src, n + 16, comp, 128, nt)
            assert 0 < fit < n + 16
            for destsize in (n + 16, fit - 1):
                want_n, want = compress(orc, "orc_compress_ctx", clevel, 1, 4, src, destsize, comp, 128, nt)
                got_n, got = _gpu_compress(pkg, clevel, 1, 4, src, destsize, comp, 128, nt)
                assert got_n == want_n == (fit if destsize > fit else 0), (comp, nt, destsize, got_n, want_n)
                m = max(got_n, 16)
                assert (got[:m] == want[:m]).all() and (got[m:] == 0xAA).all(), (comp, nt, destsize)


def test_compat_golden_chunks(pkg, cuda):
    """compat/*.cdata: every chunk written by blosc 1.3.0 ... 1.18.0 with blosclz / lz4 / lz4hc
    -- and zlib / zstd, through the decode-only GPU decoders -- decodes bit-exactly to int32
    data[i] = i (compat/filegen.c:33,61-66); snappy chunks report -5 like the stock reference
    build, which does not have snappy either."""
    want = np.arange(1000000, dtype=np.int32).view(np.uint8)
    files = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "compat", "*.cdata")))
    assert len(files) == 29
    nok = 0
    for f in files:
        chunk = np.fromfile(f, np.uint8)
        r, out = _gpu_decompress(pkg, chunk, 4000000)
        if "snappy" in f:
            assert r == -5, f
        else:
            assert r == 4000000 and (out[:4000000] == want).all(), f
            nok += 1
    assert nok == 25


def test_getitem(pkg, orc, cuda):
    """tests/test_getitem.c plus ranges crossing block boundaries."""
    n = 3000000
    src = gen("i32", n)
    for comp, ts, shuf in (("lz4", 4, 1), ("blosclz", 8, 2), ("lz4", 1, 0), ("blosclz", 4, 1)):
        cb, chunk = _gpu_compress(pkg, 5, shuf, ts, src, n + 16, comp)
        assert cb > 0
        nit = n // ts
        for start, cnt in ((0, nit), (0, 1), (nit - 1, 1), (12345, 54321), (nit // 2, nit // 3), (0, 0), (65536 - 3, 7)):
            out = np.zeros(n + 8, np.uint8)
            r = pkg.getitem(chunk, start, cnt, out)
            assert r == cnt * ts
            assert (out[:r] == src[start * ts:start * ts + r]).all(), (comp, ts, start, cnt)
        assert pkg.getitem(chunk, -1, 10, np.zeros(64, np.uint8)) == -1
        assert pkg.getitem(chunk, nit - 1, 5, np.zeros(64, np.uint8)) == -1


def test_device_resident_round_trip(pkg, orc, cuda):
    """Device pointers in, device pointers out: nothing crosses PCIe except the 8-byte result."""
    torch = cuda
    n = 8 << 20
    src = bench_words(n)
    d_src = torch.from_numpy(src).cuda()
    for comp, ts, shuf in (("lz4", 4, 1), ("blosclz", 8, 2)):
        d_chunk = torch.full((n + 16,), 0xAA, dtype=torch.uint8, device="cuda")
        cb = pkg.compress_ctx(5, shuf, ts, n, d_src, d_chunk, n + 16, comp)
        want_n, want = compress(orc, "orc_compress_ctx", 5, shuf, ts, src, n + 16, comp)
        assert cb == want_n and (d_chunk[:cb].cpu().numpy() == want[:cb]).all()
        d_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
        assert pkg.decompress_ctx(d_chunk, d_out, n) == n
        assert torch.equal(d_out, d_src)
        d_item = torch.zeros(4096, dtype=torch.uint8, device="cuda")
        assert pkg.getitem(d_chunk, 1000, 4096 // ts, d_item) == 4096
        assert torch.equal(d_item, d_src[1000 * ts:1000 * ts + 4096])


def test_ordered_after_default_stream_work(pkg, orc, cuda):
    """Like cudaMemcpy, a call is ordered after work the caller has queued on the (legacy) default
    stream: a buffer still being produced by PyTorch kernels is compressed correctly, and PyTorch
    work queued right after a call sees its result."""
    torch = cuda
    n = 32 << 20
    x = torch.arange(n // 4, device="cuda", dtype=torch.int32)
    for _ in range(40):                                   # a queue of kernels the host does not wait for
        x = (x * 3 + 1) & 0xFFFFF
    d_chunk = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(5, 1, 4, n, x, d_chunk, n + 16, "lz4")
    src = x.cpu().numpy().view(np.uint8)
    want_n, want = compress(orc, "orc_compress_ctx", 5, 1, 4, src, n + 16, "lz4")
    assert cb == want_n and (d_chunk[:cb].cpu().numpy() == want[:cb]).all()
    d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert pkg.decompress_ctx(d_chunk, d_out, n) == n
    assert torch.equal(d_out.view(torch.int32) + 1, x + 1)


def test_corrupted_chunks_fail_cleanly(pkg, cuda):
    """Appendix B of SURVEY.md / tests/fuzz: malformed input returns an error, never crashes."""
    n = 1 << 20
    src = bench_words(n)
    cb, chunk = _gpu_compress(pkg, 5, 1, 4, src, n + 16, "lz4")
    chunk = chunk[:cb].copy()
    out = np.zeros(n, np.uint8)

    def dec(c, size=n):
        return pkg.decompress_ctx(np.ascontiguousarray(c), out, size)
    c = chunk.copy(); c[0] = 3; assert dec(c) == -1
    c = chunk.copy(); c[1] = 2; assert dec(c) == -9
    c = chunk.copy(); c[2] |= 0x08; assert dec(c) == -1
    c = chunk.copy(); c[2] = (c[2] & 0x1f) | (2 << 5); assert dec(c) == -5
    c = chunk.copy(); c[3] = 0; assert dec(c) == -1
    c = chunk.copy(); c[8:12] = 0; assert dec(c) == -1
    assert dec(chunk, n - 1) == -1
    c = chunk.copy(); c[16:20] = np.frombuffer(np.int32(-5).tobytes(), np.uint8); assert dec(c) == -1
    c = chunk.copy(); c[16:20] = np.frombuffer(np.int32(0x7fffff00).tobytes(), np.uint8); assert dec(c) == -1
    rng = np.random.default_rng(7)
    for _ in range(40):                     # random payload corruption: must end in n or -1
        c = chunk.copy()
        pos = rng.integers(16, cb, 8)
        c[pos] = rng.integers(0, 256, 8, dtype=np.uint8)
        assert dec(c) in (n, -1)
    assert dec(chunk) == n and (out == src).all()


# ---------------------------------------------------------------- BASELINE.json full-size configs
def _checksum(a):
    return int(a.view(np.uint64).sum(dtype=np.uint64)) if len(a) % 8 == 0 else int(a.sum(dtype=np.uint64))


@pytest.mark.parametrize("comp,shuf,ts,want_cbytes", [
    ("lz4", 1, 4, 20401680),        # BASELINE config 2 (oracle output of the reference, BASELINE.md section 2)
    ("blosclz", 2, 8, 1796368),     # BASELINE config 3
    ("lz4", 1, 8, 7313680),         # config 5 rows
    ("lz4", 1, 16, 10199056),
    ("lz4", 1, 2, 37749776),
    ("lz4", 1, 1, 268435472),       # falls back to a MEMCPYED chunk
])
def test_baseline_configs_full_size(pkg, cuda, comp, shuf, ts, want_cbytes):
    """256 MiB bench.c buffer, device resident: compressed size equals the reference's own
    (deterministic) cbytes; round trip is exact (checksum of the decoded buffer == source)."""
    torch = cuda
    n = 256 << 20
    src = bench_words(n)
    d_src = torch.from_numpy(src).cuda()
    d_chunk = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    cb = pkg.compress_ctx(5, shuf, ts, n, d_src, d_chunk, n + 16, comp)
    assert cb == want_cbytes
    d_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
    assert pkg.decompress_ctx(d_chunk, d_out, n) == n
    assert torch.equal(d_out, d_src)
    assert _checksum(d_out.cpu().numpy()) == _checksum(src)

"""A plain-Python zstd frame writer (RFC 8878) that writes exactly what it is told: test infrastructure for the zstd
decoder (csrc/dev_zstd.cuh).

There is no compression search.  A frame is described by its header fields and a list of blocks, and every choice the
format leaves open is the caller's: literals mode, size format and stream count, Huffman weights (direct or FSE-coded
with a chosen distribution), the sequences, each sequence table's mode and FSE distribution.  So the tests can spell
forms that no encoder in this project writes: treeless literals, repeat table modes across raw blocks, every size
format at its thresholds, 255 FSE-coded weights, all window descriptors, checksums, skippable frames.

FSE encoding walks the decoding table backwards: for the symbol before, it picks the state of that symbol whose
[base, base + 2^nbits) holds the current state and emits the difference, so no separate encoding table is needed.
Huffman codes are canonical from the weights in the RFC's order (longer codes first, natural symbol order within a
length).  Bitstreams are backward, closed by an end mark.

Block descriptions (dicts):
  {"type": "raw", "data": bytes}
  {"type": "rle", "byte": int, "size": int}
  {"type": "compressed", "lit": LIT, "seqs": [(ll, ml, offset_value)], "modes": {"ll": M, "of": M, "ml": M},
   "count_bytes": 1 | 2 | 3 (optional)}
  LIT: {"mode": "raw" | "rle" | "huf" | "treeless", "data": bytes, "sf": size format (optional), "streams": 1 | 4,
        "weights": [weight of each byte value] (optional, last nonzero implied), "wmode": "direct" | "fse",
        "wnorm": (norm, log) (optional)}
  M: "predefined" | ("rle", code) | ("fse", norm, log) | ("fse", None, log) (normalised from the codes) | "repeat"
Any block may carry "bsize" (the size written in its header, for damaged frames) and "last".
"""
import heapq

import zstd_frame as zf

MAGIC = zf.MAGIC
SKIPPABLE = 0x184D2A50


xxh64 = zf.xxh64                                     # content checksums (zstd_frame.py, checked against published values)


# ---------------------------------------------------------------------------------------------------------------
# bit writers
# ---------------------------------------------------------------------------------------------------------------
class _Fwd:
    """forward bit writer, LSB first"""

    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value, nbits):
        assert 0 <= value < (1 << nbits) or nbits == 0 and value == 0, (value, nbits)
        self.v |= value << self.n
        self.n += nbits

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def backward(items):
    """a backward bitstream whose reader meets `items` ((value, nbits), in reading order) first to last"""
    w = _Fwd()
    for value, nbits in reversed(items):
        w.put(value, nbits)
    w.put(1, 1)                                     # end mark
    return w.bytes()


# ---------------------------------------------------------------------------------------------------------------
# FSE
# ---------------------------------------------------------------------------------------------------------------
def fse_description(norm, log):
    """RFC 8878 4.1.1 table description of `norm` (the list ends at its last nonzero entry)"""
    norm = list(norm)
    while norm and norm[-1] == 0:
        norm.pop()
    assert sum(abs(c) for c in norm) == 1 << log, (norm, log)
    w = _Fwd()
    w.put(log - 5, 4)
    remaining, threshold, nbits = (1 << log) + 1, 1 << log, log + 1
    s, prev0 = 0, False
    while remaining > 1:
        if prev0:
            start = s
            while norm[s] == 0:
                s += 1
            z = s - start
            while z >= 3:
                w.put(3, 2)
                z -= 3
            w.put(z, 2)
        count = norm[s]
        s += 1
        mx = 2 * threshold - 1 - remaining
        remaining -= abs(count)
        count += 1
        if count >= threshold:
            count += mx
        w.put(count, nbits - 1 if count < mx else nbits)
        prev0 = count == 1
        while remaining < threshold:
            nbits -= 1
            threshold >>= 1
    return w.bytes()


def normalize(counts, log):
    """counts (one per symbol) -> a normalised distribution summing to 2^log, every present symbol at least 1"""
    total = sum(counts)
    size = 1 << log
    norm = [max(1, c * size // total) if c else 0 for c in counts]
    big = max(range(len(counts)), key=lambda i: norm[i])
    norm[big] += size - sum(norm)
    assert norm[big] > 0, (counts, log)
    return norm


def fse_states(table, symbols, last_needs_bits=False):
    """states for `symbols` in decoding order such that each state follows from the one before; returns (states,
    bits of each transition as (value, nbits)).  With last_needs_bits the last state must read at least one bit."""
    n = len(symbols)
    states = [None] * n
    cand = [u for u, (s, nb, _) in enumerate(table) if s == symbols[-1] and (nb > 0 or not last_needs_bits)]
    assert cand, ("symbol has no state", symbols[-1])
    states[-1] = cand[0]
    bits = [None] * (n - 1)
    for k in range(n - 2, -1, -1):
        nxt = states[k + 1]
        for u, (s, nb, base) in enumerate(table):
            if s == symbols[k] and base <= nxt < base + (1 << nb):
                states[k] = u
                bits[k] = (nxt - base, nb)
                break
        else:
            raise AssertionError(("no state reaches", nxt, symbols[k]))
    return states, bits


# ---------------------------------------------------------------------------------------------------------------
# Huffman literals
# ---------------------------------------------------------------------------------------------------------------
def weights_for(data, maxbits=11):
    """Huffman weights (one per byte value) of a complete code for the bytes in `data`: Huffman's lengths when they
    fit in maxbits, otherwise a flat code.  A lone symbol gets a partner."""
    counts = [0] * 256
    for b in data:
        counts[b] += 1
    syms = [s for s in range(256) if counts[s]]
    if len(syms) == 1:
        other = 1 if syms[0] == 0 else 0
        syms, counts[other] = sorted(syms + [other]), 1
    heap = [(counts[s], i, [s]) for i, s in enumerate(syms)]
    heapq.heapify(heap)
    depth = {s: 0 for s in syms}
    k = len(heap)
    while len(heap) > 1:
        c1, _, a = heapq.heappop(heap)
        c2, _, b = heapq.heappop(heap)
        for s in a + b:
            depth[s] += 1
        heapq.heappush(heap, (c1 + c2, k, a + b))
        k += 1
    if max(depth.values()) > maxbits:
        L = (len(syms) - 1).bit_length()
        nshort = (1 << L) - len(syms)
        depth = {s: (L - 1 if i < nshort else L) for i, s in enumerate(syms)}
    maxb = max(depth.values())
    w = [0] * 256
    for s, d in depth.items():
        w[s] = maxb + 1 - d
    return w


def huffman_codes(weights):
    """weights (one per byte value, including the implied last) -> {symbol: (code, nbits)}"""
    total = sum(1 << (x - 1) for x in weights if x)
    maxb = total.bit_length() - 1
    assert total == 1 << maxb, "weights do not give a complete tree"
    codes, at = {}, 0
    for wt in range(1, maxb + 1):
        for s, x in enumerate(weights):
            if x == wt:
                codes[s] = (at >> (wt - 1), maxb + 1 - wt)
                at += 1 << (wt - 1)
    return codes


def huffman_stream(data, codes):
    return backward([codes[b] for b in data])


def huffman_tree(weights, wmode=None, wnorm=None):
    """the tree description: header byte, then direct 4-bit weights or an FSE-coded weight stream (by default FSE
    when the explicit weights take two values or more, which FSE coding needs)"""
    last = max(s for s in range(256) if weights[s])
    explicit = list(weights[:last])
    if wmode is None:
        wmode = "fse" if len(set(explicit)) > 1 else "direct"
    if wmode == "direct":
        assert 1 <= len(explicit) <= 128
        w = explicit + [0]
        return bytes([127 + len(explicit)]) + bytes((w[i] << 4) | w[i + 1] for i in range(0, len(explicit), 2))
    assert len(explicit) >= 2
    if wnorm is None:
        hist = [explicit.count(v) for v in range(13)]
        wnorm = (normalize(hist, 6), 6)
    norm, log = wnorm
    desc = fse_description(norm, log)
    table = zf.build_fse_table(list(norm), log)
    # two interleaved states: even weights from the first, odd from the second; the stream ends where the update
    # after the second-to-last weight reads past its start
    chains = (explicit[0::2], explicit[1::2])
    n = len(explicit)
    st, bits = [], []
    for c, chain in enumerate(chains):
        s, b = fse_states(table, chain, last_needs_bits=(n - 2) % 2 == c)
        st.append(s)
        bits.append(b)
    items = [(st[0][0], log), (st[1][0], log)]
    for k in range(n - 2):
        items.append(bits[k % 2][k // 2])
    stream = backward(items)
    body = desc + stream
    assert len(body) < 128
    return bytes([len(body)]) + body


# ---------------------------------------------------------------------------------------------------------------
# blocks
# ---------------------------------------------------------------------------------------------------------------
def _lit_size_format(mode, regen, comp, streams):
    if mode in ("raw", "rle"):
        return 0 if regen < 32 else (1 if regen < 4096 else 3)
    big = max(regen, comp)
    if streams == 1:
        assert big < 1024
        return 0
    return 1 if big < 1024 else (2 if big < 16384 else 3)


def literals_section(lit, st):
    mode, data = lit["mode"], bytes(lit.get("data", b""))
    regen = len(data)
    sf = lit.get("sf")
    if mode in ("raw", "rle"):
        if sf is None:
            sf = _lit_size_format(mode, regen, 0, 1)
        lt = 0 if mode == "raw" else 1
        if sf in (0, 2):
            hdr = bytes([lt | (sf << 2) | (regen << 3)])
            assert regen < 32
        elif sf == 1:
            assert regen < 4096
            hdr = (lt | (1 << 2) | (regen << 4)).to_bytes(2, "little")
        else:
            assert regen < (1 << 20)
            hdr = (lt | (3 << 2) | (regen << 4)).to_bytes(3, "little")
        if mode == "raw":
            return hdr + data
        assert len(set(data)) <= 1
        return hdr + bytes([lit.get("byte", data[0] if data else 0)])
    if mode == "huf":
        weights = lit.get("weights") or weights_for(data)
        tree = huffman_tree(weights, lit.get("wmode"), lit.get("wnorm"))
        st["huf"] = huffman_codes(weights)
    else:
        tree = b""
    codes = st["huf"]
    streams = lit.get("streams", 1 if regen < 256 else 4)
    if streams == 1:
        payload = tree + huffman_stream(data, codes)
    else:
        seg = (regen + 3) // 4
        parts = [huffman_stream(data[k * seg:(k + 1) * seg] if k < 3 else data[3 * seg:], codes) for k in range(4)]
        jump = b"".join(len(p).to_bytes(2, "little") for p in parts[:3])
        payload = tree + jump + b"".join(parts)
    comp = len(payload)
    if sf is None:
        sf = _lit_size_format(mode, regen, comp, streams)
    assert (sf == 0) == (streams == 1)
    lt = 2 if mode == "huf" else 3
    hh, bits = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[sf]
    assert regen < (1 << bits) and comp < (1 << bits), (regen, comp, sf)
    hdr = (lt | (sf << 2) | (regen << 4) | (comp << (4 + bits))).to_bytes(hh, "little")
    return hdr + payload


def ll_code(ll):
    return max(c for c in range(36) if zf.LL_BASE[c] <= ll)


def ml_code(ml):
    return max(c for c in range(53) if zf.ML_BASE[c] <= ml)


def seq_count(n, nbytes=None):
    if nbytes is None:
        nbytes = 1 if n < 128 else (2 if n < 0x7F00 else 3)
    if nbytes == 1:
        assert n < 128
        return bytes([n])
    if nbytes == 2:
        assert n < 0x8000
        return bytes([128 + (n >> 8), n & 255])
    assert 0x7F00 <= n < 0x7F00 + 65536
    return bytes([255]) + (n - 0x7F00).to_bytes(2, "little")


def sequences_section(seqs, modes, st, count_bytes=None):
    out = seq_count(len(seqs), count_bytes)
    if not seqs:
        return out
    codes = {"ll": [ll_code(s[0]) for s in seqs], "ml": [ml_code(s[1]) for s in seqs],
             "of": [s[2].bit_length() - 1 for s in seqs]}
    mb, tabs, body = 0, {}, b""
    for name, shift in (("ll", 6), ("of", 4), ("ml", 2)):
        m = modes.get(name, "predefined")
        if m == "predefined":
            norm, log = zf.PREDEF[name]
            tabs[name] = (zf.build_fse_table(norm, log), log)
            mb |= 0 << shift
        elif m == "repeat":
            tabs[name] = st["fse"][name]
            mb |= 3 << shift
        elif m[0] == "rle":
            tabs[name] = ([(m[1], 0, 0)], 0)
            body += bytes([m[1]])
            mb |= 1 << shift
        else:
            _, norm, log = m
            if norm is None:
                hist = [0] * (zf.MAX_SYM[name] + 1)
                for c in codes[name]:
                    hist[c] += 1
                norm = normalize(hist, log)
            tabs[name] = (zf.build_fse_table(list(norm), log), log)
            body += fse_description(norm, log)
            mb |= 2 << shift
    st["fse"] = dict(tabs)
    states = {}
    for name in ("ll", "of", "ml"):
        table, log = tabs[name]
        states[name] = fse_states(table, codes[name])
    items = [(states[n][0][0], tabs[n][1]) for n in ("ll", "of", "ml")]
    for i, (ll, ml, ov) in enumerate(seqs):
        oc, mc, lc = codes["of"][i], codes["ml"][i], codes["ll"][i]
        items += [(ov - (1 << oc), oc), (ml - zf.ML_BASE[mc], zf.ML_BITS[mc]), (ll - zf.LL_BASE[lc], zf.LL_BITS[lc])]
        if i + 1 < len(seqs):
            items += [states["ll"][1][i], states["ml"][1][i], states["of"][1][i]]
    return out + bytes([mb]) + body + backward(items)


def apply_sequences(out, lits, seqs, rep):
    """what the sequences produce after `out` (the frame's output so far); updates `rep` in place"""
    li = 0
    for ll, ml, ov in seqs:
        out += lits[li:li + ll]
        li += ll
        if ov > 3:
            off = ov - 3
            rep[:] = [off, rep[0], rep[1]]
        elif ll > 0:
            off = rep[ov - 1]
            if ov == 2:
                rep[:] = [rep[1], rep[0], rep[2]]
            elif ov == 3:
                rep[:] = [rep[2], rep[0], rep[1]]
        elif ov == 1:
            off = rep[1]
            rep[:] = [rep[1], rep[0], rep[2]]
        else:
            off = rep[2] if ov == 2 else rep[0] - 1
            rep[:] = [off, rep[0], rep[1]]
        assert 1 <= off <= len(out), ("offset out of range", off, len(out))
        for _ in range(ml):
            out.append(out[-off])
    assert li <= len(lits)
    out += lits[li:]


def block(b, st, out, last):
    """one block (header included); appends what it produces to `out`"""
    t = b["type"]
    if t == "raw":
        body, size, btype = bytes(b["data"]), len(b["data"]), 0
        out += body
    elif t == "rle":
        body, size, btype = bytes([b["byte"]]), b["size"], 1
        out += body * size
    else:
        lit = b["lit"]
        body = literals_section(lit, st)
        body += sequences_section(b.get("seqs", []), b.get("modes", {}), st, b.get("count_bytes"))
        size, btype = len(body), 2
        data = bytes(lit.get("data", b""))
        apply_sequences(out, data, b.get("seqs", []), st["rep"])
    size = b.get("bsize", size)
    last = b.get("last", last)
    return (int(last) | (btype << 1) | (size << 3)).to_bytes(3, "little") + body


def window_descriptor(size):
    """the smallest window descriptor whose window holds `size` bytes"""
    for wd in range(256):
        exp, mant = (wd >> 3) + 10, wd & 7
        if (1 << exp) + ((1 << exp) >> 3) * mant >= size:
            return wd
    raise ValueError(size)


def frame(blocks, *, single=None, wd=None, fcs="auto", fcs_bytes=None, did_bytes=0, checksum=False,
          reserved=False, bad_checksum=False, content=None):
    """a whole frame.  fcs="auto" writes the content size, fcs=None omits it; the window
    descriptor defaults to the smallest that holds the content and every block.
    Returns (frame bytes, content bytes)."""
    st = {"rep": [1, 4, 8]}
    out = bytearray()
    body, bigblock = b"", 1
    for i, b in enumerate(blocks):
        blk = block(b, st, out, i == len(blocks) - 1)
        body += blk
        bigblock = max(bigblock, len(blk) - 3)
    if content is None:
        content = bytes(out)
    n = len(content)
    if fcs == "auto":
        fcs = n
    if single is None:
        single = False
    if fcs is None:
        assert not single
        fcs_flag, fcs_field = 0, b""
    else:
        if fcs_bytes is None:
            fcs_bytes = 1 if (single and fcs < 256) else (2 if 256 <= fcs < 65536 + 256 else (4 if fcs < 1 << 32 else 8))
        if fcs_bytes == 1:
            assert single
            fcs_flag, fcs_field = 0, bytes([fcs])
        else:
            fcs_flag = {2: 1, 4: 2, 8: 3}[fcs_bytes]
            fcs_field = (fcs - 256 if fcs_bytes == 2 else fcs).to_bytes(fcs_bytes, "little")
    did_flag = {0: 0, 1: 1, 2: 2, 4: 3}[did_bytes]
    fhd = (fcs_flag << 6) | (int(single) << 5) | (int(checksum) << 2) | did_flag | (8 if reserved else 0)
    hdr = MAGIC.to_bytes(4, "little") + bytes([fhd])
    if not single:
        hdr += bytes([window_descriptor(max(n, bigblock)) if wd is None else wd])
    hdr += bytes(did_bytes) + fcs_field
    tail = b""
    if checksum:
        tail = ((xxh64(content) ^ (1 if bad_checksum else 0)) & 0xFFFFFFFF).to_bytes(4, "little")
    return hdr + body + tail, content


def skippable(payload, variant=0):
    return (SKIPPABLE + variant).to_bytes(4, "little") + len(payload).to_bytes(4, "little") + bytes(payload)

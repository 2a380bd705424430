"""A plain-Python zstd frame decoder (RFC 8878) that also reports what it parsed: test infrastructure for the zstd
encoder (csrc/dev_zstdenc.cuh).

It is written from the RFC, with its own copy of the RFC's code tables and predefined distributions, so that a
mistake shared by the library's encoder and decoder (which share dev_zstd.cuh's tables) still shows.  It is stricter
than ZSTD_decompress where the RFC allows it: every Huffman and sequence bitstream must be used up exactly, FSE
descriptions must sum exactly to 2^log within the RFC's accuracy limits, Huffman weights must give a complete tree,
no block may produce more than 128 KiB, and the content size must equal the bytes produced, with nothing after the
last block.  A content checksum is verified with XXH64; a dictionary-ID field must be zero (no dictionary).

decode_frame(data) -> (bytes, FrameInfo) for one frame that fills `data`.  decode_stream(data) -> (bytes, [FrameInfo])
decodes frames and skippable frames one after the other until `data` is used up, as ZSTD_decompress does.
FrameInfo.blocks holds one dict per block:
  {"type": "raw" | "rle" | "compressed", "size": bytes in the frame, "last": bool, "out": bytes produced,
   "lit": {...}, "seq": {...}}   (lit / seq for compressed blocks only)
lit: {"type": "raw" | "rle" | "compressed" | "treeless", "size_format": 0..3, "streams": 1 | 4, "regen": int,
      "comp": int, "weights": "direct" | "fse" | None, "weights_log": int | None, "max_bits": int, "lengths": [code length of
      each byte value, 0 if absent], "literals": bytes}
seq: {"count": int, "count_bytes": 1 | 2 | 3, "modes": {"ll": m, "of": m, "ml": m} (m: "predefined" | "rle" | "fse"
      | "repeat"), "logs": {...} (accuracy log of each FSE description), "zero_runs": {...} (the zero-count runs each
      FSE description spelled with repeat flags), "seqs": [(ll_code, ml_code, of_code, offset_value, offset, case,
      ll, ml, rep1 before it)]} with case one of "new", "rep1", "rep2", "rep3" (LL > 0), "rep2_ll0", "rep3_ll0",
      "rep1m1_ll0".
"""

MAGIC = 0xFD2FB528
BLOCK_MAX = 128 * 1024

# RFC 8878 3.1.1.3.2.1.1: literals length codes (baseline, extra bits)
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384,
                             32768, 65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
# match length codes
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195,
                                16387, 32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
# RFC 8878 3.1.1.3.2.2: predefined distributions (accuracy logs 6, 6, 5)
LL_NORM = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1,
           -1, -1, -1, -1]
ML_NORM = [1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7
OF_NORM = [1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5
PREDEF = {"ll": (LL_NORM, 6), "of": (OF_NORM, 5), "ml": (ML_NORM, 6)}
MAX_LOG = {"ll": 9, "of": 8, "ml": 9}
MAX_SYM = {"ll": 35, "of": 31, "ml": 52}
MODES = ("predefined", "rle", "fse", "repeat")


M64 = (1 << 64) - 1


# ---------------------------------------------------------------------------------------------------------------
# XXH64 (seed 0 by default), for content checksums
# ---------------------------------------------------------------------------------------------------------------
_P1, _P2, _P3, _P4, _P5 = (11400714785074694791, 14029467366897019727, 1609587929392839161, 9650029242287828579,
                           2870177450012600261)


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def _round(acc, lane):
    return (_rotl((acc + lane * _P2) & M64, 31) * _P1) & M64


def xxh64(data, seed=0):
    data = bytes(data)
    n, p = len(data), 0
    if n >= 32:
        v = [(seed + _P1 + _P2) & M64, (seed + _P2) & M64, seed, (seed - _P1) & M64]
        while p + 32 <= n:
            for i in range(4):
                v[i] = _round(v[i], int.from_bytes(data[p:p + 8], "little"))
                p += 8
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & M64
        for i in range(4):
            h = ((h ^ _round(0, v[i])) * _P1 + _P4) & M64
    else:
        h = (seed + _P5) & M64
    h = (h + n) & M64
    while p + 8 <= n:
        h ^= _round(0, int.from_bytes(data[p:p + 8], "little"))
        h = (_rotl(h, 27) * _P1 + _P4) & M64
        p += 8
    if p + 4 <= n:
        h ^= (int.from_bytes(data[p:p + 4], "little") * _P1) & M64
        h = (_rotl(h, 23) * _P2 + _P3) & M64
        p += 4
    while p < n:
        h ^= (data[p] * _P5) & M64
        h = (_rotl(h, 11) * _P1) & M64
        p += 1
    h ^= h >> 33
    h = (h * _P2) & M64
    h ^= h >> 29
    h = (h * _P3) & M64
    h ^= h >> 32
    return h



class ZstdError(Exception):
    pass


def _check(cond, what):
    if not cond:
        raise ZstdError(what)


def _hb(v):
    return v.bit_length() - 1


class FrameInfo:
    def __init__(self):
        self.fhd = 0
        self.fcs_bytes = 0
        self.fcs = None
        self.single_segment = False
        self.checksum = False
        self.window = None
        self.did_bytes = 0
        self.blocks = []


class _Fwd:
    """forward bit reader (LSB first), for FSE descriptions"""

    def __init__(self, data, start, end):
        self.d, self.pos, self.end = data, start * 8, end * 8

    def read(self, n):
        _check(self.pos + n <= self.end, "FSE description runs past its bytes")
        lo = self.pos >> 3
        v = int.from_bytes(self.d[lo:((self.pos + n + 7) >> 3)], "little") >> (self.pos & 7)
        self.pos += n
        return v & ((1 << n) - 1)

    def peek(self, n):
        lo = self.pos >> 3
        v = int.from_bytes(self.d[lo:min((self.pos + n + 7) >> 3, self.end >> 3)], "little") >> (self.pos & 7)
        return v & ((1 << n) - 1)


class _Back:
    """backward bit reader over data[a:b) (RFC 8878 4.1: read from the end, after the end mark); reads past the
    start yield zeros and are counted as overflow"""

    def __init__(self, data, a, b):
        _check(b > a, "empty bitstream")
        last = data[b - 1]
        _check(last != 0, "bitstream without an end mark in its last byte")
        self.d, self.a = data, a
        self.pos = (b - 1 - a) * 8 + _hb(last)          # bits below the end mark

    def read(self, n):
        if n == 0:
            return 0
        self.pos -= n
        p = self.pos
        if p < 0:
            v = self.peek_at(0, n + p) << -p if n + p > 0 else 0
            return v
        return self.peek_at(p, n)

    def peek(self, n):
        p = self.pos - n
        if p < 0:
            return (self.peek_at(0, self.pos) << -p) if self.pos > 0 else 0
        return self.peek_at(p, n)

    def peek_at(self, p, n):
        lo = self.a + (p >> 3)
        hi = self.a + ((p + n + 7) >> 3)
        return (int.from_bytes(self.d[lo:hi], "little") >> (p & 7)) & ((1 << n) - 1)


def read_fse_description(data, start, end, max_log, max_sym):
    """RFC 8878 4.1.1: returns (normalised counts, accuracy log, bytes used, zero runs)"""
    br = _Fwd(data, start, end)
    log = br.read(4) + 5
    _check(log <= max_log, f"accuracy log {log} above {max_log}")
    remaining = (1 << log) + 1
    threshold = 1 << log
    nbits = log + 1
    norm, runs = [], []
    while remaining > 1:
        _check(len(norm) <= max_sym, "FSE description has too many symbols")
        mx = (2 * threshold - 1) - remaining
        low = br.peek(nbits - 1)
        if low < mx:
            count = low
            br.read(nbits - 1)
        else:
            count = br.peek(nbits)
            if count >= threshold:
                count -= mx
            br.read(nbits)
        count -= 1
        norm.append(count)
        remaining -= abs(count)
        _check(remaining >= 1, "FSE description sums past 2^log")
        while remaining < threshold:
            nbits -= 1
            threshold >>= 1
        if count == 0:
            run = 0
            while True:
                flag = br.read(2)
                run += flag
                if flag != 3:
                    break
            if run:
                runs.append(run)
            norm.extend([0] * run)
            _check(len(norm) <= max_sym + 1, "zero run past the last symbol")
    _check(remaining == 1, "FSE description does not sum to 2^log")
    _check(len(norm) <= max_sym + 1, "FSE description has too many symbols")
    return norm, log, (br.pos + 7) // 8 - start, runs


def build_fse_table(norm, log):
    """RFC 8878 4.1.1: decoding table of (symbol, nbBits, baseline)"""
    size = 1 << log
    sym = [0] * size
    high = size - 1
    nxt = []
    for s, c in enumerate(norm):
        if c == -1:
            sym[high] = s
            high -= 1
            nxt.append(1)
        else:
            nxt.append(c)
    step = (size >> 1) + (size >> 3) + 3
    pos = 0
    for s, c in enumerate(norm):
        for _ in range(max(c, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    _check(pos == 0, "FSE spread did not return to 0")
    table = []
    for u in range(size):
        s = sym[u]
        ns = nxt[s]
        nxt[s] += 1
        nb = log - _hb(ns)
        table.append((s, nb, (ns << nb) - size))
    return table


class _Fse:
    def __init__(self, table, log, rle=None):
        self.t, self.log, self.rle = table, log, rle

    def init(self, br):
        self.state = 0 if self.rle is not None else br.read(self.log)

    def sym(self):
        return self.rle if self.rle is not None else self.t[self.state][0]

    def update(self, br):
        if self.rle is None:
            _, nb, base = self.t[self.state]
            self.state = base + br.read(nb)


def _huffman_weights(data, p, end):
    """RFC 8878 4.2.1: returns (weights of the listed symbols, bytes used, "direct" | "fse", log)"""
    _check(p < end, "no Huffman tree description")
    hb = data[p]
    if hb >= 128:
        nw = hb - 127
        nbytes = (nw + 1) // 2
        _check(p + 1 + nbytes <= end, "direct weights past the literals section")
        w = []
        for i in range(nw):
            b = data[p + 1 + i // 2]
            w.append(b >> 4 if i % 2 == 0 else b & 15)
        return w, 1 + nbytes, "direct", None
    _check(hb > 0 and p + 1 + hb <= end, "bad FSE-coded weights size")
    norm, log, used, _ = read_fse_description(data, p + 1, p + 1 + hb, 6, 12)
    table = build_fse_table(norm, log)
    br = _Back(data, p + 1 + used, p + 1 + hb)
    s1, s2 = _Fse(table, log), _Fse(table, log)
    s1.init(br)
    s2.init(br)
    _check(br.pos >= 0, "weight stream shorter than its states")
    w = []
    while True:                                   # the two states alternate; overflow ends it (RFC 8878 4.2.1.2)
        _check(len(w) < 255, "more than 255 weights")
        w.append(s1.sym())
        s1.update(br)
        if br.pos < 0:
            w.append(s2.sym())
            break
        _check(len(w) < 255, "more than 255 weights")
        w.append(s2.sym())
        s2.update(br)
        if br.pos < 0:
            w.append(s1.sym())
            break
    return w, 1 + hb, "fse", log


def _huffman_table(weights):
    """weights of symbols 0..n-2 -> (decode table indexed by max_bits bits: (symbol, nbits), max_bits)"""
    _check(all(x <= 11 for x in weights), "Huffman weight above 11")
    total = sum(1 << (x - 1) for x in weights if x)
    _check(total > 0, "all Huffman weights zero")
    maxb = _hb(total) + 1
    _check(maxb <= 11, "Huffman code longer than 11 bits")
    left = (1 << maxb) - total
    _check(left > 0 and left & (left - 1) == 0, "Huffman weights do not give a complete tree")
    weights = list(weights) + [_hb(left) + 1]
    _check(len(weights) <= 256, "more than 256 Huffman symbols")
    n1 = sum(1 for x in weights if x == 1)
    _check(n1 >= 2 and n1 % 2 == 0, "odd count of longest Huffman codes")
    table = [None] * (1 << maxb)
    at = 0
    for wt in range(1, maxb + 1):
        for s, x in enumerate(weights):
            if x == wt:
                span = 1 << (wt - 1)
                for i in range(at, at + span):
                    table[i] = (s, maxb + 1 - wt)
                at += span
    _check(at == 1 << maxb, "Huffman table not full")
    return table, maxb


def _huffman_stream(data, a, b, n, table, maxb):
    br = _Back(data, a, b)
    out = bytearray(n)
    for i in range(n):
        s, nb = table[br.peek(maxb)]
        out[i] = s
        br.pos -= nb
        _check(br.pos >= 0, "Huffman stream overread")
    _check(br.pos == 0, f"Huffman stream not used up ({br.pos} bits left)")
    return bytes(out)


def _literals(data, p, end, st):
    b0 = data[p]
    lt, sf = b0 & 3, (b0 >> 2) & 3
    lit = {"type": ("raw", "rle", "compressed", "treeless")[lt], "size_format": sf, "streams": None, "comp": None,
           "weights": None, "weights_log": None, "max_bits": None}
    if lt < 2:
        if sf in (0, 2):                          # one bit of size format: 0b00 and 0b10 are the same form
            regen, hh = b0 >> 3, 1
            lit["size_format"] = 0
        elif sf == 1:
            _check(p + 2 <= end, "literals header")
            regen, hh = (b0 >> 4) | (data[p + 1] << 4), 2
        else:
            _check(p + 3 <= end, "literals header")
            regen, hh = (b0 >> 4) | (data[p + 1] << 4) | (data[p + 2] << 12), 3
        _check(regen <= BLOCK_MAX, "literals above 128 KiB")
        lit["regen"] = regen
        if lt == 0:
            _check(p + hh + regen <= end, "raw literals past the block")
            lit["literals"] = bytes(data[p + hh:p + hh + regen])
            return lit, hh + regen
        _check(p + hh + 1 <= end, "RLE literal past the block")
        lit["literals"] = bytes([data[p + hh]]) * regen
        return lit, hh + 1
    hh, bits = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[sf]
    _check(p + hh <= end, "literals header")
    h = int.from_bytes(data[p:p + hh], "little")
    regen, comp = (h >> 4) & ((1 << bits) - 1), (h >> (4 + bits)) & ((1 << bits) - 1)
    _check(regen <= BLOCK_MAX, "literals above 128 KiB")
    _check(p + hh + comp <= end, "compressed literals past the block")
    streams = 1 if sf == 0 else 4
    lit.update(regen=regen, comp=comp, streams=streams)
    q, qend = p + hh, p + hh + comp
    if lt == 2:
        w, used, kind, wlog = _huffman_weights(data, q, qend)
        table, maxb = _huffman_table(w)
        st["huf"] = (table, maxb)
        lit.update(weights=kind, weights_log=wlog)
        q += used
    else:
        _check(st.get("huf") is not None, "treeless literals without a previous table")
        table, maxb = st["huf"]
    lit["max_bits"] = maxb
    lengths = [0] * 256
    for sym, nb in table:
        lengths[sym] = nb
    lit["lengths"] = lengths
    if streams == 1:
        lit["literals"] = _huffman_stream(data, q, qend, regen, table, maxb)
    else:
        _check(q + 6 <= qend, "jump table")
        s = [data[q] | data[q + 1] << 8, data[q + 2] | data[q + 3] << 8, data[q + 4] | data[q + 5] << 8]
        s.append(qend - q - 6 - sum(s))
        _check(s[3] > 0, "fourth Huffman stream empty")
        lit["stream_sizes"] = s
        seg = (regen + 3) // 4
        _check(regen - 3 * seg >= 0, "four streams of fewer than 4 literals")
        out, a = b"", q + 6
        for k in range(4):
            out += _huffman_stream(data, a, a + s[k], seg if k < 3 else regen - 3 * seg, table, maxb)
            a += s[k]
        lit["literals"] = out
    return lit, qend - p


def _sequences(data, p, end, st, lits, out, frame_start):
    _check(p < end, "no sequences section")
    b0 = data[p]
    if b0 < 128:
        ns, nb = b0, 1
    elif b0 < 255:
        _check(p + 2 <= end, "sequence count")
        ns, nb = ((b0 - 128) << 8) + data[p + 1], 2
    else:
        _check(p + 3 <= end, "sequence count")
        ns, nb = data[p + 1] + (data[p + 2] << 8) + 0x7F00, 3
    seq = {"count": ns, "count_bytes": nb, "modes": {}, "logs": {}, "zero_runs": {}, "seqs": []}
    p += nb
    if ns == 0:
        _check(p == end, "bytes after a sequences section of no sequences")
        out += lits
        return seq
    _check(p < end, "no symbol compression modes")
    mb = data[p]
    p += 1
    _check(mb & 3 == 0, "reserved bits of the modes byte set")
    dec = {}
    for name, shift in (("ll", 6), ("of", 4), ("ml", 2)):
        m = MODES[(mb >> shift) & 3]
        seq["modes"][name] = m
        if m == "predefined":
            norm, log = PREDEF[name]
            dec[name] = _Fse(build_fse_table(norm, log), log)
        elif m == "rle":
            _check(p < end, "RLE symbol")
            _check(data[p] <= MAX_SYM[name], "RLE symbol out of range")
            dec[name] = _Fse(None, 0, data[p])
            p += 1
        elif m == "fse":
            norm, log, used, runs = read_fse_description(data, p, end, MAX_LOG[name], MAX_SYM[name])
            seq["logs"][name], seq["zero_runs"][name] = log, runs
            dec[name] = _Fse(build_fse_table(norm, log), log)
            p += used
        else:
            _check(name in st.get("fse", {}), "repeat mode without a previous table")
            dec[name] = st["fse"][name]
    st["fse"] = dec
    br = _Back(data, p, end)
    lld, ofd, mld = dec["ll"], dec["of"], dec["ml"]
    lld.init(br)
    ofd.init(br)
    mld.init(br)
    rep = st["rep"]
    li = 0
    for i in range(ns):
        oc, mc, lc = ofd.sym(), mld.sym(), lld.sym()
        _check(lc <= 35 and mc <= 52 and oc <= 31, "code out of range")
        ofv = (1 << oc) + br.read(oc)
        ml = ML_BASE[mc] + br.read(ML_BITS[mc])
        ll = LL_BASE[lc] + br.read(LL_BITS[lc])
        r1_before = rep[0]
        if ofv > 3:                             # RFC 8878 3.1.2.5
            off, case = ofv - 3, "new"
            rep[:] = [off, rep[0], rep[1]]
        elif ll > 0:
            case = ("rep1", "rep2", "rep3")[ofv - 1]
            off = rep[ofv - 1]
            if ofv == 2:
                rep[:] = [rep[1], rep[0], rep[2]]
            elif ofv == 3:
                rep[:] = [rep[2], rep[0], rep[1]]
        else:
            case = ("rep2_ll0", "rep3_ll0", "rep1m1_ll0")[ofv - 1]
            if ofv == 1:
                off = rep[1]
                rep[:] = [rep[1], rep[0], rep[2]]
            else:
                off = rep[2] if ofv == 2 else rep[0] - 1
                _check(off > 0, "offset 0 from rep1 - 1")
                rep[:] = [off, rep[0], rep[1]]
        seq["seqs"].append((lc, mc, oc, ofv, off, case, ll, ml, r1_before))
        _check(li + ll <= len(lits), "sequences use more literals than the block has")
        out += lits[li:li + ll]
        li += ll
        pos = len(out) - frame_start
        _check(1 <= off <= pos, f"offset {off} reaches before the frame ({pos} bytes produced)")
        if off >= ml:
            out += out[len(out) - off:len(out) - off + ml]
        else:
            pat = bytes(out[len(out) - off:])
            out += (pat * (ml // off + 1))[:ml]
        if i + 1 < ns:
            lld.update(br)
            mld.update(br)
            ofd.update(br)
        _check(br.pos >= 0, "sequence bitstream overread")
    _check(br.pos == 0, f"sequence bitstream not used up ({br.pos} bits left)")
    out += lits[li:]
    return seq


def decode_frame(data):
    """one frame, which must fill `data` exactly -> (bytes, FrameInfo)"""
    data = bytes(data)
    out, info, end = _frame(data, 0)
    _check(end == len(data), f"{len(data) - end} bytes after the last block")
    return out, info


def decode_stream(data):
    """frames and skippable frames until `data` is used up -> (bytes, [FrameInfo of each frame])"""
    data = bytes(data)
    out, infos, p = b"", [], 0
    while p < len(data):
        _check(len(data) - p >= 5, "1 to 4 bytes after the last frame")
        magic = int.from_bytes(data[p:p + 4], "little")
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            _check(len(data) - p >= 8, "skippable frame header past the data")
            n = int.from_bytes(data[p + 4:p + 8], "little")
            _check(p + 8 + n <= len(data), "skippable frame past the data")
            p += 8 + n
            continue
        o, info, p = _frame(data, p)
        out += o
        infos.append(info)
    return out, infos


def _frame(data, start):
    """the frame at data[start:] -> (bytes, FrameInfo, end of the frame)"""
    info = FrameInfo()
    _check(len(data) - start >= 6 and int.from_bytes(data[start:start + 4], "little") == MAGIC, "no zstd frame magic")
    fhd = data[start + 4]
    info.fhd = fhd
    fcs_flag, single, cks, dict_flag = fhd >> 6, bool(fhd & 0x20), bool(fhd & 4), fhd & 3
    _check(not fhd & 8, "reserved frame header bit set")
    info.single_segment = single
    info.checksum = cks
    p = start + 5
    window = None
    if not single:
        _check(p < len(data), "frame header past the data")
        wd = data[p]
        exp, mant = (wd >> 3) + 10, wd & 7
        _check(exp <= 31, "window above 2 GiB")
        window = (1 << exp) + ((1 << exp) >> 3) * mant
        info.window = window
        p += 1
    did_bytes = (0, 1, 2, 4)[dict_flag]
    info.did_bytes = did_bytes
    _check(p + did_bytes <= len(data), "frame header past the data")
    _check(not any(data[p:p + did_bytes]), "a dictionary is required")
    p += did_bytes
    fcs_bytes = (1 if single else 0, 2, 4, 8)[fcs_flag]
    info.fcs_bytes = fcs_bytes
    _check(p + fcs_bytes <= len(data), "frame header past the data")
    if fcs_bytes:
        fcs = int.from_bytes(data[p:p + fcs_bytes], "little")
        info.fcs = fcs + 256 if fcs_bytes == 2 else fcs
    p += fcs_bytes
    if single:
        window = info.fcs
    bmax = min(BLOCK_MAX, window) if window is not None else BLOCK_MAX
    out = bytearray()
    st = {"rep": [1, 4, 8]}
    while True:
        _check(p + 3 <= len(data), "block header past the data")
        bh = int.from_bytes(data[p:p + 3], "little")
        last, btype, bsize = bool(bh & 1), (bh >> 1) & 3, bh >> 3
        p += 3
        _check(btype != 3, "reserved block type")
        blk = {"type": ("raw", "rle", "compressed")[btype], "size": bsize, "last": last}
        before = len(out)
        if btype == 0:
            _check(p + bsize <= len(data), "raw block past the data")
            out += data[p:p + bsize]
            p += bsize
        elif btype == 1:
            _check(p + 1 <= len(data), "RLE block past the data")
            out += bytes([data[p]]) * bsize
            p += 1
        else:
            _check(bsize <= bmax, "compressed block above the block maximum")
            end = p + bsize
            _check(end <= len(data), "compressed block past the data")
            lit, used = _literals(data, p, end, st)
            blk["lit"] = lit
            blk["seq"] = _sequences(data, p + used, end, st, lit["literals"], out, 0)
            p = end
        blk["out"] = len(out) - before
        blk["rep_after"] = tuple(st["rep"])
        _check(blk["out"] <= bmax, "block produced more than the block maximum")
        info.blocks.append(blk)
        if last:
            break
    if info.fcs is not None:
        _check(info.fcs == len(out), f"content size {info.fcs} but {len(out)} bytes produced")
    if cks:
        _check(p + 4 <= len(data), "checksum past the data")
        _check(int.from_bytes(data[p:p + 4], "little") == xxh64(bytes(out)) & 0xFFFFFFFF, "wrong content checksum")
        p += 4
    return bytes(out), info, p


def huffman_depth(literals):
    """depth of an unconstrained Huffman tree over the byte histogram of `literals` (0 for fewer than 2 symbols)"""
    import heapq
    counts = {}
    for b in literals:
        counts[b] = counts.get(b, 0) + 1
    if len(counts) < 2:
        return 0
    heap = [(c, 0, i) for i, c in enumerate(counts.values())]
    heapq.heapify(heap)
    k = len(heap)
    while len(heap) > 1:
        c1, d1, _ = heapq.heappop(heap)
        c2, d2, _ = heapq.heappop(heap)
        heapq.heappush(heap, (c1 + c2, max(d1, d2) + 1, k))
        k += 1
    return heap[0][1]

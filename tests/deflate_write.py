"""A plain-Python DEFLATE (RFC 1951) / zlib (RFC 1950) writer that writes exactly what it is told: test
infrastructure for the inflate decoder (csrc/dev_inflate.cuh).

Blocks are stored, fixed or dynamic.  A dynamic block takes its code lengths as given (complete or not, over-
subscribed or not), and HLIT / HDIST / HCLEN, the code-length code and the run-length items that spell the lengths
may each be set by hand, so malformed headers can be written as easily as valid ones.  Block contents are lists of
items:
  int 0..255                     a literal
  ("match", length, distance)    a length / distance pair, coded with the usual codes and extra bits
  ("len", code, extra)           length code 257..287 with an explicit extra-bits value
  ("dist", code, extra)          distance code 0..31 with an explicit extra-bits value
  ("bits", value, n)             raw bits
The end-of-block code 256 is appended unless end=False.  Huffman codes are canonical (RFC 1951 3.2.2) and written
most significant bit first; everything else least significant bit first.
"""
import zlib

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258]
LEN_EXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXT = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32


class Bits:
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value, nbits):
        assert 0 <= value < (1 << nbits) or nbits == 0, (value, nbits)
        self.v |= value << self.n
        self.n += nbits

    def code(self, code, length):
        """a Huffman code, most significant bit first"""
        self.put(int(format(code, f"0{length}b")[::-1], 2) if length else 0, length)

    def align(self):
        self.n += -self.n % 8

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def canonical(lengths):
    """RFC 1951 3.2.2: {symbol: (code, length)} for the symbols of nonzero length (used as given, even when the
    lengths do not make a prefix code)"""
    maxb = max(lengths + [0])
    count = [0] * (maxb + 2)
    for x in lengths:
        if x:
            count[x] += 1
    nxt, code = [0] * (maxb + 2), 0
    for b in range(1, maxb + 1):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = {}
    for s, x in enumerate(lengths):
        if x:
            out[s] = (nxt[x] & ((1 << x) - 1), x)
            nxt[x] += 1
    return out


def _len_code(length):
    c = max(i for i in range(29) if LEN_BASE[i] <= length)
    return 257 + c, length - LEN_BASE[c], LEN_EXT[c]


def _dist_code(dist):
    c = max(i for i in range(30) if DIST_BASE[i] <= dist)
    return c, dist - DIST_BASE[c], DIST_EXT[c]


def _items(w, items, lit, dist, end):
    for it in list(items) + ([256] if end else []):
        if isinstance(it, int):
            w.code(*lit[it])
        elif it[0] == "match":
            lc, le, ln = _len_code(it[1])
            w.code(*lit[lc])
            w.put(le, ln)
            dc, de, dn = _dist_code(it[2])
            w.code(*dist[dc])
            w.put(de, dn)
        elif it[0] == "len":
            w.code(*lit[it[1]])
            w.put(it[2], LEN_EXT[it[1] - 257] if it[1] < 286 else 0)
        elif it[0] == "dist":
            w.code(*dist[it[1]])
            w.put(it[2], DIST_EXT[it[1]] if it[1] < 30 else 0)
        else:
            w.put(it[1], it[2])


def stored(w, data, final=False, length=None, nlength=None):
    w.put(int(final), 1)
    w.put(0, 2)
    w.align()
    n = len(data) if length is None else length
    w.put(n, 16)
    w.put((~n & 0xFFFF) if nlength is None else nlength, 16)
    for b in data:
        w.put(b, 8)


def fixed(w, items, final=False, end=True):
    w.put(int(final), 1)
    w.put(1, 2)
    _items(w, items, canonical(FIXED_LIT), canonical(FIXED_DIST), end)


def dynamic(w, lit_lengths, dist_lengths, items, final=False, end=True, hlit=None, hdist=None, hclen=None,
            cl_lengths=None, cl_items=None):
    """lit_lengths / dist_lengths: code lengths as given; cl_items: the code-length symbols as (symbol, extra) --
    by default every length spelled as itself; cl_lengths: the code-length code's 19 lengths (by default a flat
    complete code over the symbols used)"""
    nlit, ndist = len(lit_lengths), len(dist_lengths)
    if cl_items is None:
        cl_items = [(x, 0) for x in list(lit_lengths) + list(dist_lengths)]
    if cl_lengths is None:
        used = sorted({s for s, _ in cl_items})
        if len(used) == 1:
            used.append(0 if used[0] else 1)
        nb = (len(used) - 1).bit_length()
        nshort = (1 << nb) - len(used)
        cl_lengths = [0] * 19
        for i, s in enumerate(used):
            cl_lengths[s] = nb - 1 if i < nshort else nb
    ordered = [cl_lengths[s] for s in CL_ORDER]
    if hclen is None:
        hclen = max(4, max((i + 1 for i, x in enumerate(ordered) if x), default=4))
    w.put(int(final), 1)
    w.put(2, 2)
    w.put(nlit - 257 if hlit is None else hlit, 5)
    w.put(ndist - 1 if hdist is None else hdist, 5)
    w.put(hclen - 4, 4)
    for x in ordered[:hclen]:
        w.put(x, 3)
    cl = canonical(list(cl_lengths))
    for s, extra in cl_items:
        w.code(*cl[s])
        w.put(extra, {16: 2, 17: 3, 18: 7}.get(s, 0))
    _items(w, items, canonical(list(lit_lengths)), canonical(list(dist_lengths)), end)


def zlib_stream(body, content, cmf=0x78, flg=None, fdict=False, adler=None):
    """RFC 1950 framing around a DEFLATE body: header (FCHECK made right unless flg is given), Adler-32 of
    `content` (or `adler`)"""
    if flg is None:
        flg = 0x20 if fdict else 0
        flg += (31 - ((cmf << 8) | flg) % 31) % 31
    a = zlib.adler32(content) if adler is None else adler
    return bytes([cmf, flg]) + body + a.to_bytes(4, "big")


def lit_lengths(codes, n=257):
    """a literal/length length list of n entries with the given {symbol: length}"""
    out = [0] * n
    for s, x in codes.items():
        out[s] = x
    return out

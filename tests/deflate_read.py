"""A plain-Python reader of zlib streams (RFC 1950 / RFC 1951) that reports how each DEFLATE block was written.

It decodes the stream and returns, per block, its BFINAL and BTYPE, and for dynamic blocks HLIT, HDIST, HCLEN, the
code-length code, the literal/length and distance code lengths and the code-length symbols used with their repeat
counts.  Stored blocks report their LEN.  It raises ValueError on anything inflate() would refuse, and also on codes
that are incomplete where zlib's inflate_table refuses them, so a test can name the branch of the encoder it reached."""

ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
LBASE = (3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258)
LEXT = (0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0)
DBASE = (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
         6145, 8193, 12289, 16385, 24577)
DEXT = (0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13)


class _Bits:
    def __init__(self, data, pos):
        self.d, self.pos, self.bit = data, pos, 0

    def get(self, n):
        v = 0
        for i in range(n):
            if self.pos >= len(self.d):
                raise ValueError("input ends inside the stream")
            v |= ((self.d[self.pos] >> self.bit) & 1) << i
            self.bit += 1
            if self.bit == 8:
                self.bit, self.pos = 0, self.pos + 1
        return v

    def align(self):
        if self.bit:
            self.bit, self.pos = 0, self.pos + 1


def _table(lengths, kind):
    """canonical decoding table {(length, code): symbol}; kind 'cl' must be complete, 'lit'/'dist' may be a lone
    1-bit code (inftrees.c)"""
    count = [0] * 16
    for n in lengths:
        count[n] += 1
    count[0] = 0
    left = 1
    for n in range(1, 16):
        left = 2 * left - count[n]
        if left < 0:
            raise ValueError(f"over-subscribed {kind} code")
    if left > 0 and any(lengths) and (kind == "cl" or max(lengths) != 1):
        raise ValueError(f"incomplete {kind} code")
    code, nxt = 0, [0] * 16
    for n in range(1, 16):
        code = (code + count[n - 1]) << 1
        nxt[n] = code
    t = {}
    for s, n in enumerate(lengths):
        if n:
            t[(n, nxt[n])] = s
            nxt[n] += 1
    return t


def _sym(b, t):
    code = 0
    for n in range(1, 16):
        code = (code << 1) | b.get(1)
        if (n, code) in t:
            return t[(n, code)]
    raise ValueError("no such code")


def read(stream):
    """-> (output bytes, [block dict]); the zlib header and the Adler-32 are checked"""
    d = bytes(stream)
    if len(d) < 6 or d[0] & 15 != 8 or d[0] >> 4 > 7 or ((d[0] << 8) | d[1]) % 31 or d[1] & 0x20:
        raise ValueError("bad zlib header")
    b, out, blocks = _Bits(d, 2), bytearray(), []
    while True:
        final, btype = b.get(1), b.get(2)
        blk = {"bfinal": final, "btype": btype, "start": len(out)}
        if btype == 0:
            b.align()
            ln, nln = b.get(16), b.get(16)
            if ln != (~nln & 0xffff):
                raise ValueError("stored LEN / NLEN mismatch")
            blk["len"] = ln
            out += bytes(b.get(8) for _ in range(ln))
        elif btype == 3:
            raise ValueError("reserved block type")
        else:
            if btype == 1:
                ll = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
                dl = [5] * 32                                 # 30 and 31 occur in no valid stream
            else:
                hlit, hdist, hclen = b.get(5) + 257, b.get(5) + 1, b.get(4) + 4
                if hlit > 286 or hdist > 30:
                    raise ValueError("too many length or distance symbols")
                cl = [0] * 19
                for i in range(hclen):
                    cl[ORDER[i]] = b.get(3)
                ct = _table(cl, "cl")
                lens, items = [], []
                while len(lens) < hlit + hdist:
                    s = _sym(b, ct)
                    if s < 16:
                        lens.append(s)
                        items.append((s, 1))
                        continue
                    if s == 16:
                        if not lens:
                            raise ValueError("repeat with no first length")
                        r, v = 3 + b.get(2), lens[-1]
                    elif s == 17:
                        r, v = 3 + b.get(3), 0
                    else:
                        r, v = 11 + b.get(7), 0
                    if len(lens) + r > hlit + hdist:
                        raise ValueError("too many code lengths")
                    lens += [v] * r
                    items.append((s, r))
                ll, dl = lens[:hlit], lens[hlit:]
                if ll[256] == 0:
                    raise ValueError("no end-of-block code")
                blk.update(hlit=hlit, hdist=hdist, hclen=hclen, cl=cl, items=items)
            blk["ll"], blk["dl"] = ll, dl
            lt, dt = _table(ll, "lit"), _table(dl, "dist")
            nlit = nmatch = 0
            lengths, dists = set(), set()
            while True:
                s = _sym(b, lt)
                if s < 256:
                    out.append(s)
                    nlit += 1
                    continue
                if s == 256:
                    break
                if s > 285:
                    raise ValueError("invalid length symbol")
                n = LBASE[s - 257] + b.get(LEXT[s - 257])
                ds = _sym(b, dt)
                if ds > 29:
                    raise ValueError("invalid distance symbol")
                dist = DBASE[ds] + b.get(DEXT[ds])
                if dist > len(out):
                    raise ValueError("distance too far back")
                for _ in range(n):
                    out.append(out[-dist])
                nmatch += 1
                lengths.add(n)
                dists.add(dist)
            blk.update(nlit=nlit, nmatch=nmatch, lengths=lengths, dists=dists)
        blk["end"] = len(out)
        blocks.append(blk)
        if final:
            break
    b.align()
    if b.pos + 4 != len(d):
        raise ValueError("trailer is not the last 4 bytes")
    a, c = 1, 0
    for x in out:
        a = (a + x) % 65521
        c = (c + a) % 65521
    if int.from_bytes(d[b.pos:b.pos + 4], "big") != (c << 16) | a:
        raise ValueError("Adler-32 mismatch")
    return bytes(out), blocks

"""A snappy stream reader written from snappy's format_description.txt, independent of the library's decoder.

read(stream, n) returns (decoded bytes, None) or (None, reason) with the checks of snappy_uncompress plus Blosc's size
check: the preamble is a varint of at most 5 bytes that fits in 32 bits and equals n; offset 0 and offsets past the
output produced so far, and any tag, length or offset past the input or element past the output are refused, as are
input left over once the output is full and input that ends before it.  elements(stream) lists the parsed elements.
"""

REASONS = ("preamble", "length", "tag_input", "literal_input", "output", "offset", "leftover", "short")


def _preamble(s):
    v = 0
    for k in range(5):
        if k >= len(s):
            return None, 0
        b = s[k]
        if k == 4 and b >= 16:
            return None, 0
        v |= (b & 127) << (7 * k)
        if b < 128:
            return v, k + 1
    return None, 0


def elements(s):
    """[(kind, length, offset)] with kind 'lit' (offset = input position of the literals), 'c1', 'c2' or 'c4'"""
    v, ip = _preamble(s)
    assert v is not None
    out = []
    while ip < len(s):
        tag = s[ip]
        ip += 1
        t = tag & 3
        if t == 0:
            ln = (tag >> 2) + 1
            if ln > 60:
                nb = ln - 60
                ln = int.from_bytes(s[ip:ip + nb], "little") + 1
                ip += nb
            out.append(("lit", ln, ip))
            ip += ln
        elif t == 1:
            out.append(("c1", 4 + ((tag >> 2) & 7), ((tag >> 5) << 8) | s[ip]))
            ip += 1
        elif t == 2:
            out.append(("c2", (tag >> 2) + 1, int.from_bytes(s[ip:ip + 2], "little")))
            ip += 2
        else:
            out.append(("c4", (tag >> 2) + 1, int.from_bytes(s[ip:ip + 4], "little")))
            ip += 4
    return out


def read(s, n):
    s = bytes(s)
    v, ip = _preamble(s)
    if v is None:
        return None, "preamble"
    if v != n:
        return None, "length"
    out = bytearray()
    while len(out) < n:
        if ip >= len(s):
            return None, "short"
        tag = s[ip]
        ip += 1
        t = tag & 3
        if t == 0:
            ln = (tag >> 2) + 1
            if ln > 60:
                nb = ln - 60
                if ip + nb > len(s):
                    return None, "tag_input"
                ln = int.from_bytes(s[ip:ip + nb], "little") + 1
                ip += nb
            if ln > len(s) - ip:
                return None, "literal_input"
            if ln > n - len(out):
                return None, "output"
            out += s[ip:ip + ln]
            ip += ln
            continue
        nb = (1, 2, 4)[t - 1]
        if ip + nb > len(s):
            return None, "tag_input"
        if t == 1:
            ln, off = 4 + ((tag >> 2) & 7), ((tag >> 5) << 8) | s[ip]
        else:
            ln, off = (tag >> 2) + 1, int.from_bytes(s[ip:ip + nb], "little")
        ip += nb
        if off == 0 or off > len(out):
            return None, "offset"
        if ln > n - len(out):
            return None, "output"
        for _ in range(ln):
            out.append(out[-off])
    if ip != len(s):
        return None, "leftover"
    return bytes(out), None

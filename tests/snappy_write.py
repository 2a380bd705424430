"""Assembles snappy streams from explicit element lists (snappy's format_description.txt), for decoder tests.

Elements: ("lit", data[, nbytes]) -- a literal run, its length in the tag (nbytes 0) or in 1..4 following bytes (the
default is the smallest form); ("c1" | "c2" | "c4", length, offset) -- a copy.  stream(n, elems) puts the varint
preamble n in front; raw(b) is the bytes as given, for hand-made damage.
"""


def varint(v):
    out = bytearray()
    while v >= 128:
        out.append((v & 127) | 128)
        v >>= 7
    out.append(v)
    return bytes(out)


def lit(data, nbytes=None):
    ln = len(data) - 1
    if nbytes is None:
        nbytes = 0 if ln < 60 else (1 if ln < 1 << 8 else (2 if ln < 1 << 16 else (3 if ln < 1 << 24 else 4)))
    if nbytes == 0:
        assert ln < 60
        return bytes([ln << 2]) + bytes(data)
    return bytes([(59 + nbytes) << 2]) + ln.to_bytes(nbytes, "little") + bytes(data)


def copy(kind, length, offset):
    if kind == "c1":
        assert 4 <= length <= 11 and offset < 2048
        return bytes([1 | ((length - 4) << 2) | ((offset >> 8) << 5), offset & 255])
    assert 1 <= length <= 64
    if kind == "c2":
        return bytes([2 | ((length - 1) << 2)]) + offset.to_bytes(2, "little")
    return bytes([3 | ((length - 1) << 2)]) + offset.to_bytes(4, "little")


def elements(elems):
    out = bytearray()
    for e in elems:
        out += lit(*e[1:]) if e[0] == "lit" else copy(*e)
    return bytes(out)


def stream(n, elems):
    return varint(n) + elements(elems)


def expand(elems):
    """the bytes the elements decode to (the reference for a decoder)"""
    out = bytearray()
    for e in elems:
        if e[0] == "lit":
            out += bytes(e[1])
        else:
            for _ in range(e[1]):
                out.append(out[-e[2]])
    return bytes(out)

"""LZ4 blocks and BloscLZ streams written from explicit sequences, with the output they stand for.

No compression search: the caller says which literals, offsets and lengths a stream holds, and how each length is
spelled, so that the forms a real encoder never writes (255-chains of any length, a match at the very end of a block,
offset 0, offsets before the block, lengths whose extension bytes sit exactly at a decoder's bound) are spelled out.
The expected output is computed by applying the sequences in plain Python, byte by byte; it is None when a sequence
reaches before the start of the output (the stream is invalid for every decoder)."""


# ------------------------------------------------------------------------------------------------
# LZ4 block format (lz4 Block_format.md)
# ------------------------------------------------------------------------------------------------
def seq(lits=b"", off=1, ml=4, lit_ext=None, ml_ext=None):
    """one sequence: literals, then a match of `ml` (>= 4) bytes at distance `off`.  lit_ext / ml_ext, when given,
    are the exact extension bytes written after a length nibble of 15 (the decoders add them up)"""
    return dict(lits=bytes(lits), off=off, ml=ml, lit_ext=lit_ext, ml_ext=ml_ext)


def length_bytes(n):
    """the extension bytes of a length field whose nibble is 15: n - 15 as 255s and a remainder"""
    assert n >= 15
    rest = n - 15
    return [255] * (rest // 255) + [rest % 255]


def _nibble(n, ext):
    if ext is not None:
        return 15, list(ext)
    return (15, length_bytes(n)) if n >= 15 else (n, [])


def apply_match(out, off, ml):
    """append a match to `out` (a bytearray) as LZ4_decompress_safe does; False when it reaches before the start"""
    if off == 0:
        out += bytes(ml)               # every copy routine clears its destination first: offset 0 decodes to zeros
        return True
    if off > len(out):
        return False
    for _ in range(ml):
        out.append(out[-off])
    return True


def lz4_block(seqs, last=b"", last_ext=None, end=True):
    """(block, expected output or None).  `seqs` are seq() dicts; `last` is the literals-only final sequence,
    written unless end=False (a block whose last sequence carries a match)."""
    blk = bytearray()
    out = bytearray()
    valid = True
    for s in seqs:
        lits, ml = s["lits"], s["ml"]
        ln, lx = _nibble(len(lits), s["lit_ext"])
        mn, mx = _nibble(ml - 4, s["ml_ext"])
        blk.append(ln << 4 | mn)
        blk += bytes(lx)
        blk += lits
        blk += (s["off"] & 0xFFFF).to_bytes(2, "little")
        blk += bytes(mx)
        out += lits
        if valid:
            valid = apply_match(out, s["off"], ml)
    if end:
        ln, lx = _nibble(len(last), last_ext)
        blk.append(ln << 4)
        blk += bytes(lx)
        blk += bytes(last)
        out += bytes(last)
    return bytes(blk), (bytes(out) if valid else None)


# ------------------------------------------------------------------------------------------------
# BloscLZ (blosclz.c, the decoder's view)
# ------------------------------------------------------------------------------------------------
BLZ_MAX_DISTANCE = 8191


def blz_lit(data):
    """a literal run of 1..32 bytes"""
    assert 1 <= len(data) <= 32
    return dict(kind="lit", data=bytes(data))


def blz_match(dist, ml, ext=None, far=None):
    """a match of ml >= 3 bytes at distance dist: 1..8191 in the 13-bit form, 8192..73727 in the far form
    (ctrl & 31 == 31, code 255, then 16 bits, + 8191).  ml >= 9 uses ctrl >> 5 == 7 and length bytes (`ext` overrides
    them: ml = 9 + sum(ext)).  far=True forces the far form (far=False, the near one)"""
    return dict(kind="match", dist=dist, ml=ml, ext=ext, far=far)


def blz_stream(items, marker=1):
    """(stream, expected output or None).  The first item must be a literal run (the first byte is read as a literal
    ctrl, its top three bits -- the encoder's level marker, `marker` -- ignored).  A match that is the stream's last
    item is dropped by the decoders when its bytes end exactly at the end of the input (the reference's quirk); the
    expected output leaves it out, but the decoders still refuse the stream unless `maxout` has room for it."""
    st = bytearray()
    out = bytearray()
    valid = True
    for k, it in enumerate(items):
        if it["kind"] == "lit":
            ctrl = len(it["data"]) - 1
            st.append(ctrl | (marker << 5 if k == 0 else 0))
            st += it["data"]
            out += it["data"]
            continue
        assert k > 0, "a stream starts with literals"
        dist, ml = it["dist"], it["ml"]
        far = it["far"] if it["far"] is not None else dist > BLZ_MAX_DISTANCE
        if ml >= 9 or it["ext"] is not None:
            lcode, ext = 7, (list(it["ext"]) if it["ext"] is not None else _blz_len_bytes(ml - 9))
        else:
            assert 3 <= ml <= 8
            lcode, ext = ml - 2, []
        if far:
            d = dist - BLZ_MAX_DISTANCE - 1
            assert 0 <= d <= 0xFFFF
            st.append(lcode << 5 | 31)
            st += bytes(ext)
            st += bytes([255, d >> 8, d & 255])
        else:
            assert 1 <= dist <= BLZ_MAX_DISTANCE
            d = dist - 1
            st.append(lcode << 5 | d >> 8)
            st += bytes(ext)
            st.append(d & 255)
        if k == len(items) - 1:
            # ends the input: the reference does not copy it.  Only a match with length bytes or the far form can
            # end there: before the code byte of a short near match the decoders want two more bytes, and refuse
            if lcode != 7 and not far or dist > len(out):
                valid = False
            break
        if dist > len(out):
            valid = False
        if valid:
            for _ in range(ml):
                out.append(out[-dist])
    return bytes(st), (bytes(out) if valid else None)


def _blz_len_bytes(n):
    return [255] * (n // 255) + [n % 255]

"""Encoder inputs built to order: the counterpart of lz_write.py for the LZ4 and BloscLZ encoders.

A scenario places what it needs -- a repeat at a chosen distance and length, a literal run of a chosen length, a
position whose hash equals another's -- into incompressible filler drawn from a seeded generator, so every input is
deterministic.  The hashes are the reference's: LZ4_hash4 (byU16 table), LZ4_hash5 (byU32 table) and BloscLZ's
HASH_FUNCTION with its hashlog.

Two facts of the encoders make positions predictable without a model of the whole parse:
- A zeroed LZ4 table reads position 0 for every hash never stored, so a key written at position 0 is the candidate
  of any later position with the same bytes whose bucket is still empty: that puts a candidate at an exact distance.
- A repeat of the stream's first bytes is caught up to position 0 (catch-up stops there at the latest), so the
  literal run before it is exactly the distance of the repeat, wherever the search first lands in it."""
import numpy as np

from test_lz4_team import hash_u16, hash_u32  # noqa: F401 (the LZ4 hashes, for scenarios that need them)


def blz_hash(b, p, hashlog):
    """blosclz.c HASH_FUNCTION of the four bytes at p"""
    return ((int.from_bytes(bytes(b[p:p + 4]), "little") * 2654435761) & 0xffffffff) >> (32 - hashlog)


def rnd(n, seed):
    return bytearray(np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes())


def probe_offset(it, accel):
    """offset from the search start of LZ4_compress_fast's it-th probe (lz4.c:1043-1053): the first step is 1, the
    k-th after it accel + (k >> 6)"""
    pos = 0
    for k in range(it):
        pos += 1 if k == 0 else accel + ((k - 1) >> 6)
    return pos


class Stream:
    """a byte string grown piece by piece from seeded noise"""

    def __init__(self, seed):
        self.b = bytearray()
        self.seed = seed

    def noise(self, n, ends=None):
        """n incompressible bytes.  ends=d: the first one differs from the byte d back, so a repeat at distance d
        ends here"""
        self.seed += 1
        r = rnd(n, self.seed)
        if ends and n and len(self.b) >= ends and r[0] == self.b[len(self.b) - ends]:
            r[0] ^= 0xFF
        self.b += r
        return self

    def put(self, data):
        self.b += bytes(data)
        return self

    def repeat(self, dist, length):
        """the bytes `dist` back, `length` of them (periodic when length > dist)"""
        for _ in range(length):
            self.b.append(self.b[-dist])
        return self

    def noise_to(self, pos, ends=None):
        assert pos >= len(self.b), (pos, len(self.b))
        return self.noise(pos - len(self.b), ends)

    def array(self):
        return np.frombuffer(bytes(self.b), np.uint8).copy()

    def __len__(self):
        return len(self.b)


def hash_twin(ref, hashf, seed=0):
    """bytes of ref's length, different from ref, whose hash (hashf of a bytes object at 0) equals ref's"""
    rng = np.random.default_rng(seed)
    want = hashf(bytes(ref))
    while True:
        c = bytes(rng.integers(0, 256, len(ref), dtype=np.uint8))
        if c != bytes(ref) and hashf(c) == want:
            return c


# ------------------------------------------------------------------------------------------------
# BloscLZ's entropy probe: windows with a chosen ip / oc
# ------------------------------------------------------------------------------------------------
def blz_cratio(w):
    """the entropy probe's estimate for the window w (at most its first 4096 bytes are read): the bytes it consumed
    over the bytes it would have written, with hashlog 12, ipshift 3, minlen 3 and no far-distance rule.  A model
    of the encoder's accounting, kept to find windows whose ratio equals a threshold exactly."""
    limit = min(len(w), 4096)
    ip_bound, ip_limit = limit - 1, limit - 12
    tab = [0] * 4096
    ip, oc, copy = 0, 5, 4

    def lit():
        nonlocal ip, oc, copy
        oc += 1
        ip += 1
        copy += 1
        if copy == 32:
            oc += 1
            copy = 0
    while ip < ip_limit:
        anchor = ip
        h = blz_hash(w, ip, 12)
        ref = tab[h]
        dist = anchor - ref
        tab[h] = anchor
        if dist == 0 or dist >= 65535 + 8191 - 1 or w[ref:ref + 4] != w[ip:ip + 4]:
            lit()
            continue
        p, q = anchor + 4, ref + 4
        while p < ip_bound and w[p] == w[q]:
            p += 1
            q += 1
        end = p + 1 if p < ip_bound else ip_bound
        ip = end - 3
        ln = ip - anchor
        if ln < 3:
            ip = anchor
            lit()
            continue
        if not copy:
            oc -= 1
        copy = 0
        if ln >= 7:
            oc += (ln - 7) // 255 + 1
        oc += 2 if dist - 1 < 8191 else 4
        tab[blz_hash(w, ip, 12)] = ip
        ip += 2
        oc += 1
    return ip, oc


def probe_window(want, which, seed):
    """a probe window whose ip / oc is `want` exactly (which="equal"), or the nearest ratio just below / above it
    (one byte more / less of oc): a run of z equal bytes, then noise.  ip ends at ip_limit (the tail is all
    literals), so the window's length fixes ip; z is found by bisection, oc falling as z grows.  want: a Fraction."""
    ip = (4084 // want.numerator) * want.numerator
    oc = ip * want.denominator // want.numerator + {"equal": 0, "below": 1, "above": -1}[which]
    base = rnd(ip + 12, seed)

    def window(z):
        w = bytearray(base)
        w[:z] = bytes([0x5A]) * z
        return w
    lo, hi = 0, ip
    while lo < hi:                                   # the smallest z with oc(z) <= target
        mid = (lo + hi) // 2
        if blz_cratio(window(mid))[1] <= oc:
            hi = mid
        else:
            lo = mid + 1
    for z in range(max(lo - 8, 0), lo + 8):
        got = blz_cratio(window(z))
        if got == (ip, oc):
            return bytes(window(z))
    raise AssertionError(("no window", want, which))

"""A plain statement of CRC-32C (bit by bit, no tables) and of zlib's crc32_combine, for the tests of the device kernels
and of tf_bundle's host CRC."""
POLY = 0x82F63B78


def crc32c(data: bytes, crc: int = 0) -> int:
    """CRC-32C of `data` continuing from the CRC `crc` of what came before (0 for none)."""
    c = crc ^ 0xFFFFFFFF
    for b in bytes(data):
        c ^= b
        for _ in range(8):
            c = (c >> 1) ^ POLY if c & 1 else c >> 1
    return c ^ 0xFFFFFFFF


def mask(c: int) -> int:
    return ((((c >> 15) | (c << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


def _mulmodp(a: int, b: int) -> int:
    p = 0
    for i in range(32):
        if a & (0x80000000 >> i):
            p ^= b
        b = (b >> 1) ^ POLY if b & 1 else b >> 1
    return p


def _xpow8(n: int) -> int:
    p, sq = 0x80000000, 0x80000000
    for _ in range(8):
        sq = (sq >> 1) ^ POLY if sq & 1 else sq >> 1
    while n:
        if n & 1:
            p = _mulmodp(sq, p)
        sq = _mulmodp(sq, sq)
        n >>= 1
    return p


def combine(crc_a: int, crc_b: int, len_b: int) -> int:
    """CRC-32C of A || B from crc(A), crc(B) and |B|."""
    return _mulmodp(_xpow8(len_b), crc_a) ^ crc_b


def combine_many(crcs, seg_bytes: int) -> int:
    acc = 0
    for c in crcs:
        acc = combine(acc, int(c), seg_bytes)
    return acc

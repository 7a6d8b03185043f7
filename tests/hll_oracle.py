"""hll_add_agg restated in numpy, for the parity tests: the reference's value hash (ExprValue::hash, include/common/expr_value.h:667-702:
MurmurHash3_x64_128 of the value's native bytes, seed 0x110, first half), hll_row_add (src/common/hll_common.cpp:422-431, register index
and run length from hll_pat_len, :41-56), hll_merge_agg (:630-703) and hll_estimate (:523-600, Redis's histogram estimator).

A sketch here is the 16400-byte RAW layout hll_row_init builds: "HYLL", encoding 255, three zero bytes, eight bytes of cached cardinality
(bit 7 of the last = not cached), then 16384 one-byte registers."""
import math
from typing import Optional

import numpy as np

from baikaldb_b200.plan import PrimitiveType as T

P = 14
REGISTERS = 1 << P
HDR = 16
RAW_BYTES = HDR + REGISTERS
SEED = 0x110
M64 = (1 << 64) - 1
C1, C2 = 0x87C37B91114253D5, 0x4CF5AD432745937F

# bytes ExprValue::hash reads, by the argument's type after inference
KEY_BYTES = {T.BOOL: 1, T.INT8: 1, T.UINT8: 1, T.INT16: 2, T.UINT16: 2, T.INT32: 4, T.UINT32: 4, T.FLOAT: 4, T.TIMESTAMP: 4, T.DATE: 4,
             T.TIME: 4, T.INT64: 8, T.UINT64: 8, T.DOUBLE: 8, T.DATETIME: 8}


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def _fmix(k):
    k ^= k >> 33
    k = (k * 0xFF51AFD7ED558CCD) & M64
    k ^= k >> 33
    k = (k * 0xC4CEB9FE1A85EC53) & M64
    return k ^ (k >> 33)


def murmur3_x64_128(data: bytes, seed: int):
    """MurmurHash3_x64_128 (Austin Appleby's SMHasher, public domain) of any key: (h1, h2)."""
    n = len(data)
    h1 = h2 = seed & 0xFFFFFFFF
    nblocks = n // 16
    for i in range(nblocks):
        k1 = int.from_bytes(data[16 * i:16 * i + 8], "little")
        k2 = int.from_bytes(data[16 * i + 8:16 * i + 16], "little")
        k1 = (_rotl((k1 * C1) & M64, 31) * C2) & M64
        h1 ^= k1
        h1 = (_rotl(h1, 27) + h2) & M64
        h1 = (h1 * 5 + 0x52DCE729) & M64
        k2 = (_rotl((k2 * C2) & M64, 33) * C1) & M64
        h2 ^= k2
        h2 = (_rotl(h2, 31) + h1) & M64
        h2 = (h2 * 5 + 0x38495AB5) & M64
    tail = data[16 * nblocks:]
    if len(tail) > 8:
        k2 = int.from_bytes(tail[8:], "little")
        h2 ^= (_rotl((k2 * C2) & M64, 33) * C1) & M64
    if tail:
        k1 = int.from_bytes(tail[:8], "little")
        h1 ^= (_rotl((k1 * C1) & M64, 31) * C2) & M64
    h1 ^= n
    h2 ^= n
    h1 = (h1 + h2) & M64
    h2 = (h2 + h1) & M64
    h1, h2 = _fmix(h1), _fmix(h2)
    h1 = (h1 + h2) & M64
    h2 = (h2 + h1) & M64
    return h1, h2


def smhasher_verification() -> int:
    """SMHasher's VerificationTest: hash keys {0}, {0,1}, ..., {0..254} with seed 256 - len, then the concatenated hashes with seed 0;
    the first four bytes of that (MurmurHash3_x64_128's published value is 0x6384BA69)."""
    out = b""
    for i in range(256):
        h1, h2 = murmur3_x64_128(bytes(range(i)), 256 - i)
        out += h1.to_bytes(8, "little") + h2.to_bytes(8, "little")
    h1, _ = murmur3_x64_128(out, 0)
    return h1 & 0xFFFFFFFF


def hash_images(img: np.ndarray, nbytes: int, seed: int = SEED) -> np.ndarray:
    """MurmurHash3_x64_128(...)[0] of the low `nbytes` bytes of each uint64 image, vectorised (keys of at most 8 bytes: the tail alone)."""
    with np.errstate(over="ignore"):
        k1 = np.asarray(img, dtype=np.uint64)
        if nbytes < 8:
            k1 = k1 & np.uint64((1 << (8 * nbytes)) - 1)
        k1 = k1 * np.uint64(C1)
        k1 = (k1 << np.uint64(31)) | (k1 >> np.uint64(33))
        k1 = k1 * np.uint64(C2)
        h1 = np.full(k1.shape, seed, dtype=np.uint64) ^ k1 ^ np.uint64(nbytes)
        h2 = np.full(k1.shape, seed ^ nbytes, dtype=np.uint64)
        h1 = h1 + h2
        h2 = h2 + h1

        def fmix(k):
            k = k ^ (k >> np.uint64(33))
            k = k * np.uint64(0xFF51AFD7ED558CCD)
            k = k ^ (k >> np.uint64(33))
            k = k * np.uint64(0xC4CEB9FE1A85EC53)
            return k ^ (k >> np.uint64(33))
        return fmix(h1) + fmix(h2)


def pat_len(h: np.ndarray):
    """hll_pat_len: (register index, 1 + trailing zeros of the bits above it with a guard bit at 50)."""
    h = np.asarray(h, dtype=np.uint64)
    idx = (h & np.uint64(REGISTERS - 1)).astype(np.int64)
    x = (h >> np.uint64(P)) | np.uint64(1 << (64 - P))
    low = x & (~x + np.uint64(1))                     # the lowest set bit, a power of two <= 2^50 (exact as a double)
    count = np.log2(low.astype(np.float64)).astype(np.int64) + 1
    return idx, count


def key_images(values: np.ndarray, prim: int) -> np.ndarray:
    """The bytes ExprValue::hash reads, as the low bytes of a uint64: a column's storage values of type `prim`."""
    v = np.asarray(values)
    if v.dtype == np.float32:
        return v.view(np.uint32).astype(np.uint64)
    if v.dtype == np.float64:
        return v.view(np.uint64)
    if v.dtype.itemsize == 8:
        return v.view(np.uint64)
    return v.astype(np.int64).view(np.uint64)       # (sign-extended: only the low KEY_BYTES bytes are hashed)


def registers(values: np.ndarray, prim: int, groups: Optional[np.ndarray] = None, n_groups: int = 1, valid: Optional[np.ndarray] = None) -> np.ndarray:
    """The registers of every group's sketch after hll_row_add of each non-NULL value: uint8[n_groups, 16384]."""
    regs = np.zeros((n_groups, REGISTERS), dtype=np.uint8)
    img = key_images(values, prim)
    g = np.zeros(len(img), dtype=np.int64) if groups is None else np.asarray(groups, dtype=np.int64)
    if valid is not None:
        img, g = img[valid], g[valid]
    idx, count = pat_len(hash_images(img, KEY_BYTES[T(prim)]))
    np.maximum.at(regs, (g, idx), count.astype(np.uint8))
    return regs


def raw_sketch(regs: np.ndarray, invalidated: bool) -> bytes:
    """hll_row_init's header over `regs`; `invalidated`: some register grew (hll_row_add / hll_merge_agg set bit 7 of byte 15)."""
    hdr = bytearray(b"HYLL" + bytes([255, 0, 0, 0]) + bytes(8))
    if invalidated:
        hdr[15] |= 0x80
    return bytes(hdr) + np.asarray(regs, dtype=np.uint8).tobytes()


def sketches(values, prim, groups=None, n_groups=1, valid=None):
    """hll_add_agg per group: the RAW sketch each group returns (a group whose every argument is NULL: the empty sketch, cache byte 0)."""
    regs = registers(values, prim, groups, n_groups, valid)
    g = np.zeros(len(values), dtype=np.int64) if groups is None else np.asarray(groups, dtype=np.int64)
    has = np.zeros(n_groups, dtype=bool)
    has[g if valid is None else g[valid]] = True
    return [raw_sketch(regs[i], bool(has[i])) for i in range(n_groups)]


def merge(dst: bytes, src: bytes) -> bytes:
    """hll_merge_agg of a RAW source into a RAW destination: register-wise max, and the cache is invalidated whether or not a register grew."""
    r = np.maximum(np.frombuffer(dst, np.uint8, offset=HDR), np.frombuffer(src, np.uint8, offset=HDR))
    return raw_sketch(r, True)


def _sigma(x):
    if x == 1.0:
        return math.inf
    zp, y, z = 0.0, 1.0, x
    while True:
        x *= x
        zp = z
        z += x * y
        y += y
        if zp == z:
            return z


def _tau(x):
    if x == 0.0 or x == 1.0:
        return 0.0
    zp, y, z = 0.0, 1.0, 1 - x
    while True:
        x = math.sqrt(x)
        zp = z
        y *= 0.5
        z -= pow(1 - x, 2) * y
        if zp == z:
            return z / 3


def estimate(sketch: bytes) -> int:
    """hll_estimate over a RAW sketch: the cached value when bit 7 of byte 15 is clear, else the histogram estimator."""
    if not sketch[15] & 0x80:
        return int.from_bytes(sketch[8:16], "little")
    m = float(REGISTERS)
    histo = np.bincount(np.frombuffer(sketch, np.uint8, offset=HDR), minlength=64)
    q = 64 - P
    z = m * _tau((m - histo[q + 1]) / m)
    for j in range(q, 0, -1):
        z += histo[j]
        z *= 0.5
    z += m * _sigma(histo[0] / m)
    if abs(z) < 1e-9:
        return 0
    e = 0.721347520444481703680 * m * m / z
    return int(math.floor(e + 0.5)) if e >= 0 else -int(math.floor(-e + 0.5))   # llroundl: halves away from zero

"""Synthetic tables of SURVEY.md §8(d) / BASELINE.md — host (numpy) statement of the generator.

Counter-based: every value is a pure function of (seed, column_id, absolute row index), so any
region (row range) of any table can be produced independently and the CUDA generator
(``bkgpu_gen_column`` in csrc/gen.cu) produces the same bits.  Only integer arithmetic and exactly
rounded double operations are used, which is what makes host and device agree bit for bit.

    key_k   = mix64(seed + column_id * C1 + k * C2)
    r_k(i)  = mix64(key_k + (i + 1) * GOLDEN)                     (splitmix64 stream)
    dist 0  uniform integer in [lo, hi):   lo + r_0 % (hi - lo)
    dist 1  uniform double in [0, 1):      (r_0 >> 11) * 2^-53
    dist 2  approx. normal (Irwin-Hall 4): (u_0 + u_1 + u_2 + u_3 - 2.0) * scale
    dist 3  full-range int64:              r_0 reinterpreted
    dist 4  permutation of [0, hi):        4-round Feistel over ceil(log2 hi) bits + cycle walking
"""
from __future__ import annotations

from typing import List

import numpy as np

from .column import Column, make_column
from .plan import PrimitiveType as T

GOLDEN = np.uint64(0x9E3779B97F4A7C15)
C1 = np.uint64(0xD1B54A32D192ED03)
C2 = np.uint64(0x8CB92BA72F3D8DD7)
M1 = np.uint64(0xBF58476D1CE4E5B9)
M2 = np.uint64(0x94D049BB133111EB)

DIST_UNIFORM_INT, DIST_UNIFORM_01, DIST_NORMAL_IH4, DIST_INT64_FULL, DIST_PERMUTATION = 0, 1, 2, 3, 4
NORMAL_SCALE_1E3 = 1000.0 * 1.7320508075688772  # sd of Irwin-Hall(4) is 1/sqrt(3)


def mix64(z: np.ndarray) -> np.ndarray:
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * M1
        z = (z ^ (z >> np.uint64(27))) * M2
        return z ^ (z >> np.uint64(31))


def _key(seed: int, column_id: int, k: int) -> np.uint64:
    with np.errstate(over="ignore"):
        s = np.uint64(seed) + np.uint64(column_id) * C1 + np.uint64(k) * C2
    return mix64(np.array([s], dtype=np.uint64))[0]


def raw64(seed: int, column_id: int, row0: int, n: int, k: int = 0) -> np.ndarray:
    idx = np.arange(row0 + 1, row0 + 1 + n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        return mix64(_key(seed, column_id, k) + idx * GOLDEN)


def _u01(r: np.ndarray) -> np.ndarray:
    return (r >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def gen_values(prim_type: int, dist: int, seed: int, column_id: int, row0: int, n: int,
               lo: int = 0, hi: int = 0, scale: float = 1.0) -> np.ndarray:
    if dist == DIST_UNIFORM_INT:
        r = raw64(seed, column_id, row0, n)
        span = np.uint64(hi - lo)
        v = (r % span).astype(np.int64) + np.int64(lo)
        return v.astype(np.int32) if prim_type == T.INT32 else v
    if dist == DIST_UNIFORM_01:
        return _u01(raw64(seed, column_id, row0, n))
    if dist == DIST_NORMAL_IH4:
        s = _u01(raw64(seed, column_id, row0, n, 0))
        for k in (1, 2, 3):
            s = s + _u01(raw64(seed, column_id, row0, n, k))
        return (s - 2.0) * scale
    if dist == DIST_INT64_FULL:
        return raw64(seed, column_id, row0, n).view(np.int64)
    if dist == DIST_PERMUTATION:
        return permutation(seed, column_id, row0, n, hi).astype(np.int32 if prim_type == T.INT32 else np.int64)
    raise ValueError(dist)


def permutation(seed: int, column_id: int, row0: int, n: int, domain: int) -> np.ndarray:
    """Bijection of [0, domain) evaluated at row0..row0+n-1."""
    bits = max(2, int(domain - 1).bit_length())
    bits += bits & 1
    half = np.uint64(bits // 2)
    mask = np.uint64((1 << (bits // 2)) - 1)
    keys = [_key(seed, column_id, 16 + r) for r in range(4)]
    x = np.arange(row0, row0 + n, dtype=np.uint64)
    todo = np.ones(n, dtype=bool)
    while todo.any():
        xs = x[todo]
        left, right = xs >> half, xs & mask
        for rk in keys:
            with np.errstate(over="ignore"):
                f = mix64(right + rk) & mask
            left, right = right, left ^ f
        xs = (left << half) | right
        x[todo] = xs
        todo = x >= np.uint64(domain)
    return x.astype(np.int64)


# ---------------------------------------------------------------------------------------------
# Tables of the BASELINE.json configs (SURVEY.md §8d).  `row0`/`n` select a region (row range).
# ---------------------------------------------------------------------------------------------
C2_COLUMNS = [  # (slot, prim_type, dist, lo, hi, scale)
    (1, T.INT32, DIST_UNIFORM_INT, 0, 1000, 1.0),           # 0_1 group key
    (2, T.INT32, DIST_UNIFORM_INT, 0, 1 << 20, 1.0),        # 0_2 filter column
    (3, T.DOUBLE, DIST_UNIFORM_01, 0, 0, 1.0),              # 0_3
    (4, T.DOUBLE, DIST_NORMAL_IH4, 0, 0, NORMAL_SCALE_1E3), # 0_4
]


def c1_table(row0: int, n: int, seed: int = 1) -> List[Column]:
    return [make_column(0, 1, T.INT32, gen_values(T.INT32, DIST_UNIFORM_INT, seed, 1, row0, n, 0, 1 << 20))]


def c2_table(row0: int, n: int, seed: int = 2, n_groups: int = 1000) -> List[Column]:
    cols = []
    for slot, pt, dist, lo, hi, scale in C2_COLUMNS:
        if slot == 1:
            hi = n_groups
        cols.append(make_column(0, slot, pt, gen_values(pt, dist, seed, slot, row0, n, lo, hi, scale)))
    return cols


def c3_fact(row0: int, n: int, n_dim: int, seed: int = 3) -> List[Column]:
    return [make_column(0, 1, T.INT32, gen_values(T.INT32, DIST_UNIFORM_INT, seed, 1, row0, n, 0, n_dim)),
            make_column(0, 2, T.DOUBLE, gen_values(T.DOUBLE, DIST_UNIFORM_01, seed, 2, row0, n))]


def c3_dim(row0: int, n: int, n_dim: int, seed: int = 3, n_groups: int = 1000) -> List[Column]:
    return [make_column(1, 1, T.INT32, gen_values(T.INT32, DIST_PERMUTATION, seed, 11, row0, n, 0, n_dim)),
            make_column(1, 2, T.INT32, gen_values(T.INT32, DIST_UNIFORM_INT, seed, 12, row0, n, 0, n_groups))]


PART_KEY_STRIDE, PART_KEY_BASE = 7, 3   # part keys are sparse (stride 7): the join index is the packed table, not the dense array


def c6_tables(n_fact: int, n_date: int = 2_556, n_part: int = 1_000_000, n_supp: int = 100_000, seed: int = 6):
    """The star tables of config C6 (queries.STAR_TUPLES): date and supplier keys are a permutation of [0, n) (dense index), part keys
    PART_KEY_BASE + PART_KEY_STRIDE * a permutation of [0, n) (sparse); the fact's foreign keys are drawn uniformly from those key sets.
    Returns (fact, date, part, supplier) column lists."""
    g = lambda pt, dist, cid, n, lo=0, hi=0: gen_values(pt, dist, seed, cid, 0, n, lo, hi)
    dkey = g(T.INT32, DIST_PERMUTATION, 11, n_date, 0, n_date)
    date = [make_column(1, 1, T.INT32, dkey), make_column(1, 2, T.INT32, (1992 + dkey // 365).astype(np.int32))]
    pkey = (PART_KEY_BASE + PART_KEY_STRIDE * g(T.INT64, DIST_PERMUTATION, 21, n_part, 0, n_part)).astype(np.int32)
    part = [make_column(2, 1, T.INT32, pkey), make_column(2, 2, T.INT32, g(T.INT32, DIST_UNIFORM_INT, 22, n_part, 0, 1000)),
            make_column(2, 3, T.INT32, g(T.INT32, DIST_UNIFORM_INT, 23, n_part, 0, 25))]
    supp = [make_column(3, 1, T.INT32, g(T.INT32, DIST_PERMUTATION, 31, n_supp, 0, n_supp)),
            make_column(3, 2, T.INT32, g(T.INT32, DIST_UNIFORM_INT, 32, n_supp, 0, 5))]
    fact = [make_column(0, 1, T.INT32, g(T.INT32, DIST_UNIFORM_INT, 1, n_fact, 0, n_date)),
            make_column(0, 2, T.INT32, (PART_KEY_BASE + PART_KEY_STRIDE * g(T.INT64, DIST_UNIFORM_INT, 2, n_fact, 0, n_part)).astype(np.int32)),
            make_column(0, 3, T.INT32, g(T.INT32, DIST_UNIFORM_INT, 3, n_fact, 0, n_supp)),
            make_column(0, 4, T.DOUBLE, g(T.DOUBLE, DIST_UNIFORM_01, 4, n_fact))]
    return fact, date, part, supp


def c5_table(row0: int, n: int, seed: int = 5) -> List[Column]:
    return [make_column(0, 1, T.INT64, gen_values(T.INT64, DIST_INT64_FULL, seed, 1, row0, n)),
            make_column(0, 2, T.INT32, gen_values(T.INT32, DIST_UNIFORM_INT, seed, 2, row0, n, 0, 1 << 30))]

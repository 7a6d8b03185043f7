"""Region layouts and the top-k cases of tests/test_gpu_region_merge.py (several regions' partial states exported and merged on one GPU),
with the plain reference of ORDER BY ... LIMIT k OFFSET o over the whole table that tests/test_region_merge_reference.py checks against
the row-engine oracle on the CPU.

Top-k tables: tuple 0 = the key (slot 1, any type, NULLs) and the row's global number (slot 2, INT32).  Keys are drawn from a small pool
(the type's edges without NaN, +-0.0 several times over, a few small values), so that equal keys span every region and only the arrival
order breaks their ties: MemRowCompare orders equal keys, -0.0 and +0.0 included, by arrival, under DESC as well."""
import math
from typing import List, Optional, Sequence, Tuple

import numpy as np

from baikaldb_b200 import plan as P
from baikaldb_b200.column import Column, make_column
from baikaldb_b200.plan import PrimitiveType as T
from tests.agg_type_cases import FLOATS, TYPES, column_array, edges, small_values

REGION_COUNTS = (2, 3, 5)


# ---------------------------------------------------------------- region layouts
def ragged_cut(m: int) -> int:
    """a cut near m / 2 whose left part holds 3 rows modulo 4 (the aggregate kernels' ragged tail)"""
    a = m // 2
    return max(0, a - (a - 3) % 4) if m >= 3 else m


def contiguous(n: int, regions: int) -> List[Tuple[int, int]]:
    """[start, stop) of each region over n rows in arrival order: 2 regions cut raggedly; 3 regions; 5 regions with an empty one and
    one of a single row between the others"""
    a = ragged_cut(n)
    if regions == 2:
        return [(0, a), (a, n)]
    b = a + ragged_cut(n - a)
    if regions == 3:
        return [(0, a), (a, b), (b, n)]
    assert regions == 5
    return [(0, a), (a, a), (a, a + 1), (a + 1, b), (b, n)]


def role_layout(n: int, regions: int, null_rows: np.ndarray, lonely: np.ndarray) -> List[np.ndarray]:
    """row indices of each region, by role: `null_rows` (NULL keys, or NULL values where the keys are never NULL) all in one region of
    their own, the rows of a `lonely` group all in the last region, one region of a single row, an empty one (5 regions), and the
    rest cut raggedly.  2 regions: [NULL rows + half the rest, the other half + the lonely group + one row]"""
    nulls = np.flatnonzero(null_rows & ~lonely)
    rest = np.flatnonzero(~null_rows & ~lonely)
    one, rest = rest[:1], rest[1:]
    a = ragged_cut(len(rest))
    bulk_a, bulk_b, lone = rest[:a], rest[a:], np.flatnonzero(lonely)
    if regions == 2:
        parts = [np.concatenate([nulls, bulk_a]), np.concatenate([one, bulk_b, lone])]
    elif regions == 3:
        parts = [nulls, np.concatenate([one, bulk_a]), np.concatenate([bulk_b, lone])]
    else:
        parts = [bulk_a, np.zeros(0, np.int64), one, nulls, np.concatenate([bulk_b, lone])]
    parts = [np.sort(p) for p in parts]
    assert sum(len(p) for p in parts) == n and len(np.unique(np.concatenate(parts))) == n
    return parts


def take(cols: Sequence[Column], ix) -> List[Column]:
    """the rows `ix` (an index array, or a (start, stop) pair) of every column"""
    if isinstance(ix, tuple):
        ix = slice(*ix)
    return [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[ix], None if c.valid is None else c.valid[ix]) for c in cols]


# ---------------------------------------------------------------- top-k
TOPK_N = 40_007
# (k, offset): k in {1, 1000, 4096 - offset}.  "dense": a tenth of the keys NULL; "sparse": 95 % NULL, so that LIMIT + OFFSET crosses
# from the present keys into the NULL class (or out of it) in the middle of the returned rows
TOPK_KO = {"dense": ((1, 0), (1000, 333), (2596, 1500), (4096, 0)), "sparse": ((1, 1000), (3996, 100))}
TOPK_NULLS = {"dense": 0.1, "sparse": 0.95}


def topk_key_pool(rng, kt: int) -> list:
    pool = [x for x in edges(kt) if not (isinstance(x, (float, np.floating)) and math.isnan(x))] + small_values(rng, kt, 12)
    if kt in FLOATS:
        pool += [0.0, -0.0] * 4
    return pool


def topk_table(kt: int, kind: str, n: int = TOPK_N, seed: int = 0) -> Tuple[List[Column], np.ndarray, np.ndarray]:
    """(columns, key array, key validity)"""
    rng = np.random.default_rng(10_000 + 16 * int(kt) + (kind == "sparse") + 2 * seed)
    pool = topk_key_pool(rng, kt)
    keys = column_array(kt, [pool[i] for i in rng.integers(0, len(pool), n)])
    valid = rng.random(n) >= TOPK_NULLS[kind]
    return [make_column(0, 1, kt, keys, valid), make_column(0, 2, T.INT32, np.arange(n, dtype=np.int32))], keys, valid


def topk_plan(kt: int, asc: bool, null_first: bool, k: int, offset: int) -> P.Plan:
    """SELECT key, row ORDER BY key [DESC] NULLS FIRST|LAST LIMIT k OFFSET offset"""
    s = P.sort(P.scan(0), [P.slot_ref(0, 1, kt)], [asc], [null_first], tuple_id=0)
    return P.Plan(P.limit(s, k, offset), {0: [(1, kt), (2, T.INT32)]})


def topk_reference(keys: np.ndarray, valid: Optional[np.ndarray], asc: bool, null_first: bool, k: int, offset: int) -> np.ndarray:
    """the global row numbers of rows [offset, offset + k) of a stable sort of the whole table: present keys by value (-0.0 equals
    +0.0), DESC by the reversed value, equal keys and the NULL class by arrival"""
    n = len(keys)
    present = np.arange(n) if valid is None else np.flatnonzero(valid)
    nulls = np.zeros(0, np.int64) if valid is None else np.flatnonzero(~valid)
    x = keys[present]
    if x.dtype.kind == "f":
        s = x.astype(np.float64) if asc else -x.astype(np.float64)
    else:
        s = x if asc else ~x   # (~ reverses the order of a signed and of an unsigned integer alike, without overflow)
    ordered = present[np.argsort(s, kind="stable")]
    rows = np.concatenate([nulls, ordered] if null_first else [ordered, nulls])
    return rows[offset:offset + k]


def topk_cases():
    """(key type, table kind, asc, null_first, k, offset) of every top-k merge"""
    return [(kt, kind, asc, nf, k, o) for kt in TYPES for kind in TOPK_KO for asc in (True, False) for nf in (True, False)
            for k, o in TOPK_KO[kind]]


# a region of more than half the selection's candidate buffer (sort.cu: 2^22 pairs): its selection samples before it collects
BIG = 2_200_003


def big_table() -> Tuple[List[Column], np.ndarray, np.ndarray]:
    """BIG + 20,003 INT64 keys from 5000 values (every key repeats across both regions), 1 % NULL"""
    rng = np.random.default_rng(10_999)
    n = BIG + 20_003
    keys = rng.integers(0, 5000, n).astype(np.int64)
    valid = rng.random(n) >= 0.01
    return [make_column(0, 1, T.INT64, keys, valid), make_column(0, 2, T.INT32, np.arange(n, dtype=np.int32))], keys, valid


BIG_CASES = ((True, True, 1000, 0), (False, False, 1000, 7), (True, False, 96, 4000))   # (asc, null_first, k, offset)

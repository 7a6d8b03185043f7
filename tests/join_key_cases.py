"""Join-key cases shared by tests/test_gpu_join_keys.py (GPU against the oracle) and tests/test_join_key_lowering.py (host only).

Every result of these tables is exact, so a wrong key image, a lost sign bias or a misread load cannot hide inside a tolerance:
- the summed fact value is an integer-valued double, so every SUM over it is exact in any order;
- each dimension row carries an INT64 attribute that is a fixed function of its key (`attr64`), aggregated with SUM, MIN and MAX:
  a lookup that lands on the wrong dimension row changes the result;
- SUM of a fact row id (INT64) changes when a fact row is lost or joined twice.

Layout: fact tuple 0 = row id (slot 1, INT64), value (2, DOUBLE), group (3, INT32), foreign key of dimension d (10 + d);
dimension tuple d = key (slot 1), attr64(key) (2, INT64), key % 7 (3, INT32)."""
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from baikaldb_b200 import plan as P
from baikaldb_b200.column import Column, make_column
from baikaldb_b200.plan import PrimitiveType as T, storage_dtype

AT = 7   # the aggregate tuple (the oracle takes tuple ids below 8)
SIGNED = (T.INT8, T.INT16, T.INT32, T.INT64)
UNSIGNED = (T.UINT8, T.UINT16, T.UINT32, T.UINT64)
SAME = SIGNED + UNSIGNED + (T.DATE, T.DATETIME)
# (dimension key type, foreign key type): every type against itself, and mixed pairs that meet in INT64 or in UINT64
MIXED = ((T.INT8, T.INT32), (T.INT16, T.INT64), (T.INT32, T.INT64), (T.INT64, T.INT32), (T.UINT8, T.UINT32), (T.UINT32, T.UINT64), (T.UINT64, T.UINT16))
PAIRS = tuple((t, t) for t in SAME) + MIXED
# pairs the lowering refuses (the reference compares them as strings): signed with unsigned, DATE with DATETIME, BOOL with an integer,
# FLOAT / DOUBLE keys, STRING keys.  BOOL = BOOL is among them: the reference's comparison typing (fn_manager.cpp:316-409) takes two
# BOOL operands as neither integer nor date / time nor double, so the equality itself is a STRING comparison and no join over it lowers.
REFUSED = ((T.INT32, T.UINT32), (T.UINT64, T.INT64), (T.INT8, T.UINT8), (T.DATE, T.DATETIME), (T.DATETIME, T.DATE), (T.DATE, T.UINT32),
           (T.BOOL, T.BOOL), (T.BOOL, T.INT32), (T.DOUBLE, T.DOUBLE), (T.FLOAT, T.FLOAT), (T.FLOAT, T.DOUBLE), (T.INT64, T.DOUBLE), (T.STRING, T.STRING))

RANGE = {T.BOOL: (0, 1), T.INT8: (-2**7, 2**7 - 1), T.INT16: (-2**15, 2**15 - 1), T.INT32: (-2**31, 2**31 - 1), T.INT64: (-2**63, 2**63 - 1),
         T.UINT8: (0, 2**8 - 1), T.UINT16: (0, 2**16 - 1), T.UINT32: (0, 2**32 - 1), T.UINT64: (0, 2**64 - 1)}


def pair_id(pair) -> str:
    return f"{T(pair[0]).name}-{T(pair[1]).name}"


def cast_of(dk: int, fk: int) -> int:
    """the type both keys are compared in (lower_join_agg / lower_star_agg)"""
    if dk == fk:
        return dk
    return T.INT64 if dk in SIGNED and fk in SIGNED else T.UINT64


def key_bytes(t: int) -> int:
    return np.dtype(storage_dtype(t)).itemsize


def date_img(y, m, d):
    return ((y * 13 + m) << 5) | d


def datetime_img(y, m, d, h=0, mi=0, s=0, us=0):
    return ((y * 13 + m) << 46) | (d << 41) | (h << 36) | (mi << 30) | (s << 24) | us


def in_range(t: int, x: int) -> bool:
    if t in RANGE:
        lo, hi = RANGE[t]
        return lo <= x <= hi
    return 0 <= x < 2**(8 * key_bytes(t))


def edges(t: int) -> List[int]:
    """each type's minimum and maximum, -1 / 0 / 1, and values at and around 2^31, 2^32 and 2^63 where the type holds them"""
    if t == T.DATE:
        return [date_img(1, 1, 1), date_img(9999, 12, 31), date_img(1970, 1, 1), date_img(2000, 2, 29)]
    if t == T.DATETIME:
        return [datetime_img(1, 1, 1), datetime_img(9999, 12, 31, 23, 59, 59, 999_999), datetime_img(1970, 1, 1), datetime_img(2024, 2, 29, 12, 0, 0, 1)]
    lo, hi = RANGE[t]
    e = [lo, hi, lo + 1, hi - 1, -1, 0, 1, 2**31 - 1, 2**31, 2**31 + 1, -2**31 - 1, 2**32, 2**63 - 1, 2**63, 2**63 + 1]
    return list(dict.fromkeys(x for x in e if lo <= x <= hi))


def draw(rng, t: int, n: int, lo: Optional[int] = None, hi: Optional[int] = None) -> List[int]:
    """`n` values of type `t` (within [lo, hi] when given): half spread over the whole range, half small"""
    if t == T.DATE:
        return [date_img(int(y), int(m), int(d)) for y, m, d in zip(rng.integers(1, 10000, n), rng.integers(1, 13, n), rng.integers(1, 29, n))]
    if t == T.DATETIME:
        return [datetime_img(int(y), int(m), int(d), int(h), int(mi), int(s), int(us)) for y, m, d, h, mi, s, us in
                zip(rng.integers(1, 10000, n), rng.integers(1, 13, n), rng.integers(1, 29, n), rng.integers(0, 24, n), rng.integers(0, 60, n),
                    rng.integers(0, 60, n), rng.integers(0, 1_000_000, n))]
    tlo, thi = RANGE[t]
    lo, hi = max(tlo, tlo if lo is None else lo), min(thi, thi if hi is None else hi)
    wide = [lo + int(o) for o in rng.integers(0, hi - lo, n - n // 2, endpoint=True, dtype=np.uint64)]
    small = [int(x) for x in rng.integers(-1000, 1000, n // 2) if lo <= x <= hi]
    return wide + small


def unique_keys(rng, dk: int, fk: int, nd: int) -> List[int]:
    """`nd` distinct keys of type `dk` (fewer when the type has fewer values): the edges of both types, then values of the whole range and
    values inside the foreign key's range, in random order"""
    cand = edges(dk) + [x for x in edges(fk) if in_range(dk, x)]
    lo, hi = RANGE.get(fk, (None, None))
    cand += [x for pair in zip(draw(rng, dk, 2 * nd), draw(rng, dk, 2 * nd, lo, hi)) for x in pair]
    if dk in RANGE and 2 < RANGE[dk][1] - RANGE[dk][0] + 1 < 4 * nd:   # a small type: three quarters of its values, so that some have no row
        cand += list(range(RANGE[dk][0], RANGE[dk][1] + 1))
        nd = min(nd, (RANGE[dk][1] - RANGE[dk][0] + 1) * 3 // 4)
    out = list(dict.fromkeys(cand))[:nd]
    rng.shuffle(out)
    return out


def misses_for(rng, keys: List[int], fk: int) -> List[int]:
    """foreign-key values without a partner: the foreign key type's edges, values that equal a key in their low 8, 16 or 32 bits or
    differ from one in the sign bit only, and random values"""
    have = set(keys)
    cand = list(edges(fk))
    for k in keys[:64]:
        cand += [k + 2**8, k - 2**8, k + 2**16, k - 2**16, k + 2**32, k - 2**32, k ^ 2**63, k - 2**64, k + 2**64]
    cand += draw(rng, fk, 256)
    return [x for x in dict.fromkeys(cand) if in_range(fk, x) and x not in have]


def attr64(k: int) -> int:
    return (k * 40503) % 1_000_003 - 500_001


def arr(prim: int, values) -> np.ndarray:
    return np.array([int(v) for v in values], dtype=np.dtype(storage_dtype(prim)))


@dataclass
class Dim:
    tid: int
    key_type: int
    fk_type: int
    keys: List[int]                            # the key of each row (the value under a NULL is a real key of another row)
    valid: Optional[np.ndarray] = None         # key validity, None = no NULLs

    def columns(self) -> List[Column]:
        return [make_column(self.tid, 1, self.key_type, arr(self.key_type, self.keys), self.valid),
                make_column(self.tid, 2, T.INT64, arr(T.INT64, [attr64(k) for k in self.keys])),
                make_column(self.tid, 3, T.INT32, arr(T.INT32, [k % 7 for k in self.keys]))]

    def live_keys(self) -> List[int]:
        return [k for i, k in enumerate(self.keys) if self.valid is None or self.valid[i]]


def make_dim(rng, tid, dk, fk, nd, null_keys=0.0, keys=None) -> Dim:
    keys = list(keys) if keys is not None else unique_keys(rng, dk, fk, nd)
    valid = None
    if null_keys and len(keys) > 2:
        valid = rng.random(len(keys)) >= null_keys
        valid[:2] = True
        for i in np.flatnonzero(~valid):   # a NULL key's value repeats a live key: a probe that ignores the validity finds a duplicate
            keys[i] = keys[0]
    return Dim(tid, dk, fk, keys, valid)


def foreign_keys(rng, dim: Dim, n: int, miss=0.1, null=0.05, weights=None) -> Tuple[List[int], Optional[np.ndarray]]:
    """`n` foreign keys into `dim`: partners (drawn by `weights` over the distinct live keys), a share without a partner, and a share of
    NULLs whose value is a partner"""
    partners = [k for k in dict.fromkeys(dim.live_keys()) if in_range(dim.fk_type, k)]
    assert partners, "no key of the dimension fits the foreign key type"
    p = None if weights is None else np.asarray(weights, dtype=float) / np.sum(weights)
    vals = [partners[i] for i in rng.choice(len(partners), n, p=p)]
    misses = misses_for(rng, dim.keys, dim.fk_type) if miss else []
    if misses:
        for i in np.flatnonzero(rng.random(n) < miss):
            vals[i] = misses[int(rng.integers(0, len(misses)))]
    valid = rng.random(n) >= null if null else None
    return vals, valid


@dataclass
class Case:
    """one fact table joined to one dimension (the two-table join) or to two to four (a star join)"""
    dims: List[Dim]
    fk: Dict[int, Tuple[List[int], Optional[np.ndarray]]]
    n: int
    rowid0: int = 0
    value: np.ndarray = field(default=None)
    group: np.ndarray = field(default=None)

    def fact_columns(self) -> List[Column]:
        cols = [make_column(0, 1, T.INT64, np.arange(self.n, dtype=np.int64) * 3 + self.rowid0), make_column(0, 2, T.DOUBLE, self.value),
                make_column(0, 3, T.INT32, self.group)]
        for d in self.dims:
            vals, valid = self.fk[d.tid]
            cols.append(make_column(0, 10 + d.tid, d.fk_type, arr(d.fk_type, vals), valid))
        return cols

    def dim_columns(self) -> List[List[Column]]:
        return [d.columns() for d in self.dims]

    def all_columns(self) -> List[Column]:
        return self.fact_columns() + [c for d in self.dim_columns() for c in d]

    def batches(self) -> List[List[Column]]:
        return self.dim_columns() + [self.fact_columns()]


def make_case(rng, dims: List[Dim], n: int, miss=0.1, null=0.05, weights=None) -> Case:
    fk = {d.tid: foreign_keys(rng, d, n, miss, null, None if weights is None else weights.get(d.tid)) for d in dims}
    return Case(dims, fk, n, int(rng.integers(0, 1 << 20)), rng.integers(-512, 512, n).astype(np.float64), rng.integers(0, 5, n).astype(np.int32))


# ---- plans ----
def on(d: Dim):
    return P.eq(P.slot_ref(d.tid, 1, d.key_type), P.slot_ref(0, 10 + d.tid, d.fk_type))


def aggregates(dims: List[Dim]):
    """COUNT(*), SUM(row id), SUM(value), and SUM / MIN / MAX of each dimension's attribute (SUM and one of MIN / MAX with four
    dimensions: an aggregate node holds at most 12 functions)"""
    aggs = [P.agg_expr("count_star", AT, 1), P.agg_expr("sum", AT, 2, None, P.slot_ref(0, 1, T.INT64)), P.agg_expr("sum", AT, 3, None, P.slot_ref(0, 2, T.DOUBLE))]
    types = [T.INT64, T.INT64, T.DOUBLE]
    for i, d in enumerate(dims):
        for fn in (("sum", "min", "max") if len(dims) <= 3 else ("sum", "min" if i % 2 else "max")):
            aggs.append(P.agg_expr(fn, AT, len(aggs) + 1, None, P.slot_ref(d.tid, 2, T.INT64)))
            types.append(T.INT64)
    return aggs, types


def tuples(dims: List[Dim]):
    t = {0: [(1, T.INT64), (2, T.DOUBLE), (3, T.INT32)] + [(10 + d.tid, d.fk_type) for d in dims]}
    for d in dims:
        t[d.tid] = [(1, d.key_type), (2, T.INT64), (3, T.INT32)]
    return t


def join_tree(dims: List[Dim], leaf=None):
    """right-deep: JOIN(D_n, ... JOIN(D_1, F)), each dimension the outer (build) child as the reference plans it"""
    j = P.scan(0)
    for d in dims:
        j = P.join(leaf(d) if leaf else P.scan(d.tid), j, [on(d)])
    return j


def group_keys(dims: List[Dim]) -> List[str]:
    return ["0_3", f"{dims[0].tid}_3"]


def agg_plan(dims: List[Dim], grouped=True, leaf=None) -> P.Plan:
    """GROUP BY the fact's group and the first dimension's key % 7 (or no GROUP BY) over the join of the fact with `dims`: with one
    dimension the two-table join (PK_JOIN_AGG), with more a star join (PK_STAR_AGG)"""
    aggs, types = aggregates(dims)
    group = [P.slot_ref(0, 3, T.INT32), P.slot_ref(dims[0].tid, 3, T.INT32)] if grouped else []
    a = P.agg(join_tree(dims, leaf), AT, group, aggs)
    return P.Plan(a if grouped else P.packet(a), {**tuples(dims), AT: P.agg_tuple_slots(aggs, types)})


def fused_plan(dim: Dim) -> P.Plan:
    """the shape of the two-table join's fused probe: the only dimension column read is the 4-byte GROUP BY attribute"""
    aggs = [P.agg_expr("count_star", AT, 1), P.agg_expr("sum", AT, 2, None, P.slot_ref(0, 2, T.DOUBLE))]
    a = P.agg(P.join(P.scan(dim.tid), P.scan(0), [on(dim)]), AT, [P.slot_ref(dim.tid, 3, T.INT32)], aggs)
    return P.Plan(a, {**tuples([dim]), AT: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})


# ---- what the build picks (join_build_index in csrc/join.cu) ----
def index_mode(dim: Dim, cast: Optional[int] = None) -> str:
    """"dense" when the biased key range is at most 4 * rows + 1024 (and 2^30), else "packed" for keys of at most 4 bytes, else (and
    whenever a key repeats) "multimap".  Signed keys are biased by 2^63, so that their order is the unsigned order of the image."""
    cast = cast or cast_of(dim.key_type, dim.fk_type)
    live = dim.live_keys()
    if len(set(live)) != len(live):
        return "multimap"
    img = [(k + 2**63) if cast in SIGNED else k for k in live]
    lo, hi = (min(img), max(img)) if img else (2**64 - 1, 0)
    span = (hi - lo + 1) % 2**64 if hi >= lo else 0
    if 0 < span <= 4 * len(dim.keys) + 1024 and span <= 2**30:
        return "dense"
    return "packed" if key_bytes(cast) <= 4 else "multimap"


def packed_wrap_keys(nd: int) -> List[int]:
    """`nd` distinct INT32 keys that are multiples of 2^20 plus one offset, chosen so that every key hashes to a slot 10 before the end
    of the packed table (2 * nd rounded up to a power of two, at least 1024 slots): the linear probing collides on every key and wraps"""
    cap = 1024
    while cap < 2 * nd:
        cap <<= 1
    off = ((cap - 11) * pow(0x9E3779B1, -1, 2**32)) % 2**32 & (2**20 - 1)
    assert (off * 0x9E3779B1) % 2**32 % cap == cap - 11
    return [k * 2**20 + off for k in range(-(nd // 2), nd - nd // 2)]


# ---- a plain Python reference of agg_plan over a small case ----
def reference(case: Case, grouped=True, dim_ok=None) -> Dict[tuple, tuple]:
    """every joined row enumerated in Python: {group: (COUNT(*), SUM(row id), SUM(value), per dimension SUM / MIN / MAX of attr64)}.
    `dim_ok(dim, row)`: a dimension's own conjuncts"""
    import itertools
    rows_of = []
    for d in case.dims:
        m = {}
        for i, k in enumerate(d.keys):
            if (d.valid is None or d.valid[i]) and (dim_ok is None or dim_ok(d, i)):
                m.setdefault(k, []).append(i)
        rows_of.append(m)
    out: Dict[tuple, list] = {}
    for f in range(case.n):
        parts = []
        for d, m in zip(case.dims, rows_of):
            vals, valid = case.fk[d.tid]
            parts.append([] if valid is not None and not valid[f] else m.get(vals[f], []))
        for combo in itertools.product(*parts):
            key = (int(case.group[f]), case.dims[0].keys[combo[0]] % 7) if grouped else ()
            acc = out.setdefault(key, [0, 0, 0.0] + [None] * (3 * len(case.dims)))
            acc[0] += 1
            acc[1] += f * 3 + case.rowid0
            acc[2] += float(case.value[f])
            for j, (d, r) in enumerate(zip(case.dims, combo)):
                a = attr64(d.keys[r])
                s, lo, hi = acc[3 + 3 * j: 6 + 3 * j]
                acc[3 + 3 * j: 6 + 3 * j] = [(s or 0) + a, a if lo is None else min(lo, a), a if hi is None else max(hi, a)]
    return {k: tuple(v) for k, v in out.items()}

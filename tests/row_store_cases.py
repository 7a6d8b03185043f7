"""Rows that pass through the device row store (csrc/prims.cu RowStore) unchanged: tables whose payload columns carry every column
type under five NULL layouts, the plans that drive each user of the store, and a NumPy reference of which input rows come out.
Shared by tests/test_row_store_plans.py (host only: lowering, the oracle against the reference) and tests/test_gpu_row_store.py.

Every table has a unique INT64 row id in slot 1, so an output row names the input rows it came from.  A payload is copied, never
computed, so the check is exact: each output cell has the bytes and the validity bit of the input cell its row id points at (floats
by bit pattern: -0.0 is not +0.0, a NaN keeps its payload).  The aggregates over joins (MIN / MAX / COUNT) are computed in NumPy
over the same joined row ids.

The users of the store and the plans that reach them:
- retention of ORDER BY / filter rows (sort.cu): where_plan (store_copy_out, with a LIMIT that ends mid-batch: its skip), sort_plan
  (store_gather through the sort's permutation);
- the window stage's rows, and the window rows handed to an outer ORDER BY (window.cu -> bkgpu_plan::post): window_plan;
- a join's build side and the joined rows it returns (join.cu: k_join_rows_gather into the post input): join_rows_plan;
- the FK -> PK gather (k_join_gather into the join chunk, reserved without null bytes): join_agg_plan, INNER over unique build keys;
- the FULL join's chunk under an aggregate, every column packed: join_agg_plan, FULL;
- the star join's chunk (null bytes reserved only for a source with validity): star_plan."""
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from baikaldb_b200 import plan as P
from baikaldb_b200.column import Column, make_column
from baikaldb_b200.plan import PrimitiveType as T, storage_dtype
from tests.agg_type_cases import FLOATS, RANGES, TYPES, column_array, edges, tname

# the 15 payload types, five per table: a plan references at most 16 input columns (MAX_COLS), a join two tables' worth
GROUPS = {"bool_ints": TYPES[0:5], "uints_float": TYPES[5:10], "double_dates": TYPES[10:15]}
LAYOUTS = ("none", "all", "seam", "late", "early")
# batch sizes of the large tables: the cumulative cuts (1, 8, 17, 65_536, 65_539, 131_076, 131_093) cross the retained store's 65,536-row
# floor and its first doubling at offsets that are not multiples of 8
CUTS = [1, 7, 9, 65_519, 3, 65_537, 17]
N_BIG = 140_000
ID, KEY, GRP, PAY = 1, 2, 3, 4      # slots: row id (INT64), join key (INT32), group (INT32), first payload
AT = 5                              # aggregate tuple (the oracle takes tuple ids below 8)
WT = 6                              # window output tuple


def gname(types) -> str:
    return "-".join(tname(t) for t in types)


# ---------------------------------------------------------------- tables
def payload_values(rng, t: int, n: int, nans: bool = True) -> np.ndarray:
    """n values of type t in its storage dtype: random values over the type's range, a fifth of them replaced by its edges
    (min / max, +-0.0, +-inf, FLOAT subnormals, NaNs with distinct payload bits); `nans=False` leaves the NaNs out (MIN / MAX)"""
    dt = np.dtype(storage_dtype(t))
    if t in FLOATS:
        x = (rng.normal(size=n) * 10.0 ** rng.integers(-3, 4, n)).astype(dt)
    else:
        lo, hi = RANGES[t]
        x = rng.integers(lo, hi, n, endpoint=True, dtype=np.uint64 if t in (T.UINT64, T.DATETIME) else np.int64).astype(dt)
    e = [v for v in edges(t) if nans or not (t in FLOATS and v != v)]
    ebits = column_array(t, e).view(f"u{dt.itemsize}")
    u = x.view(f"u{dt.itemsize}")   # (edges go in by their bits: a float assignment could quieten a signalling NaN)
    pos = np.flatnonzero(rng.random(n) < 0.2)
    u[pos] = ebits[rng.integers(0, len(ebits), len(pos))]
    u[:min(n, len(ebits))] = ebits[:min(n, len(ebits))]
    return x


def bounds(n: int, cuts: Sequence[int]) -> List[int]:
    """the batch boundaries [0, c0, c0 + c1, ..., n] of `cuts` and the rest"""
    b = [0]
    for c in cuts:
        b.append(min(n, b[-1] + c))
    return b + [n] if b[-1] < n else b


def validity(layout: str, n: int, cuts: Sequence[int], rng) -> Optional[np.ndarray]:
    """one payload column's NULLs (False = NULL) by layout: none, all, seam (the rows either side of every batch boundary), late (only
    in the last batch: no bitmap before), early (only in the first batch: no bitmap after)"""
    b = bounds(n, cuts)
    if layout == "none" or n == 0:
        return None
    if layout == "all":
        return np.zeros(n, bool)
    v = np.ones(n, bool)
    if layout == "seam":
        for x in b[1:-1]:
            v[max(x - 1, 0)] = v[min(x, n - 1)] = False
        v[0] = v[n - 1] = False
    elif layout == "late":
        lo = b[-2]
        v[lo:] = rng.random(n - lo) > 0.3
        v[n - 1] = False
    elif layout == "early":
        v[:b[1]] = rng.random(b[1]) > 0.3
        v[0] = False
    return v


class Table:
    """tuple `tid`: row id (slot 1, unique, shuffled, from `id0`), [join key (2)], [group (3)], payloads (4 ..) of `types`"""

    def __init__(self, rng, tid: int, n: int, types, layout: str, cuts=CUTS, key=None, grp=None, id0: int = 0, nans: bool = True,
                 key_valid=None):
        self.tid, self.types, self.cuts, self.n = tid, tuple(types), list(cuts), n
        self.cols = [make_column(tid, ID, T.INT64, id0 + rng.permutation(n).astype(np.int64))]
        if key is not None:
            self.cols.append(make_column(tid, KEY, T.INT32, key, key_valid))
        if grp is not None:
            self.cols.append(make_column(tid, GRP, T.INT32, grp))
        for i, t in enumerate(self.types):
            self.cols.append(make_column(tid, PAY + i, t, payload_values(rng, t, n, nans), validity(layout, n, cuts, rng)))
        self.id0 = id0

    def slots(self) -> List[Tuple[int, int]]:
        return [(c.slot_id, c.prim_type) for c in self.cols]

    def col(self, slot: int) -> Column:
        return next(c for c in self.cols if c.slot_id == slot)

    def payloads(self) -> List[Column]:
        return [c for c in self.cols if c.slot_id >= PAY]

    def ref(self, slot: int) -> P.Expr:
        c = self.col(slot)
        return P.slot_ref(self.tid, slot, c.prim_type)

    def index_of(self, ids: np.ndarray) -> np.ndarray:
        """the input row of each row id (-1 stays -1: the NULL-extended side)"""
        inv = np.empty(self.n, np.int64)
        inv[self.col(ID).values - self.id0] = np.arange(self.n)
        ids = np.asarray(ids, np.int64)
        return np.where(ids >= 0, inv[np.clip(ids - self.id0, 0, max(self.n - 1, 0))], -1)


def empty_like(t: Table) -> List[Column]:
    return [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[:0]) for c in t.cols]


# ---------------------------------------------------------------- plans
def where_plan(t: Table, limit: int = -1, offset: int = 0) -> P.Plan:
    """WHERE id % 3 <> 1 [LIMIT limit OFFSET offset]: retention, store_copy_out"""
    root = P.where(P.scan(t.tid), P.ne(P.mod(t.ref(ID), P.int_lit(3)), P.int_lit(1)))
    return P.Plan(P.limit(root, limit, offset) if limit >= 0 else root, {t.tid: t.slots()})


def where_ids(t: Table, limit: int = -1, offset: int = 0) -> np.ndarray:
    ids = t.col(ID).values
    keep = ids[ids % 3 != 1]
    return keep[offset:] if limit < 0 else keep[offset:offset + limit]


def sort_plan(t: Table, asc: bool = False) -> P.Plan:
    """ORDER BY id: retention, store_gather through the sort's permutation"""
    return P.Plan(P.sort(P.scan(t.tid), [t.ref(ID)], [asc], tuple_id=t.tid), {t.tid: t.slots()})


def sort_ids(t: Table, asc: bool = False) -> np.ndarray:
    ids = np.sort(t.col(ID).values)
    return ids if asc else ids[::-1]


def window_plan(t: Table, outer: Optional[Tuple[int, int]] = None) -> P.Plan:
    """ROW_NUMBER() OVER (PARTITION BY grp ORDER BY id) with every payload; `outer` = (limit, offset): ORDER BY id DESC LIMIT OFFSET
    above the window stage (its rows become the post fragment's input)"""
    st = P.window_stage(P.scan(t.tid), [P.window_expr("row_number", WT, 1)], [t.ref(GRP)], [t.ref(ID)])
    if outer is not None:
        st = P.limit(P.sort(st, [t.ref(ID)], [False], tuple_id=7), outer[0], outer[1])
    return P.Plan(st, {t.tid: t.slots(), WT: [(1, T.INT64)]})


def window_rows(t: Table, outer: Optional[Tuple[int, int]] = None) -> Tuple[np.ndarray, np.ndarray]:
    """(row ids, ROW_NUMBER) in output order"""
    ids, grp = t.col(ID).values, t.col(GRP).values
    o = np.lexsort((ids, grp))
    g = grp[o]
    start = np.r_[0, np.flatnonzero(g[1:] != g[:-1]) + 1] if len(g) else np.zeros(0, np.int64)
    rn = np.arange(len(g)) - np.repeat(start, np.diff(np.r_[start, len(g)])) + 1
    ids, rn = ids[o], rn
    if outer is not None:
        d = np.argsort(-ids, kind="stable")
        ids, rn = ids[d][outer[1]:outer[1] + outer[0]], rn[d][outer[1]:outer[1] + outer[0]]
    return ids, rn


JOIN_TYPES = ("INNER_JOIN", "LEFT_JOIN", "RIGHT_JOIN", "FULL_JOIN")


def on(build: Table, probe: Table) -> P.Expr:
    return P.eq(build.ref(KEY), probe.ref(KEY))


def join_rows_plan(build: Table, probe: Table, jt: str) -> P.Plan:
    """a two-table join that returns its rows: the build side (outer child) retained, the pairs gathered into the post input"""
    return P.Plan(P.join(P.scan(build.tid), P.scan(probe.tid), [on(build, probe)], join_type=getattr(P.JoinType, jt)),
                  {build.tid: build.slots(), probe.tid: probe.slots()})


ARGS_PER_PLAN = 3   # COUNT(*) and three aggregates per argument: a plan takes at most 12 aggregate functions


def arg_chunks(args: Sequence[Column]) -> List[List[Column]]:
    return [list(args[i:i + ARGS_PER_PLAN]) for i in range(0, len(args), ARGS_PER_PLAN)]


def agg_fns(cols: Sequence[Column]) -> Tuple[List[P.Expr], List[int]]:
    """COUNT(*), then MIN, MAX and COUNT of every column"""
    fns, types = [P.agg_expr("count_star", AT, 1)], [T.INT64]
    for i, c in enumerate(cols):
        x = P.slot_ref(c.tuple_id, c.slot_id, c.prim_type)
        fns += [P.agg_expr("min", AT, 2 + 3 * i, None, x), P.agg_expr("max", AT, 3 + 3 * i, None, x), P.agg_expr("count", AT, 4 + 3 * i, None, x)]
        types += [c.prim_type, c.prim_type, T.INT64]
    return fns, types


def join_agg_plan(build: Table, probe: Table, jt: str, args: Sequence[Column]) -> P.Plan:
    """GROUP BY the probe side's group column, agg_fns(args) over the join: the FK -> PK gather (INNER, unique build keys) or the
    FULL join's chunk"""
    fns, types = agg_fns(args)
    j = P.join(P.scan(build.tid), P.scan(probe.tid), [on(build, probe)], join_type=getattr(P.JoinType, jt))
    return P.Plan(P.agg(j, AT, [probe.ref(GRP)], fns), {build.tid: build.slots(), probe.tid: probe.slots(), AT: P.agg_tuple_slots(fns, types)})


def star_plan(fact: Table, dims: Sequence[Table], args: Sequence[Column]) -> P.Plan:
    """fact (FK of dimension d in slot KEY + d - 1 ... see star_tables) INNER-joined to two dimensions, GROUP BY the fact's group,
    agg_fns(args)"""
    fns, types = agg_fns(args)
    j = P.scan(fact.tid)
    for d, dim in enumerate(dims):
        j = P.join(P.scan(dim.tid), j, [P.eq(dim.ref(KEY), P.slot_ref(fact.tid, FK_SLOTS[d], T.INT32))])
    tup = {fact.tid: fact.slots(), AT: P.agg_tuple_slots(fns, types)}
    for dim in dims:
        tup[dim.tid] = dim.slots()
    return P.Plan(P.agg(j, AT, [fact.ref(GRP)], fns), tup)


FK_SLOTS = (10, 11)   # the fact table's foreign keys of dimensions 0 and 1


# ---------------------------------------------------------------- the join reference
def inner_pairs(bkey: Column, pkey: Column) -> Tuple[np.ndarray, np.ndarray]:
    """(probe row, build row) of every pair with equal, non-NULL keys"""
    bv = np.flatnonzero(bkey.valid if bkey.valid is not None else np.ones(len(bkey), bool))
    pv = np.flatnonzero(pkey.valid if pkey.valid is not None else np.ones(len(pkey), bool))
    bo = bv[np.argsort(bkey.values[bv], kind="stable")]
    sk = bkey.values[bo]
    lo = np.searchsorted(sk, pkey.values[pv], "left")
    cnt = np.searchsorted(sk, pkey.values[pv], "right") - lo
    pi = np.repeat(pv, cnt)
    start = np.repeat(np.cumsum(cnt) - cnt, cnt)
    bi = bo[np.arange(len(pi)) - start + np.repeat(lo, cnt)]
    return pi.astype(np.int64), bi.astype(np.int64)


def join_rows(build: Table, probe: Table, jt: str) -> Tuple[np.ndarray, np.ndarray]:
    """(probe row, build row) of the join's output, -1 on the NULL-extended side.  LEFT keeps the build (outer) side's unmatched rows,
    RIGHT the probe (inner) side's, FULL both"""
    pi, bi = inner_pairs(build.col(KEY), probe.col(KEY))
    if jt in ("LEFT_JOIN", "FULL_JOIN"):
        lone = np.setdiff1d(np.arange(build.n), bi)
        pi, bi = np.r_[pi, np.full(len(lone), -1)], np.r_[bi, lone]
    if jt in ("RIGHT_JOIN", "FULL_JOIN"):
        lone = np.setdiff1d(np.arange(probe.n), pi)
        pi, bi = np.r_[pi, lone], np.r_[bi, np.full(len(lone), -1)]
    return pi, bi


def star_rows(fact: Table, dims: Sequence[Table]) -> List[np.ndarray]:
    """[fact row, dim 0 row, dim 1 row] of the star join's output"""
    fi, d0 = inner_pairs(dims[0].col(KEY), fact.col(FK_SLOTS[0]))
    fk1 = fact.col(FK_SLOTS[1])
    sub = make_column(0, 0, T.INT32, fk1.values[fi], None if fk1.valid is None else fk1.valid[fi])
    k, d1 = inner_pairs(dims[1].col(KEY), sub)
    return [fi[k], d0[k], d1]


# ---------------------------------------------------------------- comparison
def _bits(c: Column) -> np.ndarray:
    return c.values.view(f"u{c.values.dtype.itemsize}")


def _valid(c: Column) -> np.ndarray:
    return c.valid if c.valid is not None else np.ones(len(c), bool)


def assert_rows(got: Sequence[Column], sides: Sequence[Tuple[Table, np.ndarray]], ordered: bool, what: str = "gpu"):
    """`got` holds exactly the rows whose input row of each side is given (-1: that side NULL-extended): every column of every side,
    value bytes and validity bits.  Unordered results are matched by their row ids"""
    by = {c.name: c for c in got}
    n = len(sides[0][1])
    assert len(by[f"{sides[0][0].tid}_{ID}"]) == n, (what, "rows", len(by[f"{sides[0][0].tid}_{ID}"]), n)
    want_ids = [np.where(rows >= 0, t.col(ID).values[np.maximum(rows, 0)] if t.n else -1, -1) for t, rows in sides]
    got_ids = [np.where(_valid(by[f"{t.tid}_{ID}"]), by[f"{t.tid}_{ID}"].values, -1) for t, _ in sides]
    go, wo = np.arange(n), np.arange(n)
    if not ordered:
        go, wo = np.lexsort(got_ids[::-1]), np.lexsort(want_ids[::-1])
    for g, w, (t, _) in zip(got_ids, want_ids, sides):
        assert np.array_equal(g[go], w[wo]), (what, f"{t.tid}_{ID}", "row ids differ")
    for (t, rows), w in zip(sides, want_ids):
        r = rows[wo]
        for src in t.cols:
            c = by[src.name]
            assert c.prim_type == src.prim_type, (what, src.name, c.prim_type)
            want_ok = (r >= 0) & (_valid(src)[np.maximum(r, 0)] if t.n else False)
            got_ok = _valid(c)[go]
            bad = np.flatnonzero(got_ok != want_ok)
            assert not len(bad), (what, src.name, tname(src.prim_type), "validity differs at output rows", bad[:5])
            gb, sb = _bits(c)[go][want_ok], _bits(src)[r[want_ok]]
            bad = np.flatnonzero(gb != sb)
            assert not len(bad), (what, src.name, tname(src.prim_type), "bytes differ", [(hex(int(gb[i])), hex(int(sb[i]))) for i in bad[:3]])


def agg_reference(groups: np.ndarray, group_ok: np.ndarray, args: Sequence[Tuple[Column, np.ndarray]]) -> Dict[Optional[int], list]:
    """per group (None: the NULL group) [COUNT(*), then (MIN, MAX, COUNT) of each argument], each argument given as its column and the
    input row of every joined row (-1: NULL-extended).  MIN / MAX as (bits, zero_either_sign) or None"""
    out = {}
    keys = [None if not ok else int(k) for k, ok in zip(groups, group_ok)]
    uniq = sorted(set(k for k in keys if k is not None)) + ([None] if None in keys else [])
    karr = np.array([-2**40 if k is None else k for k in keys], np.int64)
    for k in uniq:
        m = karr == (-2**40 if k is None else k)
        row = [int(m.sum())]
        for c, rows in args:
            r = rows[m]
            ok = (r >= 0) & _valid(c)[np.maximum(r, 0)] if len(c) else np.zeros(len(r), bool)
            vals = c.values[r[ok]]
            for fn in ("min", "max"):
                if not len(vals):
                    row.append(None)
                    continue
                x = vals.min() if fn == "min" else vals.max()
                zero_tie = c.prim_type in FLOATS and x == 0 and bool(np.any(np.signbit(vals[vals == 0]))) and not np.all(np.signbit(vals[vals == 0]))
                row.append((int(np.array([x], vals.dtype).view(f"u{vals.dtype.itemsize}")[0]), zero_tie))
            row.append(int(ok.sum()))
        out[k] = row
    return out


def assert_agg(got: Sequence[Column], want: Dict, group_name: str, args: Sequence[Column], what: str = "gpu"):
    by = {c.name: c for c in got}
    g = by[group_name]
    keys = [int(x) if ok else None for x, ok in zip(g.values, _valid(g))]
    assert sorted(keys, key=lambda k: (k is None, k or 0)) == sorted(want, key=lambda k: (k is None, k or 0)), (what, "groups differ")
    for i, k in enumerate(keys):
        w = want[k]
        assert int(by[f"{AT}_1"].values[i]) == w[0], (what, k, "COUNT(*)")
        for j, c in enumerate(args):
            for o, fn in enumerate(("min", "max", "count")):
                col = by[f"{AT}_{2 + 3 * j + o}"]
                want_v = w[1 + 3 * j + o]
                where = (what, k, fn, c.name, tname(c.prim_type))
                if fn == "count":
                    assert int(col.values[i]) == want_v, where + (int(col.values[i]), want_v)
                elif want_v is None:
                    assert not _valid(col)[i], where + ("want NULL",)
                else:
                    assert _valid(col)[i], where + ("got NULL",)
                    gb = int(_bits(col)[i])
                    if want_v[1]:   # both signs of zero in the group: the reference keeps the first in its scan order
                        assert col.values[i] == 0, where + (col.values[i],)
                    else:
                        assert gb == want_v[0], where + (hex(gb), hex(want_v[0]))


# ---------------------------------------------------------------- the tables of each plan
SMALL_CUTS = [1, 7, 9, 500, 3, 700, 17]   # the same shape over ~2k rows (the host-only check against the oracle)
PROBE_CUTS = [3, 9_000, 13]


def scan_table(rng, types, layout, n=N_BIG, cuts=CUTS) -> Table:
    """one scanned table: row id, a group of 40 values (the window's partition), the payloads"""
    return Table(rng, 0, n, types, layout, cuts, grp=rng.integers(0, 40, n).astype(np.int32))


def join_tables(rng, types, layout, nb=N_BIG, np_=30_000, bcuts=CUTS, pcuts=PROBE_CUTS, unique=False, nans=True) -> Tuple[Table, Table]:
    """build (tuple 1) and probe (tuple 0) sides with payloads of `types` each.  unique: NULL-free build keys 0 .. nb-1, each probe key
    one of them (the FK -> PK shape); else duplicate and NULL keys on both sides, and probe keys without a partner"""
    if unique:
        bkey, bok = rng.permutation(nb).astype(np.int32), None
        pkey, pok = rng.integers(0, max(nb, 1), np_).astype(np.int32), None
    else:
        bkey, bok = rng.integers(0, max(nb, 1), nb).astype(np.int32), rng.random(nb) > 0.03
        pkey, pok = rng.integers(0, nb + nb // 10 + 1, np_).astype(np.int32), rng.random(np_) > 0.03
    build = Table(rng, 1, nb, types, layout, bcuts, key=bkey, key_valid=bok, id0=1_000_000, nans=nans)
    probe = Table(rng, 0, np_, types, layout, pcuts, key=pkey, key_valid=pok, grp=rng.integers(0, 16, np_).astype(np.int32), nans=nans)
    return build, probe


STAR_DIM_CUTS = [300, 400]
STAR_FACT_CUTS = [5_000, 20_000]


def star_tables(rng, types, nf=60_000, dim_nulls=True, fact_layout="late") -> Tuple[Table, List[Table]]:
    """fact (tuple 0): group, foreign keys of both dimensions (slots 10, 11; some without a partner), payload types[0] with validity in
    its last batch only; dimension 0 (tuple 2): unique keys, payloads types[1:3]; dimension 1 (tuple 3): duplicate keys, payloads
    types[3:5].  The dimensions' payloads are NULL in their second batch only"""
    dims = []
    for d, (nd, ts) in enumerate(((1_500, types[1:3]), (1_000, types[3:5]))):
        key = rng.permutation(nd).astype(np.int32) if d == 0 else rng.integers(0, nd // 3, nd).astype(np.int32)
        t = Table(rng, 2 + d, nd, ts, "none", STAR_DIM_CUTS, key=key, id0=10_000 * (d + 1), nans=False)
        if dim_nulls:
            b = bounds(nd, STAR_DIM_CUTS)
            for i, c in enumerate(t.cols):
                if c.slot_id >= PAY:
                    v = np.ones(nd, bool)
                    v[b[1]:b[2]] = rng.random(b[2] - b[1]) > 0.4
                    t.cols[i] = make_column(c.tuple_id, c.slot_id, c.prim_type, c.values, v)
        dims.append(t)
    fact = Table(rng, 0, nf, types[:1], fact_layout, STAR_FACT_CUTS, grp=rng.integers(0, 16, nf).astype(np.int32), nans=False)
    for d, slot in enumerate(FK_SLOTS):
        nd = dims[d].n
        fact.cols.append(make_column(0, slot, T.INT32, rng.integers(0, nd + nd // 20 + 1, nf).astype(np.int32), rng.random(nf) > 0.02))
    return fact, dims


def star_args(fact: Table, dims: Sequence[Table]) -> List[Column]:
    return fact.payloads() + dims[0].payloads() + dims[1].payloads()


def star_reference(fact: Table, dims: Sequence[Table], args: Sequence[Column]) -> Dict:
    fi, d0, d1 = star_rows(fact, dims)
    rows = {fact.tid: fi, dims[0].tid: d0, dims[1].tid: d1}
    return agg_reference(fact.col(GRP).values[fi], np.ones(len(fi), bool), [(c, rows[c.tuple_id]) for c in args])


def join_agg_reference(build: Table, probe: Table, jt: str, args: Sequence[Column]) -> Dict:
    pi, bi = join_rows(build, probe, jt)
    g = probe.col(GRP).values[np.maximum(pi, 0)] if probe.n else np.zeros(len(pi), np.int32)
    return agg_reference(g, pi >= 0, [(c, bi if c.tuple_id == build.tid else pi) for c in args])


def merge_join_case(rng, nb=70_000, np_=30_000):
    """MERGE_AGG (COUNT(*), AVG) GROUP BY a probe column over an INNER join whose build side holds partial rows: unique, NULL-free keys
    (the FK -> PK gather), the COUNT(*) partial in slot 1 and AVG's {double sum, int64 count} blob in the STRING slot 3.  Sums are
    multiples of 1/8, so every order of addition gives the same bits"""
    key = rng.permutation(nb).astype(np.int32)
    cnt = rng.integers(1, 9, nb)
    blob = np.zeros((nb, 16), np.uint8)
    blob[:, :8] = (rng.integers(-8_000, 8_000, nb) / 8.0).astype("<f8").view(np.uint8).reshape(nb, 8)
    blob[:, 8:] = cnt.astype("<i8").view(np.uint8).reshape(nb, 8)
    build = [make_column(AT, 1, T.INT64, cnt), make_column(AT, 3, T.STRING, blob), make_column(AT, KEY + 2, T.INT32, key)]
    probe = [make_column(0, KEY, T.INT32, rng.integers(0, nb, np_).astype(np.int32)), make_column(0, GRP, T.INT32, rng.integers(0, 16, np_).astype(np.int32))]
    aggs = [P.agg_expr("count_star", AT, 1), P.agg_expr("avg", AT, 2, 3, P.slot_ref(0, GRP, T.INT32))]
    j = P.join(P.scan(AT), P.scan(0), [P.eq(P.slot_ref(AT, KEY + 2, T.INT32), P.slot_ref(0, KEY, T.INT32))])
    plan = P.Plan(P.agg(j, AT, [P.slot_ref(0, GRP, T.INT32)], aggs, merge=True),
                  {AT: [(1, T.INT64), (2, T.DOUBLE), (3, T.STRING), (KEY + 2, T.INT32)], 0: [(KEY, T.INT32), (GRP, T.INT32)]})
    return plan, build, probe


def merge_join_reference(build: Sequence[Column], probe: Sequence[Column]) -> Dict[int, Tuple[int, float, int]]:
    """per probe group: merged COUNT(*), AVG's sum and count"""
    bkey = {int(k): i for i, k in enumerate(build[2].values)}
    sums = build[1].values[:, :8].copy().view("<f8").ravel()
    out: Dict[int, list] = {}
    for k, g in zip(probe[0].values, probe[1].values):
        i = bkey[int(k)]
        r = out.setdefault(int(g), [0, 0.0, 0])
        r[0] += int(build[0].values[i]); r[1] += float(sums[i]); r[2] += int(build[0].values[i])
    return {g: tuple(r) for g, r in out.items()}

"""Window stages above an aggregate: the plans the tests build, and their reference rows composed from two existing oracles.

    [LIMIT ->] [SORT ->] (WINDOW -> SORT)+ [HAVING ->] (MERGE_)AGG -> MERGE_AGG's partial rows / JOIN / APPLY

The aggregate's rows come from the C oracle (oracle/oracle.py) where it runs the source (MERGE_AGG over rows, INNER / LEFT / RIGHT joins,
star joins), else from the library's own aggregate without the windows, which tests/test_gpu_full_join.py and tests/test_gpu_apply.py hold
to their NumPy / Acero references (FULL joins, APPLY).  The windows over those rows, and the ORDER BY / LIMIT above them, come from
tests/window_oracle.py's sort, partition, frame and function code.

Group order is defined on neither side, so a comparison never depends on ties: functions whose value depends on the order of peers
(ROW_NUMBER, NTILE, LEAD / LAG, FIRST / LAST / NTH_VALUE, ROWS frames) get order keys that are unique per group, rows are matched on
their group key unless the outer ORDER BY is total, and DOUBLE values are small multiples of 0.25, whose sums are exact in every order.
"""
from __future__ import annotations

import math
import struct
from typing import List, Optional, Sequence, Tuple

import numpy as np

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import execute
from baikaldb_b200.plan import PlanNodeType, PrimitiveType as T
from oracle import oracle
from tests import window_oracle

JT = P.JoinType
# the fact (probe) tuple 0 and the dimension (build) tuple 1 of the joins; the store rows of MERGE_AGG use tuple 0 alone
FACT = [(1, T.INT32), (2, T.INT64), (3, T.DOUBLE), (4, T.INT32), (5, T.DATE)]   # fk, v, x (multiples of 0.25), g, d
DIM = [(1, T.INT32), (2, T.INT32), (3, T.INT64)]                                 # key, class, w
FK, V, X, G, D = (P.slot_ref(0, s, t) for s, t in FACT)
DK, DC, DW = (P.slot_ref(1, s, t) for s, t in DIM)
AGG_TUPLE, WIN_TUPLE = 4, 5
# the aggregates: COUNT(*), SUM(v) INT64, SUM(x) DOUBLE, AVG(x) (final DOUBLE + the intermediate blob), MIN(v), MAX(d)
AGGS = [P.agg_expr("count_star", AGG_TUPLE, 1), P.agg_expr("sum", AGG_TUPLE, 2, None, V), P.agg_expr("sum", AGG_TUPLE, 3, None, X),
        P.agg_expr("avg", AGG_TUPLE, 4, 5, X), P.agg_expr("min", AGG_TUPLE, 6, None, V), P.agg_expr("max", AGG_TUPLE, 7, None, D)]
AGG_SLOTS = P.agg_tuple_slots(AGGS, [T.INT64, T.INT64, T.DOUBLE, T.DOUBLE, T.INT64, T.DATE])
CNT, SUMV, SUMX, AVGX, MINV, MAXD = (P.slot_ref(AGG_TUPLE, s, t) for s, t in [(1, T.INT64), (2, T.INT64), (3, T.DOUBLE), (4, T.DOUBLE), (6, T.INT64), (7, T.DATE)])
AVG_BLOB = P.slot_ref(AGG_TUPLE, 5, T.STRING)


def wx(name, slot, *args):
    return P.window_expr(name, WIN_TUPLE, slot, *args)


def fact(seed: int, n: int, n_groups: int = 60, n_keys: int = 40, null_rate: float = 0.1, g_nulls: bool = True) -> list:
    rng = np.random.default_rng(seed)
    valid = lambda: rng.random(n) > null_rate   # noqa: E731
    return [make_column(0, 1, T.INT32, rng.integers(0, n_keys + 10, n).astype(np.int32), valid()),
            make_column(0, 2, T.INT64, rng.integers(-1000, 1000, n), valid()),
            make_column(0, 3, T.DOUBLE, rng.integers(-400, 400, n) * 0.25, valid()),
            make_column(0, 4, T.INT32, rng.integers(0, n_groups, n).astype(np.int32), valid() if g_nulls else None),
            make_column(0, 5, T.DATE, rng.integers(0, 1 << 20, n).astype(np.uint32), valid())]


def dim(seed: int, n_keys: int = 40, n_class: int = 5) -> list:
    rng = np.random.default_rng(seed + 1000)
    keys = rng.permutation(n_keys + 20)[:n_keys].astype(np.int32)    # unique keys: some fact keys miss, some dimension rows stay unmatched
    return [make_column(1, 1, T.INT32, keys), make_column(1, 2, T.INT32, rng.integers(0, n_class, n_keys).astype(np.int32), rng.random(n_keys) > 0.1),
            make_column(1, 3, T.INT64, rng.integers(0, 100, n_keys))]


def tuples(win_slots: Sequence[Tuple[int, int]] = ()) -> dict:
    return {0: FACT, 1: DIM, AGG_TUPLE: AGG_SLOTS, WIN_TUPLE: list(win_slots)}


# ---------------------------------------------------------------- the aggregate sources
def source(kind: str):
    """-> (the aggregate node below the windows, its group keys, whether its inputs are partial rows).  The group keys: the partition key
    first (a class), then the key that makes groups unique within it."""
    if kind == "merge":   # MERGE_AGG over the stores' partial rows: the partial rows' tuple is the fact tuple's (g, fk) grouping
        return P.agg(P.scan(0), AGG_TUPLE, [FK, G], AGGS, merge=True), [FK, G]
    if kind in ("semi", "anti"):   # IN / NOT IN (SELECT key FROM dim WHERE class < 3): decorrelated into a SEMI / ANTI join
        sub = P.where(P.scan(1), P.lt(DC, P.int_lit(3)))
        a = P.apply(P.scan(0), sub, [P.eq(FK, DK)], JT.SEMI_JOIN if kind == "semi" else JT.ANTI_SEMI_JOIN)
        return P.agg(a, AGG_TUPLE, [FK, G], AGGS), [FK, G]
    jt = {"inner": JT.INNER_JOIN, "left": JT.LEFT_JOIN, "right": JT.RIGHT_JOIN, "full": JT.FULL_JOIN, "full_filter": JT.FULL_JOIN}[kind]
    j = P.join(P.scan(1), P.scan(0), [P.eq(DK, FK)], join_type=jt)
    if kind == "full_filter":   # the filter above a FULL join judges the NULL-extended rows too
        j = P.where(j, P.gt(P.add(V, P.int_lit(0)), P.int_lit(-900)))
    return P.agg(j, AGG_TUPLE, [DC, G], AGGS), [DC, G]


def store_rows(cols: list, regions: int = 3) -> list:
    """the partial rows the stores ship to a MERGE_AGG: the store-side aggregate of each region's slice (the C oracle), concatenated"""
    store = P.Plan(P.agg(P.scan(0), AGG_TUPLE, [FK, G], AGGS), tuples())
    n = len(cols[0])
    step = max(1, (n + regions - 1) // regions)
    parts = [oracle.execute(store.serialize(), [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:a + step],
                                                            None if c.valid is None else c.valid[a:a + step]) for c in cols]).columns
             for a in range(0, max(n, 1), step)]
    out = []
    for cs in zip(*parts):
        vals = np.concatenate([c.values for c in cs])
        valid = None
        if any(c.valid is not None for c in cs):
            valid = np.concatenate([c.valid if c.valid is not None else np.ones(len(c), bool) for c in cs])
        c0 = cs[0]
        out.append(make_column(c0.tuple_id, c0.slot_id, c0.prim_type, vals, valid))
    return out


# ---------------------------------------------------------------- the reference
def split(root: P.PlanNode):
    """-> (LIMIT node, outer SORT, [(WINDOW, SORT)] top-down, the node below the bottom SORT: [HAVING ->] (MERGE_)AGG)"""
    n = root
    while n.node_type in (PlanNodeType.PACKET_NODE, PlanNodeType.SELECT_MANAGER_NODE):
        n = n.children[0]
    limit_node = outer = None
    if n.node_type == PlanNodeType.LIMIT_NODE:
        limit_node, n = n, n.children[0]
    if n.node_type == PlanNodeType.SORT_NODE:
        outer, n = n, n.children[0]
    stages = []
    while n.node_type == PlanNodeType.WINDOW_NODE:
        stages.append((n, n.children[0]))
        n = n.children[0].children[0]
    return limit_node, outer, stages, n


def aggregate_rows(plan: P.Plan, inputs, via: str = "oracle", batches=None) -> list:
    """the rows of [HAVING ->] (MERGE_)AGG below the windows: the C oracle's over `inputs`, or (via="device") the library's aggregate without
    windows over `batches` (default: `inputs` as one batch)"""
    below = split(plan.root)[3]
    if plan.root.node_type == PlanNodeType.PACKET_NODE:   # (a scalar aggregate under a packet emits its default row)
        below = P.packet(below)
    below = P.Plan(below, plan.tuples)
    if via == "oracle":
        return oracle.execute(below.serialize(), inputs).columns
    return execute(below, batches if batches is not None else inputs, device=0)[0]


def windows_over(plan: P.Plan, agg_cols: list) -> Tuple[List[Tuple[int, int, int]], List[dict]]:
    """window_oracle's stages, outer ORDER BY and LIMIT over the aggregate's rows -> (output columns (tuple, slot, prim), rows)"""
    limit_node, outer, stages, _ = split(plan.root)
    types = {(tid, sid): int(pt) for tid, slots in plan.tuples.items() for sid, pt in slots}
    out_cols = [(c.tuple_id, c.slot_id, int(c.prim_type)) for c in agg_cols]
    for tid, sid, pt in out_cols:
        types.setdefault((tid, sid), pt)
    n = len(agg_cols[0]) if agg_cols else 0
    data = [c.to_list() for c in agg_cols]
    rows = [{(c.tuple_id, c.slot_id): data[k][i] for k, c in enumerate(agg_cols)} for i in range(n)]
    for W, S in reversed(stages):
        rows = window_oracle._stable_sort(rows, S.order_exprs, S.is_asc, S.is_null_first, types)
        for slot, ct in window_oracle._window(rows, W, types):
            types.setdefault(slot, ct)
            out_cols.append((slot[0], slot[1], ct))
    if outer is not None:
        rows = window_oracle._stable_sort(rows, outer.order_exprs, outer.is_asc, outer.is_null_first, types)
        if outer.limit >= 0:
            rows = rows[:outer.limit]
    if limit_node is not None:
        off = limit_node.offset
        rows = rows[off:] if limit_node.limit < 0 else rows[off:off + limit_node.limit]
    return out_cols, rows


def _same(a, b, prim: int) -> bool:
    if a is None or b is None:
        return a is None and b is None
    if prim in (T.FLOAT, T.DOUBLE):
        if math.isnan(a) or math.isnan(b):
            return math.isnan(a) and math.isnan(b)
        return struct.pack("<d", float(a)) == struct.pack("<d", float(b))
    return a == b


def assert_rows(got_cols: list, want_cols, want_rows: List[dict], key: Optional[Sequence[Tuple[int, int]]] = None) -> int:
    """the device's rows equal the reference's bit for bit (an AVG blob byte for byte), in the same order — or, with `key` (the group key
    slots), as a set of rows matched on that key"""
    names = [(c.tuple_id, c.slot_id) for c in got_cols]
    # the same columns; the window outputs last, in the same order (the C oracle lists AVG's intermediate slot before its final one)
    n_win = sum(1 for t, _, _ in want_cols if t == WIN_TUPLE)
    assert sorted(names) == sorted((t, s) for t, s, _ in want_cols) and names[len(names) - n_win:] == [(t, s) for t, s, _ in want_cols if t == WIN_TUPLE], (names, want_cols)
    data = [c.to_list() for c in got_cols]
    n = len(got_cols[0]) if got_cols else 0
    assert n == len(want_rows), (n, len(want_rows))
    got_rows = [{(c.tuple_id, c.slot_id): data[k][i] for k, c in enumerate(got_cols)} for i in range(n)]
    if key is not None:
        kf = lambda r: tuple(r[k] for k in key)   # noqa: E731
        by = {kf(r): r for r in want_rows}
        assert len(by) == len(want_rows), "the group key is not unique"
        pairs = [(g, by.get(kf(g))) for g in got_rows]
    else:
        pairs = list(zip(got_rows, want_rows))
    for i, (g, w) in enumerate(pairs):
        assert w is not None, ("no reference row for", g)
        for tid, sid, prim in want_cols:
            assert _same(g[(tid, sid)], w[(tid, sid)], prim), (i, (tid, sid), g[(tid, sid)], w[(tid, sid)])
    return n


def check(plan: P.Plan, inputs, key: Optional[Sequence] = None, via: str = "oracle", batches=None, options=None, got=None) -> int:
    """the plan on the device against the composed reference; `key`: the group key slots (None: the outer ORDER BY is total)"""
    if got is None:
        got, _ = execute(plan, batches if batches is not None else inputs, device=0, options=options)
    want_cols, want_rows = windows_over(plan, aggregate_rows(plan, inputs, via, batches))
    return assert_rows(got, want_cols, want_rows, key)

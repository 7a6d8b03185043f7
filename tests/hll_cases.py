"""Plans with hll_add_agg, shared by the CPU (tests/test_hll_plan.py) and GPU (tests/test_gpu_hll.py) tests: over a scan, a two-table
join, a star join and an APPLY.  Tuple 0 holds the values (slot 1 the group key, slot 2 the hashed argument), the aggregate tuple is 9."""
from baikaldb_b200 import plan as P, queries
from baikaldb_b200.plan import JoinType, PrimitiveType as T

AGG_TUPLE = 9


def hll(slot: int, arg) -> P.Expr:
    return P.agg_expr("hll_add_agg", AGG_TUPLE, slot, None, arg)


def scan_plan(arg_prim: int, grouped: bool = True, arg=None, extra: bool = False, packet: bool = False, where=None) -> P.Plan:
    """SELECT [k,] hll_add_agg(v) [, COUNT(*), SUM(v), AVG(v), COUNT(v)] FROM t [WHERE ...] [GROUP BY k]"""
    v = arg if arg is not None else P.slot_ref(0, 2, arg_prim)
    aggs = [hll(1, v)]
    types = [T.HLL]
    if extra:
        aggs += [P.agg_expr("count_star", AGG_TUPLE, 2), P.agg_expr("sum", AGG_TUPLE, 3, None, P.slot_ref(0, 3, T.DOUBLE)),
                 P.agg_expr("avg", AGG_TUPLE, 4, 5, P.slot_ref(0, 3, T.DOUBLE)), P.agg_expr("count", AGG_TUPLE, 6, None, v)]
        types += [T.INT64, T.DOUBLE, T.DOUBLE, T.INT64]
    child = P.scan(0) if where is None else P.where(P.scan(0), where)
    root = P.agg(child, AGG_TUPLE, [P.slot_ref(0, 1, T.INT32)] if grouped else [], aggs)
    tuples = {0: [(1, T.INT32), (2, arg_prim), (3, T.DOUBLE)], AGG_TUPLE: P.agg_tuple_slots(aggs, types)}
    return P.Plan(P.packet(root) if packet else root, tuples)


def join_plan() -> P.Plan:
    """SELECT `1_2`, hll_add_agg(`0_2`) FROM fact JOIN dim ON `0_1` = `1_1` GROUP BY `1_2` (queries.c3_join_groupby's shape)"""
    aggs = [hll(1, P.slot_ref(0, 2, T.DOUBLE)), P.agg_expr("count_star", AGG_TUPLE, 2)]
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    root = P.agg(j, AGG_TUPLE, [P.slot_ref(1, 2, T.INT32)], aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.DOUBLE)], 1: [(1, T.INT32), (2, T.INT32)], AGG_TUPLE: P.agg_tuple_slots(aggs, [T.HLL, T.INT64])})


def star_plan() -> P.Plan:
    """SELECT d_year, p_brand, hll_add_agg(lo_revenue), COUNT(*) over queries.c6_star_groupby's star join"""
    base = queries.c6_star_groupby()
    aggs = [hll(1, P.slot_ref(0, 4, T.DOUBLE)), P.agg_expr("count_star", AGG_TUPLE, 2)]
    agg = base.root
    root = P.agg(agg.children[0], AGG_TUPLE, agg.group_exprs, aggs)
    tuples = {k: v for k, v in base.tuples.items() if k in queries.STAR_TUPLES}
    tuples[AGG_TUPLE] = P.agg_tuple_slots(aggs, [T.HLL, T.INT64])
    return P.Plan(root, tuples)


def apply_plan(join_type: int = JoinType.SEMI_JOIN) -> P.Plan:
    """SELECT `0_1`, hll_add_agg(`0_2`) FROM t WHERE [NOT] EXISTS (SELECT 1 FROM s WHERE s.`1_1` = t.`0_1`) GROUP BY `0_1`"""
    aggs = [hll(1, P.slot_ref(0, 2, T.INT64))]
    ap = P.apply(P.scan(0), P.where(P.scan(1), P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))), [], join_type)
    root = P.agg(ap, AGG_TUPLE, [P.slot_ref(0, 1, T.INT32)], aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.INT64)], 1: [(1, T.INT32)], AGG_TUPLE: P.agg_tuple_slots(aggs, [T.HLL])})


def merge_plan(grouped: bool = True) -> P.Plan:
    """The db side of a distributed hll_add_agg: MERGE_AGG [GROUP BY `0_1`] over the stores' rows, whose intermediate slot `9_1` holds each
    store's RAW sketch (the argument, `0_3`, is the stores' column: the merge reads only the intermediate)"""
    aggs = [hll(1, P.slot_ref(0, 3, T.INT64))]
    root = P.agg(P.scan(0), AGG_TUPLE, [P.slot_ref(0, 1, T.INT32)] if grouped else [], aggs, merge=True)
    return P.Plan(root, {0: [(1, T.INT32), (3, T.INT64)], AGG_TUPLE: P.agg_tuple_slots(aggs, [T.HLL])})


def two_sketch_plan() -> P.Plan:
    """SELECT `0_1`, hll_add_agg(`0_2`), COUNT(*), hll_add_agg(`0_3`) FROM t GROUP BY `0_1`: two sketches per group"""
    aggs = [hll(1, P.slot_ref(0, 2, T.INT64)), P.agg_expr("count_star", AGG_TUPLE, 2), hll(3, P.slot_ref(0, 3, T.DOUBLE))]
    root = P.agg(P.scan(0), AGG_TUPLE, [P.slot_ref(0, 1, T.INT32)], aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.INT64), (3, T.DOUBLE)], AGG_TUPLE: P.agg_tuple_slots(aggs, [T.HLL, T.INT64, T.HLL])})


def join_float_build_plan() -> P.Plan:
    """SELECT `0_2`, hll_add_agg(`1_2`) FROM fact JOIN dim ON `0_1` = `1_1` GROUP BY `0_2`: a FLOAT argument read on the build side"""
    aggs = [hll(1, P.slot_ref(1, 2, T.FLOAT))]
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    root = P.agg(j, AGG_TUPLE, [P.slot_ref(0, 2, T.INT32)], aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.INT32)], 1: [(1, T.INT32), (2, T.FLOAT)], AGG_TUPLE: P.agg_tuple_slots(aggs, [T.HLL])})

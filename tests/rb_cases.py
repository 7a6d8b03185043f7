"""Plans with rb_build_agg, shared by the CPU (tests/test_rb_plan.py, tests/test_agg_select_rb.py) and GPU (tests/test_gpu_rb.py) tests:
over a scan, a two-table join, a star join and an APPLY.  Tuple 0 holds the values (slot 1 the group key, slot 2 the argument, slot 3 a
DOUBLE), the aggregate tuple is 9."""
from baikaldb_b200 import plan as P, queries
from baikaldb_b200.plan import JoinType, PrimitiveType as T

AGG_TUPLE = 9


def rb(slot: int, arg, name: str = "rb_build_agg") -> P.Expr:
    return P.agg_expr(name, AGG_TUPLE, slot, None, arg)


def scan_plan(arg_prim: int, grouped: bool = True, arg=None, extra: bool = False, packet: bool = False, where=None, name: str = "rb_build_agg",
              merge: bool = False) -> P.Plan:
    """SELECT [k,] rb_build_agg(v) [, COUNT(*), SUM(d), rb_build_agg(k), COUNT(v)] FROM t [WHERE ...] [GROUP BY k]"""
    v = arg if arg is not None else P.slot_ref(0, 2, arg_prim)
    aggs = [rb(1, v, name)]
    types = [T.BITMAP]
    if extra:
        aggs += [P.agg_expr("count_star", AGG_TUPLE, 2), P.agg_expr("sum", AGG_TUPLE, 3, None, P.slot_ref(0, 3, T.DOUBLE)),
                 rb(4, P.slot_ref(0, 1, T.INT32)), P.agg_expr("count", AGG_TUPLE, 5, None, v)]
        types += [T.INT64, T.DOUBLE, T.BITMAP, T.INT64]
    child = P.scan(0) if where is None else P.where(P.scan(0), where)
    root = P.agg(child, AGG_TUPLE, [P.slot_ref(0, 1, T.INT32)] if grouped else [], aggs, merge=merge)
    tuples = {0: [(1, T.INT32), (2, arg_prim), (3, T.DOUBLE)], AGG_TUPLE: P.agg_tuple_slots(aggs, types)}
    return P.Plan(P.packet(root) if packet else root, tuples)


def join_plan(join_type: int = JoinType.INNER_JOIN) -> P.Plan:
    """SELECT `1_2`, rb_build_agg(`0_2`), COUNT(*) FROM dim JOIN fact ON `1_1` = `0_1` GROUP BY `1_2` (LEFT: every dim row, NULL-extended)"""
    aggs = [rb(1, P.slot_ref(0, 2, T.INT64)), P.agg_expr("count_star", AGG_TUPLE, 2)]
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))], join_type)
    root = P.agg(j, AGG_TUPLE, [P.slot_ref(1, 2, T.INT32)], aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.INT64)], 1: [(1, T.INT32), (2, T.INT32)], AGG_TUPLE: P.agg_tuple_slots(aggs, [T.BITMAP, T.INT64])})


def star_plan() -> P.Plan:
    """SELECT d_year, p_brand, rb_build_agg(lo_custkey), COUNT(*) over queries.c6_star_groupby's star join"""
    base = queries.c6_star_groupby()
    aggs = [rb(1, P.slot_ref(0, 1, T.INT32)), P.agg_expr("count_star", AGG_TUPLE, 2)]
    agg = base.root
    root = P.agg(agg.children[0], AGG_TUPLE, agg.group_exprs, aggs)
    tuples = {k: v for k, v in base.tuples.items() if k in queries.STAR_TUPLES}
    tuples[AGG_TUPLE] = P.agg_tuple_slots(aggs, [T.BITMAP, T.INT64])
    return P.Plan(root, tuples)


def apply_plan(join_type: int = JoinType.SEMI_JOIN) -> P.Plan:
    """SELECT `0_1`, rb_build_agg(`0_2`) FROM t WHERE [NOT] EXISTS (SELECT 1 FROM s WHERE s.`1_1` = t.`0_1`) GROUP BY `0_1`"""
    aggs = [rb(1, P.slot_ref(0, 2, T.INT64))]
    ap = P.apply(P.scan(0), P.where(P.scan(1), P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))), [], join_type)
    root = P.agg(ap, AGG_TUPLE, [P.slot_ref(0, 1, T.INT32)], aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.INT64)], 1: [(1, T.INT32)], AGG_TUPLE: P.agg_tuple_slots(aggs, [T.BITMAP])})


def many_plan(n: int) -> P.Plan:
    """n rb_build_agg over the same column, GROUP BY `0_1`"""
    aggs = [rb(i + 1, P.slot_ref(0, 2, T.INT64)) for i in range(n)]
    root = P.agg(P.scan(0), AGG_TUPLE, [P.slot_ref(0, 1, T.INT32)], aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.INT64)], AGG_TUPLE: P.agg_tuple_slots(aggs, [T.BITMAP] * n)})

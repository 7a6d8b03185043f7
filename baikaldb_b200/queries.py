"""Plan fragments of the BASELINE.json configs, built the way the reference's planner emits them
(worked example: SURVEY.md Appendix A; store-side fragment = AGG -> WHERE_FILTER -> SCAN split off by
src/physical_plan/separate.cpp:241-260)."""
from __future__ import annotations

from . import plan as P
from .plan import PrimitiveType as T


def c1_count_where(k: int = 1 << 19) -> P.Plan:
    """SELECT COUNT(*) FROM t WHERE `0_1` < k      (config C1, store-side fragment)"""
    aggs = [P.agg_expr("count_star", 1, 1)]
    root = P.agg(P.where(P.scan(0), P.lt(P.slot_ref(0, 1, T.INT32), P.int_lit(k))), 1, [], aggs)
    return P.Plan(P.packet(root), {0: [(1, T.INT32)], 1: P.agg_tuple_slots(aggs, [T.INT64])})


def c2_filter_groupby(k: int = 1 << 19, merge: bool = False) -> P.Plan:
    """SELECT `0_1`, COUNT(*), SUM(`0_3`), AVG(`0_4`) FROM t WHERE `0_2` < k GROUP BY `0_1`
    (configs C2 / C4; tuple 1 = aggregate tuple: s1 INT64 count, s2 DOUBLE sum, s3 DOUBLE avg, s4 AVG blob)"""
    aggs = [P.agg_expr("count_star", 1, 1),
            P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE)),
            P.agg_expr("avg", 1, 3, 4, P.slot_ref(0, 4, T.DOUBLE))]
    tuples = {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE), (4, T.DOUBLE)],
              1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE])}
    if merge:  # db side: MERGE_AGG over the stores' rows (separate.cpp:249-258)
        root = P.agg(P.scan(0), 1, [P.slot_ref(0, 1, T.INT32)], aggs, merge=True)
    else:
        child = P.where(P.scan(0), P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(k)))
        root = P.agg(child, 1, [P.slot_ref(0, 1, T.INT32)], aggs)
    return P.Plan(root, tuples)


def c3_join_groupby() -> P.Plan:
    """SELECT `1_2`, COUNT(*), SUM(`0_2`) FROM fact JOIN dim ON `0_1` = `1_1` GROUP BY `1_2`   (config C3).
    The reference builds the hash map on the OUTER (driver) table and probes with the inner one
    (src/exec/join_node.cpp:920-1022): dim is the outer child, fact the inner."""
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE))]
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    root = P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.DOUBLE)], 1: [(1, T.INT32), (2, T.INT32)],
                         2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})


def q17_scalar_subquery(factor: float = 0.2) -> P.Plan:
    """SELECT COUNT(*), SUM(l.price) FROM lineitem l WHERE l.qty < (SELECT factor * AVG(l2.qty) FROM lineitem l2 WHERE l2.partkey = l.partkey)
    (TPC-H Q17's core).  The planner makes the subquery an APPLY (SEMI, max_one_row) whose condition reads the subquery's aggregate as an
    AGG_EXPR; tuple 1 is the outer scan, tuple 0 the subquery's (1 partkey INT32, 2 qty INT32, 3 price DOUBLE each).  Push every batch of
    tuple 0 before the first batch of tuple 1."""
    cols = [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE)]
    avg = P.agg_expr("avg", 4, 1, None, P.slot_ref(0, 2, T.INT32))
    sub = P.agg(P.where(P.scan(0), P.eq(P.slot_ref(0, 1, T.INT32), P.slot_ref(1, 1, T.INT32))), 4, [], [avg])
    cond = P.lt(P.slot_ref(1, 2, T.INT32), P.multiplies(P.double_lit(factor), P.agg_expr("avg", 4, 1, None, P.slot_ref(0, 2, T.INT32))))
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(1, 3, T.DOUBLE))]
    root = P.agg(P.apply(P.scan(1), sub, [cond], P.JoinType.SEMI_JOIN, max_one_row=True), 2, [], aggs)
    return P.Plan(P.packet(root), {0: cols, 1: list(cols), 2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE]),
                                   4: P.agg_tuple_slots([avg], [T.INT32])})


STAR_TUPLES = {0: [(1, T.INT32), (2, T.INT32), (3, T.INT32), (4, T.DOUBLE)],   # lineorder: lo_orderdate, lo_partkey, lo_suppkey, lo_revenue
               1: [(1, T.INT32), (2, T.INT32)],                                # date: d_datekey, d_year
               2: [(1, T.INT32), (2, T.INT32), (3, T.INT32)],                  # part: p_partkey, p_brand, p_category
               3: [(1, T.INT32), (2, T.INT32)]}                                # supplier: s_suppkey, s_region


def c6_star_groupby(category: int = 12, region: int = 1) -> P.Plan:
    """SELECT d_year, p_brand, SUM(lo_revenue), COUNT(*) FROM lineorder JOIN date ON lo_orderdate = d_datekey
    JOIN part ON lo_partkey = p_partkey JOIN supplier ON lo_suppkey = s_suppkey WHERE p_category = 12 AND s_region = 1
    GROUP BY d_year, p_brand   (config C6, SSB Q2.1-like).  A chain of INNER joins whose outer (build) children are the
    dimensions (the reference's hash join builds on the outer child, src/exec/join_node.cpp:920-1022), with the dimension
    filters pushed down to their scans."""
    aggs = [P.agg_expr("sum", 4, 1, None, P.slot_ref(0, 4, T.DOUBLE)), P.agg_expr("count_star", 4, 2)]
    part = P.where(P.scan(2), P.eq(P.slot_ref(2, 3, T.INT32), P.int_lit(category)))
    supp = P.where(P.scan(3), P.eq(P.slot_ref(3, 2, T.INT32), P.int_lit(region)))
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    j = P.join(part, j, [P.eq(P.slot_ref(2, 1, T.INT32), P.slot_ref(0, 2, T.INT32))])
    j = P.join(supp, j, [P.eq(P.slot_ref(3, 1, T.INT32), P.slot_ref(0, 3, T.INT32))])
    root = P.agg(j, 4, [P.slot_ref(1, 2, T.INT32), P.slot_ref(2, 2, T.INT32)], aggs)
    return P.Plan(root, {**STAR_TUPLES, 4: P.agg_tuple_slots(aggs, [T.DOUBLE, T.INT64])})


def c6_star_window(category: int = 12, region: int = 1) -> P.Plan:
    """SELECT d_year, p_brand, SUM(lo_revenue), COUNT(*),
              RANK() OVER (PARTITION BY d_year ORDER BY SUM(lo_revenue) DESC) AS rnk,
              SUM(SUM(lo_revenue)) OVER (PARTITION BY d_year) AS year_revenue
       FROM <C6's star join> GROUP BY d_year, p_brand ORDER BY d_year, rnk, p_brand
    The top brands of every year and the year's total beside them (TPC-DS q47 / q89-like), as the planner emits it: one WINDOW -> SORT pair
    per window spec, the first function on top (select_planner.cpp:705-760), above the db-side aggregate of the join.  The window outputs land
    in tuple 5."""
    base = c6_star_groupby(category, region)
    year, brand = P.slot_ref(1, 2, T.INT32), P.slot_ref(2, 2, T.INT32)
    revenue = P.slot_ref(4, 1, T.DOUBLE)
    total = P.window_stage(base.root, [P.window_expr("sum", 5, 2, revenue)], [year])
    ranked = P.window_stage(total, [P.window_expr("rank", 5, 1)], [year], [revenue], [False])
    root = P.sort(ranked, [year, P.slot_ref(5, 1, T.INT64), brand], [True, True, True], tuple_id=6)
    return P.Plan(root, {**base.tuples, 5: [(1, T.INT64), (2, T.DOUBLE)]})


def c5_topk(k: int = 1000, asc: bool = True) -> P.Plan:
    """SELECT `0_1`, `0_2` FROM t ORDER BY `0_1` ASC LIMIT k          (config C5)"""
    root = P.sort(P.scan(0), [P.slot_ref(0, 1, T.INT64)], [asc], limit=k, tuple_id=0)
    return P.Plan(root, {0: [(1, T.INT64), (2, T.INT32)]})

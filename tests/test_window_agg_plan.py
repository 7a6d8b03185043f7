"""CPU: window stages above an aggregate — the explain text of every accepted source (MERGE_AGG over the stores' rows, aggregates over
INNER / LEFT / RIGHT / FULL joins, a FULL join under a filter, a star join, SEMI / ANTI APPLY), with and without HAVING, the outer ORDER
BY and LIMIT / OFFSET, several stages with shared sorts; each new refusal with its message; and the shapes that stay refused."""
import ctypes

import pytest

from baikaldb_b200 import _lib, plan as P, queries
from baikaldb_b200.plan import PrimitiveType as T
from tests import window_agg_cases as C

OLD = "window stages must sit on [FILTER ->] SCAN: a window over an aggregate or a join is outside the GPU path"
SOURCES = ["merge", "inner", "left", "right", "full", "full_filter", "semi", "anti", "star"]
KIND = {"merge": 1, "inner": 4, "left": 4, "right": 4, "full": 4, "full_filter": 4, "semi": 4, "anti": 4, "star": 6}


def explain(pl: P.Plan):
    b = pl.serialize()
    buf = ctypes.create_string_buffer(1 << 17)
    rc = _lib.lib().bkgpu_plan_explain(b, len(b), buf, len(buf))
    return rc, buf.value.decode()


def refused(pl: P.Plan, msg: str, code: int = -2):
    rc, text = explain(pl)
    assert rc == code and msg in text, (rc, text)


def source(kind):
    """-> (aggregate node, partition key, a key unique within it, tuples)"""
    if kind == "star":
        base = queries.c6_star_groupby()
        return base.root, P.slot_ref(1, 2, T.INT32), P.slot_ref(2, 2, T.INT32), {**base.tuples, 5: []}, P.slot_ref(4, 2, T.INT64)
    agg, (p, g) = C.source(kind)
    return agg, p, g, C.tuples(), C.CNT


def agg_explain(kind):
    agg, _, _, tup, _ = source(kind)
    rc, text = explain(P.Plan(agg, {k: v for k, v in tup.items() if k != C.WIN_TUPLE}))
    assert rc == 0, text
    return text


@pytest.mark.parametrize("having", [False, True])
@pytest.mark.parametrize("top", ["none", "order_by", "order_by_limit", "limit", "offset"])
@pytest.mark.parametrize("kind", SOURCES)
def test_explain_every_source(kind, top, having):
    agg, p, g, tup, cnt = source(kind)
    below = P.where(agg, P.gt(cnt, P.int_lit(1)), node_type=P.PlanNodeType.HAVING_FILTER_NODE) if having else agg
    s0 = P.window_stage(below, [P.window_expr("row_number", 5, 1), P.window_expr("sum", 5, 2, cnt)], [p], [cnt, g], [False, True])
    s1 = P.window_stage(s0, [P.window_expr("lag", 5, 3, cnt, P.int_lit(2), P.int_lit(-1))], [p], [cnt, g], [False, True])   # the same keys: shared
    s2 = P.window_stage(s1, [P.window_expr("rank", 5, 4)], [], [cnt], [True])
    rn = P.slot_ref(5, 1, T.INT64)
    root = {"none": s2, "order_by": P.sort(s2, [p, rn], [True, False], tuple_id=6), "order_by_limit": P.limit(P.sort(s2, [p, rn], [True, True], tuple_id=6), 10, 3),
            "limit": P.limit(s2, 7, 2), "offset": P.limit(s2, -1, 4)}[top]
    tup = {**tup, 5: [(1, T.INT64), (2, T.INT64), (3, T.INT64), (4, T.INT64)]}
    rc, text = explain(P.Plan(root, tup))
    assert rc == 0, text
    assert text.startswith(f"kind={KIND[kind]} ")
    # the aggregate is lowered exactly as without the windows: without the window lines, the explain text is the aggregate's alone
    win_line = ("window stages above the aggregate:", "window stage[", "  partition key:", "  order key:", "  fn ", "post fragment above the window:")
    assert "".join(ln for ln in text.splitlines(True) if not ln.startswith(win_line)) == agg_explain(kind)
    lim, off = {"none": (-1, 0), "order_by": (-1, 0), "order_by_limit": (-1, 0), "limit": (9, 2), "offset": (-1, 4)}[top]
    n_in = text.split("window stages above the aggregate: input columns=")[1].split(" ")[0]
    assert f"window stages above the aggregate: input columns={n_in} having pred_out={0 if having else -1} limit={lim} offset={off} stages=3\n" in text, text
    assert "window stage[0]: sort=new keys=3 partition=1" in text and "window stage[1]: sort=shared keys=3" in text, text
    assert "window stage[2]: sort=new keys=1 partition=0" in text
    assert "fn lag -> 5_3 prim=6 arg=1 default=3 n=2 method=0" in text, text
    if top.startswith("order_by"):
        want = "limit=13 offset=3" if top == "order_by_limit" else "limit=-1 offset=0"
        assert f"post fragment above the window: kind=3 keys=2 {want}\n" in text, text
    else:
        assert "post fragment above the window" not in text
    assert "post fragment above the aggregate" not in text


def test_explain_c6_star_window():
    rc, text = explain(queries.c6_star_window())
    assert rc == 0, text
    assert "kind=6 " in text and "star: fact tuple=0 dims=3" in text
    assert "window stages above the aggregate: input columns=4 having pred_out=-1 limit=-1 offset=0 stages=2" in text
    assert "fn sum -> 5_2 prim=12 arg=1" in text and "fn rank -> 5_1 prim=6" in text
    assert "post fragment above the window: kind=3 keys=3 limit=-1 offset=0" in text


def test_explain_avg_blob_rides_along():
    agg, p, g, tup, cnt = source("merge")
    rc, text = explain(P.Plan(P.window_stage(agg, [P.window_expr("avg", 5, 1, C.AVGX)], [p]), {**tup, 5: [(1, T.DOUBLE)]}))
    assert rc == 0 and "input columns=9 " in text, text


def test_the_pinned_shapes_keep_their_message():
    tup = {0: C.FACT, 1: C.DIM, 3: [(1, T.INT64), (2, T.INT64)]}
    over_scan = P.agg(P.scan(0), 3, [C.FK], [P.agg_expr("count_star", 3, 2)])                  # the store-side aggregate
    refused(P.Plan(P.window_stage(over_scan, [P.window_expr("row_number", 3, 1)]), tup), OLD)
    filtered = P.agg(P.where(P.scan(0), P.gt(C.V, P.int_lit(0))), 3, [C.FK], [P.agg_expr("count_star", 3, 2)])
    refused(P.Plan(P.window_stage(filtered, [P.window_expr("row_number", 3, 1)]), tup), OLD)
    having = P.where(over_scan, P.gt(P.slot_ref(3, 2, T.INT64), P.int_lit(0)), node_type=P.PlanNodeType.HAVING_FILTER_NODE)
    refused(P.Plan(P.window_stage(having, [P.window_expr("row_number", 3, 1)]), tup), OLD)
    join = P.join(P.scan(1), P.scan(0), [P.eq(C.DK, C.FK)])                                      # a join's returned rows
    refused(P.Plan(P.window_stage(join, [P.window_expr("row_number", 3, 1)]), tup), OLD)
    refused(P.Plan(P.window_stage(P.where(P.scan(0), P.gt(C.V, P.int_lit(0)), node_type=P.PlanNodeType.HAVING_FILTER_NODE),
                                  [P.window_expr("row_number", 3, 1)]), tup), OLD)


def test_new_refusals():
    agg, p, g, tup, cnt = source("inner")
    w = lambda below, *a, **k: P.window_stage(below, [P.window_expr("row_number", 5, 1)], *a, **k)   # noqa: E731
    tup1 = {**tup, 5: [(1, T.INT64)]}
    having = P.where(agg, P.gt(cnt, P.int_lit(1)), limit=3, node_type=P.PlanNodeType.HAVING_FILTER_NODE)
    refused(P.Plan(w(having, [p]), tup1), "LIMIT on a HAVING filter below a window is order dependent")
    # an HLL sketch / a BITMAP under a window
    hll = P.agg(P.join(P.scan(1), P.scan(0), [P.eq(C.DK, C.FK)]), 4, [p], [P.agg_expr("hll_add_agg", 4, 1, None, C.V)])
    refused(P.Plan(w(hll, [p]), {**tup1, 4: [(1, T.HLL)]}), "a window above an aggregate that returns an HLL sketch is outside the GPU path")
    rb = P.agg(P.join(P.scan(1), P.scan(0), [P.eq(C.DK, C.FK)]), 4, [p], [P.agg_expr("rb_build_agg", 4, 1, None, C.V)])
    refused(P.Plan(w(rb, [p]), {**tup1, 4: [(1, T.BITMAP)]}), "a window above an aggregate that returns a BITMAP is outside the GPU path")
    # AVG's intermediate blob in a window expression
    refused(P.Plan(P.window_stage(agg, [P.window_expr("max", 5, 1, C.AVG_BLOB)], [p]), tup1), "window max() over a STRING argument is outside the GPU path")
    refused(P.Plan(P.window_stage(agg, [P.window_expr("sum", 5, 1, P.slot_ref(4, 5, T.DOUBLE))], [p]), tup1), "STRING column 4_5 used in an expression")
    refused(P.Plan(w(agg, [p], [P.slot_ref(4, 5, T.INT64)]), tup1), "STRING column 4_5 used in an expression")
    # a column the aggregate does not output, in a window expression / in HAVING
    refused(P.Plan(w(agg, [C.V]), tup1), "a window expression reads a column the aggregate does not output")
    bad_having = P.where(agg, P.gt(C.V, P.int_lit(1)), node_type=P.PlanNodeType.HAVING_FILTER_NODE)
    refused(P.Plan(w(bad_having, [p]), tup1), "HAVING below a window references a column the aggregate does not output")


def test_existing_window_refusals_apply_above_an_aggregate():
    agg, p, g, tup, cnt = source("merge")
    tup1 = {**tup, 5: [(s, T.INT64) for s in range(1, 40)]}
    rn = lambda s=1: P.window_expr("row_number", 5, s)   # noqa: E731
    refused(P.Plan(P.window_stage(agg, [rn()], [p, g], [cnt, C.SUMV, C.MINV]), tup1), "more than 4 partition and order expressions in one window")
    refused(P.Plan(P.window_stage(agg, [rn()], [C.SUMX]), tup1), "PARTITION BY over a FLOAT / DOUBLE key is outside the GPU path")
    refused(P.Plan(P.window_stage(agg, [P.window_expr("count", 5, s, cnt) for s in range(1, 34)], [p]), tup1), "more than 32 window functions in one fragment")
    t = agg
    for s in range(9):
        t = P.window_stage(t, [rn(s + 1)], [p], [cnt if s % 2 else C.SUMV])
    refused(P.Plan(t, tup1), "more than 8 distinct window sorts in one fragment")
    fr = P.frame(P.FrameType.ROWS, P.bound("preceding", 1), P.bound("following", 1))
    refused(P.Plan(P.window_stage(agg, [P.window_expr("rank", 5, 1)], [p], [cnt], window_frame=fr), tup1), "a frame on rank() is outside the GPU path")
    wide = P.frame(P.FrameType.ROWS, P.bound("preceding", 4000), P.bound("following", 100))
    refused(P.Plan(P.window_stage(agg, [P.window_expr("sum", 5, 1, cnt)], [p], [cnt], window_frame=wide), tup1), "a bounded ROWS frame wider than 4096 rows")
    refused(P.Plan(P.window_stage(agg, [rn(1), P.window_expr("rank", 5, 1)], [p]), tup1), "window output column 5_1 appears twice", code=-1)
    refused(P.Plan(P.window_stage(agg, [P.window_expr("row_number", 4, 1)], [p]), tup1), "window output column 4_1 appears twice", code=-1)   # an aggregate's slot

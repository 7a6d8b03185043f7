"""Window fragments on the host: lowering (explain text), every refusal with its message, and the row oracle's partitions."""
import ctypes
import json
import os

import numpy as np
import pytest

from baikaldb_b200 import _lib, plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PrimitiveType as T
from tests import window_oracle

TUP = {0: [(1, T.INT64), (2, T.INT32), (3, T.DOUBLE), (4, T.DATE), (5, T.UINT32)], 1: [(s, T.INT64) for s in range(1, 40)]}
K, V, X, D, U = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32), P.slot_ref(0, 3, T.DOUBLE), P.slot_ref(0, 4, T.DATE), P.slot_ref(0, 5, T.UINT32)


def explain(root, tuples=TUP):
    b = P.Plan(root, tuples).serialize()
    buf = ctypes.create_string_buffer(1 << 16)
    rc = _lib.lib().bkgpu_plan_explain(b, len(b), buf, len(buf))
    return rc, buf.value.decode()


def refused(root, msg, tuples=TUP):
    rc, text = explain(root, tuples)
    assert rc < 0, text
    assert msg in text, text


def w(name, slot, *args):
    return P.window_expr(name, 1, slot, *args)


def test_explain_one_stage():
    rc, text = explain(P.window_stage(P.scan(0), [w("row_number", 1), w("rank", 2), w("sum", 3, X), w("lag", 4, X)], [K], [V]))
    assert rc == 0, text
    assert "kind=7 " in text and "stages=1" in text
    assert "window stage[0]: sort=new keys=2 partition=1 exprs=3 fns=4" in text
    assert "fn sum -> 1_3 prim=12 arg=2 default=-1 n=0 method=1" in text
    assert "fn lag -> 1_4 prim=12 arg=2 default=-1 n=1 method=0" in text


def test_explain_stacked_and_shared_sorts_and_no_keys():
    s0 = P.window_stage(P.where(P.scan(0), P.gt(V, P.int_lit(3))), [w("row_number", 1)], [K], [V])
    s1 = P.window_stage(s0, [w("count_star", 2)], [K], [V])          # same keys: shares the sort
    s2 = P.window_stage(s1, [w("sum", 3, U)], [], [X], [False])       # another sort
    s3 = P.window_stage(s2, [w("count", 4, X)])                       # OVER (): a SORT without keys
    rc, text = explain(s3)
    assert rc == 0, text
    assert "stages=4" in text and "pred_out=0" in text
    assert "window stage[0]: sort=new" in text and "window stage[1]: sort=shared" in text
    assert "window stage[2]: sort=new keys=1 partition=0" in text and "window stage[3]: sort=none keys=0" in text
    assert "fn sum -> 1_3 prim=6" in text   # SUM over UINT32 is INT64 here (AggFnCall's is UINT64)


def test_explain_frames_and_methods():
    fr = P.frame(P.FrameType.ROWS, P.bound("preceding", 2), P.bound("following", 3))
    rc, text = explain(P.window_stage(P.scan(0), [w("avg", 1, X), w("min", 2, D)], [K], [V], window_frame=fr))
    assert rc == 0 and "frame=ROWS 2 PRECEDING .. 3 FOLLOWING" in text and "method=4" in text, text
    fr = P.frame(P.FrameType.RANGE, P.bound("current row"), P.bound("unbounded following"))
    rc, text = explain(P.window_stage(P.scan(0), [w("max", 1, X)], [K], [V], window_frame=fr))
    assert rc == 0 and "frame=RANGE CURRENT ROW .. UNBOUNDED FOLLOWING" in text and "method=2" in text, text
    fr = P.frame(P.FrameType.RANGE, P.bound("current row"), P.bound("current row"))
    rc, text = explain(P.window_stage(P.scan(0), [w("sum", 1, V)], [K], [V], window_frame=fr))
    assert rc == 0 and "method=3" in text, text


def test_explain_outer_order_by_and_limit():
    st = P.window_stage(P.scan(0), [w("row_number", 1)], [K], [V])
    rc, text = explain(P.limit(P.sort(st, [P.slot_ref(1, 1, T.INT64)], [True], tuple_id=2), 10, 5))
    assert rc == 0, text
    assert "post fragment above the window: kind=3 keys=1 limit=15 offset=5" in text
    rc, text = explain(P.limit(st, 7, 3))
    assert rc == 0 and "rows: pred_out=-1 limit=10 offset=3 stages=1" in text, text


def test_existing_sort_refusal_is_unchanged():
    refused(P.sort(P.scan(0), [], [], tuple_id=0), "SORT node without order expressions")


@pytest.mark.parametrize("root,msg", [
    (lambda: P.window(P.sort(P.scan(0), [V], [True]), [w("row_number", 1)], [K], [V], [True]),
     "must order by its partition expressions, then its order expressions"),
    (lambda: P.window(P.sort(P.scan(0), [K, V], [True, True]), [w("row_number", 1)], [K], [V], [False]),
     "must order by its partition expressions, then its order expressions"),
    (lambda: P.window_stage(P.scan(0), [w("sum", 1, X)], [K, V, U], [X, D]), "more than 4 partition and order expressions"),
    (lambda: P.window_stage(P.scan(0), [w("sum", 1, V)], [X], [V]), "PARTITION BY over a FLOAT / DOUBLE key"),
    (lambda: P.window_stage(P.scan(0), [w("sum", 1, D)], [K], [V]), "window sum() over a date/time argument"),
    (lambda: P.window_stage(P.scan(0), [w("avg", 1, D)], [K], [V]), "window avg() over a date/time argument"),
    (lambda: P.window_stage(P.scan(0), [w("sum", 1, X)], [K], [V], window_frame=P.frame(P.FrameType.RANGE, P.bound("preceding", 2), P.bound("current row"))),
     "a RANGE frame with an offset"),
    (lambda: P.window_stage(P.scan(0), [w("sum", 1, X)], [K], [V], window_frame=P.frame(P.FrameType.ROWS, P.FrameBound(P.BoundType.FOLLOWING, True), P.bound("current row"))),
     "an unbounded frame start must be UNBOUNDED PRECEDING"),
    (lambda: P.window_stage(P.scan(0), [w("sum", 1, X)], [K], [V], window_frame=P.frame(P.FrameType.ROWS, P.bound("current row"), P.FrameBound(P.BoundType.PRECEDING, True))),
     "an unbounded frame end must be UNBOUNDED FOLLOWING"),
    (lambda: P.window_stage(P.scan(0), [w("sum", 1, X)], [K], [V], window_frame=P.frame(P.FrameType.ROWS, P.FrameBound(P.BoundType.PRECEDING, False, P.double_lit(1.0)), P.bound("current row"))),
     "a window frame offset must be an integer literal >= 0"),
    (lambda: P.window_stage(P.scan(0), [w("sum", 1, X)], [K], [V], window_frame=P.frame(P.FrameType.ROWS, P.FrameBound(P.BoundType.PRECEDING, False, P.int_lit(-1)), P.bound("current row"))),
     "a window frame offset must be an integer literal >= 0"),
    (lambda: P.window_stage(P.scan(0), [w("rank", 1)], [K], [V], window_frame=P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("current row"))),
     "a frame on rank() is outside the GPU path"),
    (lambda: P.window_stage(P.scan(0), [w("sum", 1, X)], [K], [V], window_frame=P.frame(P.FrameType.ROWS, P.bound("preceding", 3000), P.bound("following", 3000))),
     "a bounded ROWS frame wider than 4096 rows"),
    (lambda: P.window(P.sort(P.scan(0), [K, V], [True, True]), [w("row_number", 1)], [K], [V], [True], limit=1),
     "a LIMIT on a WINDOW node"),
    (lambda: P.window_stage(P.scan(0), [w("ntile", 1, P.int_lit(0))], [K], [V]), "NTILE needs an integer literal > 0"),
    (lambda: P.window_stage(P.scan(0), [w("lag", 1, X, P.int_lit(-2))], [K], [V]), "the LEAD / LAG offset must be an integer literal >= 0"),
    (lambda: P.window_stage(P.scan(0), [w("nth_value", 1, X, P.int_lit(0))], [K], [V]), "NTH_VALUE needs an integer literal > 0"),
    (lambda: P.window_stage(P.scan(0), [w(f"row_number", s) for s in range(1, 34)]), "more than 32 window functions"),
])
def test_refusals(root, msg):
    refused(root(), msg)


def test_more_than_eight_distinct_sorts_refused():
    t = P.scan(0)
    for s in range(9):   # alternating keys: every stage sorts again
        t = P.window_stage(t, [w("row_number", s + 1)], [K], [V if s % 2 else U])
    refused(t, "more than 8 distinct window sorts")


def test_many_stages_with_few_sorts():
    """one WINDOW -> SORT pair per function, as the planner emits them: 24 pairs, 3 distinct sorts"""
    t = P.scan(0)
    for s in range(24):
        t = P.window_stage(t, [w("row_number", s + 1)], [K], [V if s < 8 or s >= 16 else U])
    rc, text = explain(t)
    assert rc == 0 and "stages=24" in text and text.count("sort=new") == 3, text


def test_window_over_an_aggregate_refused():
    a = P.agg(P.scan(0), 3, [K], [P.agg_expr("count_star", 3, 2)])
    refused(P.window_stage(a, [w("row_number", 1)]), "a window over an aggregate or a join is outside the GPU path",
            {**TUP, 3: [(1, T.INT64), (2, T.INT64)]})


def test_oracle_partitions_match_the_reference_test():
    g = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "window_partitions.json")))
    rows = [{(0, 1): a, (0, 2): b, (0, 3): c} for a, b, c in g["rows"]]
    types = {(0, s): T.INT32 for s in (1, 2, 3)}
    p1, p2 = P.slot_ref(0, 1, T.INT32), P.slot_ref(0, 2, T.INT32)
    assert [list(x) for x in window_oracle.split_into_partitions(rows, [p1, p2], types)] == g["partition_by_0_1_0_2"]
    assert [list(x) for x in window_oracle.split_into_partitions(rows, [], types)] == g["no_partition"]


def test_oracle_against_sql_definitions():
    """ROW_NUMBER / RANK / DENSE_RANK / running SUM / LAG from their SQL definitions, written with numpy"""
    rng = np.random.default_rng(3)
    n = 400
    k, v, x = rng.integers(0, 7, n), rng.integers(0, 20, n).astype(np.int32), rng.normal(size=n)
    cols = [make_column(0, 1, T.INT64, k), make_column(0, 2, T.INT32, v), make_column(0, 3, T.DOUBLE, x)]
    tuples = {0: [(1, T.INT64), (2, T.INT32), (3, T.DOUBLE)], 1: [(s, T.INT64) for s in range(1, 6)]}
    ranking = P.window_stage(P.scan(0), [w("row_number", 1), w("rank", 2), w("dense_rank", 3), w("lag", 5, X)], [K], [V])
    running = P.frame(P.FrameType.RANGE, P.bound("unbounded preceding"), P.bound("current row"))   # the planner's default with ORDER BY
    _, rows = window_oracle.execute(P.Plan(P.window_stage(ranking, [w("sum", 4, X)], [K], [V], window_frame=running), tuples), cols)
    order = np.lexsort((v, k))
    ks, vs, xs = k[order], v[order], x[order]
    assert [r[(0, 1)] for r in rows] == ks.tolist()
    for i, r in enumerate(rows):
        same = np.nonzero(ks == ks[i])[0]
        p0 = same[0]
        assert r[(1, 1)] == i - p0 + 1
        assert r[(1, 2)] == int(np.sum(vs[same] < vs[i])) + 1
        assert r[(1, 3)] == len(np.unique(vs[same][vs[same] < vs[i]])) + 1
        peers_end = same[vs[same] <= vs[i]][-1]
        assert abs(r[(1, 4)] - xs[p0:peers_end + 1].sum()) <= 1e-9 * np.abs(xs[p0:peers_end + 1]).sum()
        assert r[(1, 5)] == (None if i == p0 else xs[i - 1])

"""GPU window fragments against the row oracle (tests/window_oracle.py): every result row equal, in the same order."""
import zlib

import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import execute
from baikaldb_b200.plan import PrimitiveType as T
from tests import window_oracle

pytestmark = pytest.mark.gpu

SCAN = [(1, T.INT64), (2, T.INT32), (3, T.DOUBLE), (4, T.UINT32), (5, T.DATE), (6, T.INT32)]
K, V, X, U, D, Y = (P.slot_ref(0, s, t) for s, t in SCAN)


def table(seed, n, n_keys=40, null_rate=0.1):
    rng = np.random.default_rng(seed)
    valid = lambda: rng.random(n) > null_rate   # noqa: E731
    return [make_column(0, 1, T.INT64, rng.integers(0, n_keys, n), valid()),
            make_column(0, 2, T.INT32, rng.integers(-20, 20, n).astype(np.int32), valid()),
            make_column(0, 3, T.DOUBLE, rng.normal(size=n) * 100, valid()),
            make_column(0, 4, T.UINT32, rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32), valid()),
            make_column(0, 5, T.DATE, rng.integers(0, 1 << 20, n).astype(np.uint32), valid()),
            make_column(0, 6, T.INT32, np.arange(n, dtype=np.int32))]


def run(root, cols, batches=None, out_tuple=None):
    tuples = {0: SCAN}
    if out_tuple:
        tuples[1] = out_tuple
    pl = P.Plan(root, tuples)
    got, stats = execute(pl, batches if batches is not None else cols, device=0)
    return window_oracle.assert_matches(got, pl, cols), stats


FRAMES = {
    "none": None,
    "whole": P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("unbounded following")),
    "rows_prefix": P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("current row")),
    "rows_prefix_following": P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("following", 2)),
    "rows_prefix_preceding": P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("preceding", 2)),
    "rows_suffix": P.frame(P.FrameType.ROWS, P.bound("preceding", 1), P.bound("unbounded following")),
    "rows_suffix_following": P.frame(P.FrameType.ROWS, P.bound("following", 3), P.bound("unbounded following")),
    "rows_bounded": P.frame(P.FrameType.ROWS, P.bound("preceding", 3), P.bound("following", 2)),
    "rows_bounded_empty": P.frame(P.FrameType.ROWS, P.bound("following", 2), P.bound("preceding", 1)),
    "rows_ahead": P.frame(P.FrameType.ROWS, P.bound("following", 1), P.bound("following", 4)),
    "range_prefix": P.frame(P.FrameType.RANGE, P.bound("unbounded preceding"), P.bound("current row")),
    "range_suffix": P.frame(P.FrameType.RANGE, P.bound("current row"), P.bound("unbounded following")),
    "range_peers": P.frame(P.FrameType.RANGE, P.bound("current row"), P.bound("current row")),
}


def frame_fns(arg, first_slot=1, date=False):
    names = ["min", "max", "first_value", "last_value", "count"] if date else ["count_star", "count", "sum", "avg", "min", "max", "first_value", "last_value"]
    fns = [P.window_expr(nm, 1, first_slot + i, *([] if nm == "count_star" else [arg])) for i, nm in enumerate(names)]
    fns.append(P.window_expr("nth_value", 1, first_slot + len(names), arg, P.int_lit(2)))
    return fns


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("arg", ["int32", "int64", "uint32", "double", "date", "expr"])
def test_frames_by_argument_type(frame, arg):
    cols = table(zlib.crc32(f"{frame}/{arg}".encode()), 3000)
    a = {"int32": V, "int64": K, "uint32": U, "double": X, "date": D, "expr": P.add(V, P.multiplies(X, P.double_lit(0.5)))}[arg]
    fns = frame_fns(a, date=arg == "date")
    run(P.window_stage(P.scan(0), fns, [K], [V, Y], [True, False], window_frame=FRAMES[frame]), cols)


def test_ranking_and_offsets_with_null_keys():
    cols = table(7, 5000, n_keys=30, null_rate=0.2)
    fns = [P.window_expr("row_number", 1, 1), P.window_expr("rank", 1, 2), P.window_expr("dense_rank", 1, 3), P.window_expr("percent_rank", 1, 4),
           P.window_expr("cume_dist", 1, 5), P.window_expr("ntile", 1, 6, P.int_lit(4)), P.window_expr("ntile", 1, 7, P.int_lit(1000)),
           P.window_expr("lead", 1, 8, X), P.window_expr("lag", 1, 9, V, P.int_lit(3)), P.window_expr("lead", 1, 10, U, P.int_lit(2), P.add(V, P.int_lit(100))),
           P.window_expr("lag", 1, 11, D, P.int_lit(0)), P.window_expr("lag", 1, 12, K, P.int_lit(2), P.null_lit())]
    for asc in (True, False):
        run(P.window_stage(P.scan(0), fns, [K], [V], [asc]), cols)


def test_no_partition_no_order_all_peers():
    cols = table(11, 4000)
    fns = [P.window_expr("row_number", 1, 1), P.window_expr("rank", 1, 2), P.window_expr("cume_dist", 1, 3), P.window_expr("sum", 1, 4, X),
           P.window_expr("dense_rank", 1, 5), P.window_expr("percent_rank", 1, 6)]
    run(P.window_stage(P.scan(0), fns), cols)                               # OVER (): one partition, every row a peer
    run(P.window_stage(P.scan(0), fns, [], [V]), cols)                       # ORDER BY only
    run(P.window_stage(P.scan(0), fns, [K]), cols)                           # PARTITION BY only: rank 1, cume_dist 1
    same = [make_column(0, s, t, np.full(3000, 5) if s in (1, 2) else c.values[:3000]) for (s, t), c in zip(SCAN, cols)]
    run(P.window_stage(P.scan(0), fns, [K], [V],
                       window_frame=None), same)                             # all rows peers of one partition


@pytest.mark.parametrize("asc", [True, False])
def test_signed_zero_order_keys_are_equal(asc):
    """-0.0 and +0.0 are one sort key (MemRowCompare): such rows stay in arrival order, fall through to the next ORDER BY key, and are
    peers.  ROW_NUMBER and LAG of the arrival index show the order the rows reached the window in, RANK / DENSE_RANK the peer groups."""
    rng = np.random.default_rng(23)
    n = 6000
    cols = table(23, n, n_keys=5)
    cols[2] = make_column(0, 3, T.DOUBLE, rng.choice(np.array([-0.0, 0.0, -0.0, 0.0, 1.5, -2.0]), n), rng.random(n) > 0.05)
    fns = [P.window_expr("row_number", 1, 1), P.window_expr("rank", 1, 2), P.window_expr("dense_rank", 1, 3), P.window_expr("lag", 1, 4, Y),
           P.window_expr("cume_dist", 1, 5)]
    run(P.window_stage(P.scan(0), fns, [K], [X], [asc]), cols)                     # ties between the zeros: arrival order
    run(P.window_stage(P.scan(0), fns, [K], [X, V], [asc, not asc]), cols)         # ... and then the next key


def test_ragged_batches_filter_and_zero_rows():
    cols = table(13, 20000, n_keys=7)
    cuts = [0, 1, 777, 778, 9000, 20000]
    batches = [[make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b], None if c.valid is None else c.valid[a:b]) for c in cols]
               for a, b in zip(cuts, cuts[1:])]
    fr = FRAMES["range_prefix"]
    ranked = P.window_stage(P.where(P.scan(0), P.gt(V, P.int_lit(-10))), [P.window_expr("row_number", 1, 1)], [K], [V])
    root = P.window_stage(ranked, [P.window_expr("sum", 1, 2, K)], [K], [V], window_frame=fr)
    run(root, cols, batches=batches)
    empty = [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[:0]) for c in cols]
    assert run(root, empty)[0] == 0


def test_limit_offset_and_outer_order_by():
    cols = table(17, 6000)
    st = P.window_stage(P.scan(0), [P.window_expr("row_number", 1, 1), P.window_expr("sum", 1, 2, X)], [K], [V])
    out = [(1, T.INT64), (2, T.DOUBLE)]
    run(P.limit(st, 100, 37), cols, out_tuple=out)
    run(P.limit(st, -1, 5990), cols, out_tuple=out)
    rn = P.slot_ref(1, 1, T.INT64)
    run(P.limit(P.sort(st, [rn], [True], tuple_id=2), 25), cols, out_tuple=out)            # ORDER BY rn LIMIT 25 (top-k)
    run(P.limit(P.sort(st, [rn, P.slot_ref(1, 2, T.DOUBLE)], [False, True], tuple_id=2), 5000, 100), cols, out_tuple=out)   # full sort


def test_two_stacked_specs_with_different_sorts():
    cols = table(19, 8000, n_keys=25)
    s0 = P.window_stage(P.scan(0), [P.window_expr("row_number", 1, 1), P.window_expr("lag", 1, 2, X)], [K], [V])
    s1 = P.window_stage(s0, [P.window_expr("rank", 1, 3)], [U], [X], [False])
    s2 = P.window_stage(s1, [P.window_expr("max", 1, 4, K), P.window_expr("count", 1, 5, X)], [U], [X], [False],
                        window_frame=FRAMES["rows_bounded"])                                  # same keys: shared sort
    run(s2, cols)


def test_reference_case_plan():
    """test_window.cpp case_plan: its 24 window functions over its MockScanNode table (slots 0_1 0_2 0_3 INT32), written as the
    planner emits them — one WINDOW -> SORT pair per function (select_planner.cpp:705-760), the first function on top, with the
    planner's default frame for value functions without one (RANGE UNBOUNDED PRECEDING .. CURRENT ROW with an ORDER BY, the whole
    partition without, logical_planner.cpp:2425-2442) and none for ranking / NTILE / LEAD / LAG"""
    rows = []
    for i in range(6):
        for j in range(i + 1):
            rows += [[i, i, i * 10 + j]] * (2 if i == 4 else 1)
    a = np.array(rows, dtype=np.int32)
    scan = [(1, T.INT32), (2, T.INT32), (3, T.INT32)]
    cols = [make_column(0, s, T.INT32, a[:, s - 1]) for s, _ in scan]
    c1, c2, c3 = (P.slot_ref(0, s, T.INT32) for s, _ in scan)
    rows_1p_1f = P.frame(P.FrameType.ROWS, P.bound("preceding", 1), P.bound("following", 1))
    rows_up_2f = P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("following", 2))
    range_up_cur = P.frame(P.FrameType.RANGE, P.bound("unbounded preceding"), P.bound("current row"))
    range_whole = P.frame(P.FrameType.RANGE, P.bound("unbounded preceding"), P.bound("unbounded following"))
    dflt = lambda: P.add(P.add(c1, c1), P.int_lit(1))   # noqa: E731  col1 + col1 + 1
    by_c1, by_c3 = ([c1], [c1]), ([c1], [c3])
    specs = [  # (name, args, (partition, order), frame) in the SELECT list's order
        ("count_star", [], by_c1, rows_1p_1f), ("avg", [c2], by_c1, rows_1p_1f), ("sum", [c3], by_c1, rows_up_2f),
        ("min", [c3], by_c1, rows_1p_1f), ("max", [c3], by_c1, rows_1p_1f),
        ("row_number", [], by_c3, None), ("rank", [], by_c3, None), ("dense_rank", [], by_c3, None), ("percent_rank", [], by_c3, None),
        ("cume_dist", [], by_c1, None), ("ntile", [P.int_lit(5)], by_c1, None),
        ("lead", [c1], by_c1, None), ("lead", [c1, P.int_lit(2)], by_c1, None), ("lead", [c1, P.int_lit(2), dflt()], by_c1, None),
        ("lead", [c1, P.int_lit(2), dflt()], by_c1, None), ("lead", [c1, P.int_lit(2), dflt()], by_c1, None),
        ("lag", [c1], by_c1, None), ("lag", [c1, P.int_lit(2)], by_c1, None), ("lag", [c1, P.int_lit(2), dflt()], by_c1, None),
        ("first_value", [P.add(c1, P.int_lit(2))], by_c1, rows_1p_1f), ("last_value", [c1], by_c1, rows_1p_1f),
        ("nth_value", [P.multiplies(c1, P.int_lit(3)), P.int_lit(2)], by_c1, rows_1p_1f),
        ("nth_value", [P.multiplies(c1, P.int_lit(3)), P.int_lit(2)], by_c1, range_up_cur),
        ("nth_value", [P.multiplies(c1, P.int_lit(3)), P.int_lit(2)], ([], []), range_whole),
    ]
    assert len(specs) == 24
    t = P.scan(0)
    for slot in range(len(specs), 0, -1):   # bottom-up: the last function's pair sits on the scan
        name, args, (part, order), fr = specs[slot - 1]
        t = P.window_stage(t, [P.window_expr(name, 1, slot, *args)], part, order, window_frame=fr)
    pl = P.Plan(t, {0: scan})
    got, _ = execute(pl, cols, device=0)
    assert window_oracle.assert_matches(got, pl, cols) == 26
    assert len(got) == 3 + 24


def test_one_million_rows():
    cols = table(23, 1_000_000, n_keys=5000, null_rate=0.05)
    fns = [P.window_expr("row_number", 1, 1), P.window_expr("rank", 1, 2), P.window_expr("sum", 1, 3, X), P.window_expr("lag", 1, 4, X),
           P.window_expr("count", 1, 5, V), P.window_expr("max", 1, 6, U)]
    run(P.window_stage(P.scan(0), fns, [K], [V, Y]), cols)

"""Window functions over every column type on the GPU, bit for bit: arguments and keys of all 15 types against the row oracle
(tests/window_oracle.py), the segmented scan at its thread / warp / tile / round boundaries against the numpy model
(tests/window_type_cases.py), and the functions' parameters at their edges."""
import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import execute
from baikaldb_b200.plan import PrimitiveType as T
from tests import window_oracle
from tests.window_type_cases import (FLOATS, LAYOUTS, SCAN_FNS, SCAN_SCAN, SCAN_SIZES, TYPES, arg_fns, arg_scan, arg_table,
                                     key_scan, key_table, scan_fns, scan_model, scan_table, seed_of, tname)

pytestmark = pytest.mark.gpu

FRAMES = {
    "none": None,
    "whole": P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("unbounded following")),
    "rows_prefix": P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("current row")),
    "rows_suffix": P.frame(P.FrameType.ROWS, P.bound("current row"), P.bound("unbounded following")),
    "rows_bounded": P.frame(P.FrameType.ROWS, P.bound("preceding", 3), P.bound("following", 2)),
    "range_prefix": P.frame(P.FrameType.RANGE, P.bound("unbounded preceding"), P.bound("current row")),
    "range_suffix": P.frame(P.FrameType.RANGE, P.bound("current row"), P.bound("unbounded following")),
    "range_peers": P.frame(P.FrameType.RANGE, P.bound("current row"), P.bound("current row")),
}


def valid(c) -> np.ndarray:
    return c.valid if c.valid is not None else np.ones(len(c), bool)


def run(root, tuples, cols):
    pl = P.Plan(root, tuples)
    got, _ = execute(pl, cols, device=0)
    return window_oracle.assert_matches(got, pl, cols)


# ---------------------------------------------------------------- arguments
@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("t", TYPES, ids=tname)
def test_argument_types(t, frame):
    """COUNT(*) COUNT SUM AVG MIN MAX FIRST LAST NTH(2) [LEAD LAG] over an argument of type t, through every frame method: WM_FWD
    (prefix frames, the whole partition), WM_BWD (suffix frames), WM_PEER (RANGE CURRENT ROW) and WM_DIRECT (bounded ROWS)"""
    cols = arg_table(t, seed_of("arg", int(t), frame))
    K, O, A = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32), P.slot_ref(0, 3, t)
    root = P.window_stage(P.scan(0), arg_fns(t, A, FRAMES[frame] is not None), [K], [O], window_frame=FRAMES[frame])
    assert run(root, {0: arg_scan(t)}, cols) == len(cols[0])


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("t", FLOATS, ids=tname)
def test_float_expression_argument(t, frame):
    """a DOUBLE expression over a FLOAT / DOUBLE column: x * -1.0 turns every +0.0 into -0.0 and back"""
    cols = arg_table(t, seed_of("expr", int(t), frame))
    K, O = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32)
    A = P.multiplies(P.slot_ref(0, 3, t), P.double_lit(-1.0))
    root = P.window_stage(P.scan(0), arg_fns(T.DOUBLE, A, FRAMES[frame] is not None), [K], [O], window_frame=FRAMES[frame])
    run(root, {0: arg_scan(t)}, cols)


@pytest.mark.parametrize("frame", ["whole", "rows_prefix", "rows_suffix", "rows_bounded", "range_prefix", "range_suffix", "range_peers"])
@pytest.mark.parametrize("t", FLOATS, ids=tname)
def test_signed_zero_sum_min_max(t, frame):
    """SUM of only -0.0 (and NULLs) is -0.0 and AVG of it +0.0; MIN / MAX of +0.0 and -0.0 in different peer groups keep the first
    in frame order: one partition per pattern, each starting with NULLs"""
    pats = [[None, None, -0.0, -0.0, None, -0.0], [None, 0.0, 0.0, -0.0, -0.0, None], [None, -0.0, -0.0, 0.0, 0.0, 0.0],
            [-0.0, 0.0, -0.0, 0.0, -0.0, 0.0], [0.0, -0.0, None, 0.0, -0.0, -0.0]]
    vals = [v for p in pats for v in p]
    n = len(vals)
    part = np.repeat(np.arange(len(pats)), [len(p) for p in pats])
    order = np.concatenate([np.arange(len(p)) for p in pats]).astype(np.int32)   # every row its own peer group
    arr = np.array([0.0 if v is None else v for v in vals], dtype=np.float32 if t == T.FLOAT else np.float64)
    cols = [make_column(0, 1, T.INT64, part.astype(np.int64)), make_column(0, 2, T.INT32, order),
            make_column(0, 3, t, arr, np.array([v is not None for v in vals])), make_column(0, 4, T.INT32, np.arange(n, dtype=np.int32))]
    K, O, A = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32), P.slot_ref(0, 3, t)
    fns = [P.window_expr(nm, 1, s + 1, A) for s, nm in enumerate(["sum", "avg", "min", "max"])]
    for asc in (True, False):
        run(P.window_stage(P.scan(0), fns, [K], [O], [asc], window_frame=FRAMES[frame]), {0: arg_scan(t)}, cols)


# ---------------------------------------------------------------- keys
def ranking_stages(part, order, asc):
    """ROW_NUMBER RANK DENSE_RANK PERCENT_RANK CUME_DIST NTILE(3), then a RANGE-prefix SUM under the same keys (a shared sort)"""
    names = ["row_number", "rank", "dense_rank", "percent_rank", "cume_dist"]
    fns = [P.window_expr(nm, 1, s + 1) for s, nm in enumerate(names)] + [P.window_expr("ntile", 1, 6, P.int_lit(3))]
    s0 = P.window_stage(P.scan(0), fns, part, order, asc)
    return P.window_stage(s0, [P.window_expr("sum", 1, 7, P.slot_ref(0, 3, T.INT32))], part, order, asc, window_frame=FRAMES["range_prefix"])


@pytest.mark.parametrize("t", [t for t in TYPES if t not in FLOATS], ids=tname)
def test_partition_key_types(t):
    cols = key_table(t, seed_of("part", int(t)))
    Kt, K2, Y = P.slot_ref(0, 1, t), P.slot_ref(0, 2, T.INT32), P.slot_ref(0, 4, T.INT32)
    run(ranking_stages([Kt], [K2], [True]), {0: key_scan(t)}, cols)
    run(ranking_stages([Kt, K2], [Y], [False]), {0: key_scan(t)}, cols)


@pytest.mark.parametrize("asc", [True, False])
@pytest.mark.parametrize("t", TYPES, ids=tname)
def test_order_key_types(t, asc):
    """ORDER BY a key of type t: ties (-0.0 with +0.0 included) are peers; NaN keys by their IEEE bits (DESIGN §4)"""
    cols = key_table(t, seed_of("order", int(t), asc))
    Kt, K2 = P.slot_ref(0, 1, t), P.slot_ref(0, 2, T.INT32)
    run(ranking_stages([K2], [Kt], [asc]), {0: key_scan(t)}, cols)
    run(ranking_stages([], [Kt], [asc]), {0: key_scan(t)}, cols)


@pytest.mark.parametrize("t", TYPES, ids=tname)
def test_four_keys_per_stage(t):
    """the most keys a stage takes: two PARTITION BY and two ORDER BY keys"""
    cols = key_table(t, seed_of("four", int(t)))
    Kt, K2, V, Y = (P.slot_ref(0, s, pt) for s, pt in key_scan(t))
    part, order = ([K2, V], [Kt, Y]) if t in FLOATS else ([Kt, K2], [V, Y])
    run(ranking_stages(part, order, [False, True]), {0: key_scan(t)}, cols)


# ---------------------------------------------------------------- the scan's edges (numpy model)
SCAN_FRAMES = ["whole", "rows_prefix", "rows_suffix", "range_prefix", "range_suffix", "range_peers"]
GROUPS = [1, 3, 256, 2048]   # peer-group sizes: every row, odd runs, one warp's rows, one tile


def scan_cases():
    out = []
    for n in SCAN_SIZES:
        for layout in LAYOUTS:
            if layout == "zrun" and n < 2041:
                continue
            out.append(pytest.param(n, layout, id=f"{n}-{layout}"))
    return out


@pytest.mark.parametrize("n,layout", scan_cases())
def test_scan_edges(n, layout):
    """COUNT / SUM / MIN / MAX over the forward, backward and peer scans at every boundary of the segmented scan (8 items per thread,
    256 rows per warp, 2048 per tile, 524,288 per round of the tile-carry scan), bit for bit: exact integer DOUBLE sums, runs of
    -0.0 and +-0 ties across a tile and a round boundary, INT64 SUMs that wrap"""
    group = GROUPS[seed_of(n, layout) % len(GROUPS)]
    cols = scan_table(n, layout, group, seed_of("scan", n, layout))
    K, O = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT64)
    for frame in SCAN_FRAMES:
        pl = P.Plan(P.window_stage(P.scan(0), scan_fns(), [K], [O], window_frame=FRAMES[frame]), {0: SCAN_SCAN})
        got, _ = execute(pl, cols, device=0)
        g = {(c.tuple_id, c.slot_id): c for c in got}
        assert np.array_equal(g[(0, 1)].values, cols[0].values)   # rows come back in their (already sorted) arrival order
        want = scan_model(cols, frame)
        for s, nm in enumerate(SCAN_FNS):
            c = g[(1, s + 1)]
            wv, wok = want[nm]
            ok = valid(c)
            assert np.array_equal(ok, wok), (frame, nm, np.flatnonzero(ok != wok)[:8])
            gv = c.values.view(np.uint64) if c.values.dtype == np.float64 else c.values
            bad = np.flatnonzero(wok & (gv != wv.astype(gv.dtype)))
            assert len(bad) == 0, (frame, nm, len(bad), bad[:8], gv[bad[:4]], wv[bad[:4]])


# ---------------------------------------------------------------- parameters at their edges
I64_MAX, I32_MAX = (1 << 63) - 1, (1 << 31) - 1
SIZE = 50   # every partition of the parameter table


def param_table():
    rng = np.random.default_rng(5)
    n = SIZE * 6
    return [make_column(0, 1, T.INT64, np.repeat(np.arange(6), SIZE)), make_column(0, 2, T.INT32, rng.integers(0, 10, n).astype(np.int32)),
            make_column(0, 3, T.DOUBLE, rng.integers(-50, 50, n) / 4.0, rng.random(n) > 0.1),
            make_column(0, 4, T.INT32, np.arange(n, dtype=np.int32))]


PARAM_SCAN = [(1, T.INT64), (2, T.INT32), (3, T.DOUBLE), (4, T.INT32)]


def test_lead_lag_ntile_nth_value_parameters():
    """LEAD / LAG by 0, the partition size and INT64_MAX; NTILE of 1, size, size + 1, INT64_MAX; NTH_VALUE of 1, size, size + 1
    and INT32_MAX"""
    cols = param_table()
    K, O, X = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32), P.slot_ref(0, 3, T.DOUBLE)
    fns, s = [], 1
    for off in (0, SIZE - 1, SIZE, I64_MAX):
        for nm in ("lead", "lag"):
            fns.append(P.window_expr(nm, 1, s, X, P.int_lit(off), P.double_lit(-1.5)))
            s += 1
    for k in (1, SIZE, SIZE + 1, I64_MAX):
        fns.append(P.window_expr("ntile", 1, s, P.int_lit(k)))
        s += 1
    run(P.window_stage(P.scan(0), fns, [K], [O]), {0: PARAM_SCAN}, cols)
    for fr in (None, FRAMES["rows_prefix"], FRAMES["rows_suffix"]):
        fns = [P.window_expr("nth_value", 1, s + 1, X, P.int_lit(k)) for s, k in enumerate((1, SIZE, SIZE + 1, I32_MAX))]
        run(P.window_stage(P.scan(0), fns, [K], [O], window_frame=fr), {0: PARAM_SCAN}, cols)


def test_frame_offsets_of_int32_max():
    cols = param_table()
    K, O, X = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32), P.slot_ref(0, 3, T.DOUBLE)
    fns = [P.window_expr(nm, 1, s + 1, X) for s, nm in enumerate(["count", "sum", "avg", "min", "max", "first_value", "last_value"])]
    for fr in (P.frame(P.FrameType.ROWS, P.bound("preceding", I32_MAX), P.bound("unbounded following")),
               P.frame(P.FrameType.ROWS, P.bound("following", I32_MAX), P.bound("unbounded following")),
               P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("following", I32_MAX)),
               P.frame(P.FrameType.ROWS, P.bound("unbounded preceding"), P.bound("preceding", I32_MAX))):
        run(P.window_stage(P.scan(0), fns, [K], [O], window_frame=fr), {0: PARAM_SCAN}, cols)


def test_bounded_rows_frame_4096_wide():
    """ROWS BETWEEN 2048 PRECEDING AND 2047 FOLLOWING, the widest frame WM_DIRECT takes, over 10,000 rows in three partitions
    (integer DOUBLE values: every order of addition is exact), against prefix sums"""
    n = 10_000
    rng = np.random.default_rng(9)
    part = (np.arange(n) >= 3000).astype(np.int64) + (np.arange(n) >= 9000)
    x = rng.integers(-1000, 1000, n).astype(np.float64)
    xv = rng.random(n) > 0.1
    cols = [make_column(0, 1, T.INT64, part), make_column(0, 2, T.INT32, np.arange(n, dtype=np.int32)), make_column(0, 3, T.DOUBLE, x, xv),
            make_column(0, 4, T.INT32, np.arange(n, dtype=np.int32))]
    K, O, X = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32), P.slot_ref(0, 3, T.DOUBLE)
    fr = P.frame(P.FrameType.ROWS, P.bound("preceding", 2048), P.bound("following", 2047))
    fns = [P.window_expr("count", 1, 1, X), P.window_expr("sum", 1, 2, X), P.window_expr("first_value", 1, 3, X), P.window_expr("last_value", 1, 4, X)]
    got, _ = execute(P.Plan(P.window_stage(P.scan(0), fns, [K], [O], window_frame=fr), {0: PARAM_SCAN}), cols, device=0)
    g = {(c.tuple_id, c.slot_id): c for c in got}
    i = np.arange(n)
    starts = np.array([0, 3000, 9000])
    ps = starts[part]
    pe = np.array([3000, 9000, n])[part]
    fs, fe = np.maximum(i - 2048, ps), np.minimum(i + 2048, pe)
    assert (fe - fs).max() == 4096
    pc = np.concatenate([[0], np.cumsum(xv)])
    px = np.concatenate([[0], np.cumsum(np.where(xv, x, 0).astype(np.int64))])
    cnt, s = pc[fe] - pc[fs], px[fe] - px[fs]
    assert np.array_equal(g[(1, 1)].values, cnt)
    assert np.array_equal(valid(g[(1, 2)]), cnt > 0)
    sv = s.astype(np.float64)   # (no -0.0 in x: an exact zero sum is +0.0)
    assert np.array_equal(g[(1, 2)].values.view(np.uint64)[cnt > 0], sv.view(np.uint64)[cnt > 0])
    assert np.array_equal(valid(g[(1, 3)]), xv[fs]) and np.array_equal(g[(1, 3)].values[xv[fs]], x[fs][xv[fs]])
    assert np.array_equal(valid(g[(1, 4)]), xv[fe - 1]) and np.array_equal(g[(1, 4)].values[xv[fe - 1]], x[fe - 1][xv[fe - 1]])


def test_lead_defaults_cast_per_type():
    """LEAD's literal default cast to the argument's type, on the device: INT8 <- 1000 is -24, UINT8 <- -1 is 255, INT32 <- +-2.7
    is +-2, FLOAT <- 0.1 is float32(0.1), BOOL <- 5 is 1, DATE <- -1 is 4294967295"""
    cases = [(T.INT8, P.int_lit(1000)), (T.UINT8, P.int_lit(-1)), (T.INT32, P.double_lit(2.7)), (T.INT32, P.double_lit(-2.7)),
             (T.FLOAT, P.double_lit(0.1)), (T.BOOL, P.int_lit(5)), (T.DATE, P.int_lit(-1)), (T.UINT64, P.double_lit(1e19)),
             (T.DATETIME, P.double_lit(-3.5)), (T.INT16, P.double_lit(1e10))]
    for t, lit in cases:
        cols = arg_table(t, seed_of("lead", int(t)))
        K, O, A = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32), P.slot_ref(0, 3, t)
        run(P.window_stage(P.scan(0), [P.window_expr("lead", 1, 1, A, P.int_lit(5), lit)], [K], [O]), {0: arg_scan(t)}, cols)


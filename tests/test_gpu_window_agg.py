"""GPU: window stages above an aggregate (MERGE_AGG over the stores' rows, aggregates over joins, star joins and APPLY), against the
reference composed in tests/window_agg_cases.py: the aggregate's rows from the C oracle (or the library's aggregate alone, which its own
suites hold to their references), the windows over them from tests/window_oracle.py."""
import zlib

import numpy as np
import pytest

from baikaldb_b200 import plan as P, queries
from baikaldb_b200._lib import BkgpuError
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import ColumnSource, GpuExecNode, RowBatch, RuntimeState, execute
from baikaldb_b200.plan import PrimitiveType as T
from tests import window_agg_cases as C
from tests.util import merge_regions, ragged, to_device

pytestmark = pytest.mark.gpu
I64, F64 = T.INT64, T.DOUBLE
# the C oracle runs these sources; FULL joins and APPLY come from the library's aggregate without the windows
VIA = {"merge": "oracle", "inner": "oracle", "left": "oracle", "right": "oracle", "full": "device", "full_filter": "device", "semi": "device", "anti": "device"}
ROWS_3 = P.frame(P.FrameType.ROWS, P.bound("preceding", 1), P.bound("following", 1))
RANGE_PREFIX = P.frame(P.FrameType.RANGE, P.bound("unbounded preceding"), P.bound("current row"))
ROWS_SUFFIX = P.frame(P.FrameType.ROWS, P.bound("current row"), P.bound("unbounded following"))


def inputs(kind, seed, n=4000, **kw):
    f = C.fact(seed, n, **kw)
    if kind == "merge":
        return C.store_rows(f)
    return C.dim(seed) + f


def batches_of(kind, cols):
    """the join's build side first, then its probe rows: the dimension is the build side of INNER / LEFT / FULL, the fact table of RIGHT
    (lowered as a LEFT join with the children swapped) and of SEMI / ANTI APPLY (the subquery is probed)"""
    if kind == "merge":
        return [cols]
    return [cols[3:], cols[:3]] if kind in ("right", "semi", "anti") else [cols[:3], cols[3:]]


def windowed(agg, keys, stages="all", outer=True, limit=None):
    """stacked window stages over the aggregate: ranking with ties (RANK ... over COUNT), order-dependent functions over an order made
    unique by the group key, framed aggregates, a stage that shares the previous stage's sort, and OVER ().  With the outer ORDER BY
    (the group key: a total order) the first stage and RANK.  -> (root, window slots)"""
    p, g = keys
    uniq = [C.SUMV, g]                                    # (SUM(v) DESC, g): unique within a partition of the group key p
    s1 = P.window_stage(agg, [C.wx("row_number", 1), C.wx("ntile", 2, P.int_lit(3)), C.wx("lag", 3, C.SUMX), C.wx("lead", 4, C.CNT, P.int_lit(2), C.MINV),
                              C.wx("sum", 5, C.CNT), C.wx("first_value", 6, C.AVGX)], [p], uniq, [False, True])
    slots = [(1, I64), (2, I64), (3, F64), (4, I64), (5, I64), (6, F64)]
    if stages == "one":
        top = s1
    elif outer:   # (the ORDER BY above the windows holds at most 16 columns: the aggregate's 9 and 7 window outputs)
        top = P.window_stage(s1, [C.wx("rank", 7)], [p], [C.CNT], [False])
        slots += [(7, I64)]
    else:
        s2 = P.window_stage(s1, [C.wx("rank", 7), C.wx("dense_rank", 8), C.wx("percent_rank", 9), C.wx("cume_dist", 10)], [p], [C.CNT], [False])
        s2 = P.window_stage(s2, [C.wx("sum", 11, C.SUMX), C.wx("max", 12, C.MAXD), C.wx("count", 13, C.AVGX)], [p], [C.CNT], [False],
                            window_frame=RANGE_PREFIX)                                                                   # shared sort
        s3 = P.window_stage(s2, [C.wx("sum", 14, C.SUMV), C.wx("min", 15, C.AVGX), C.wx("last_value", 16, C.CNT)], [p], uniq, [False, True], window_frame=ROWS_3)
        s4 = P.window_stage(s3, [C.wx("avg", 17, C.SUMX), C.wx("nth_value", 18, C.SUMV, P.int_lit(2))], [p], uniq, [False, True], window_frame=ROWS_SUFFIX)   # shared sort
        s5 = P.window_stage(s4, [C.wx("count_star", 19), C.wx("avg", 20, C.CNT), C.wx("max", 21, p)])                      # OVER ()
        top = s5
        slots += [(7, I64), (8, I64), (9, F64), (10, F64), (11, F64), (12, T.DATE), (13, I64), (14, I64), (15, F64), (16, I64), (17, F64), (18, I64),
                  (19, I64), (20, F64), (21, p.col_type)]
    if outer:
        top = P.sort(top, [p, g], [True, True], tuple_id=6)       # the group key: a total order
    if limit is not None:
        top = P.limit(top, *limit)
    return top, slots


def key_slots(keys):
    return [(k.tuple_id, k.slot_id) for k in keys]


@pytest.mark.parametrize("kind", list(VIA))
def test_sources_and_functions(kind):
    agg, keys = C.source(kind)
    cols = inputs(kind, zlib.crc32(kind.encode()))
    root, slots = windowed(agg, keys)
    pl = P.Plan(root, C.tuples(slots))
    assert C.check(pl, cols, via=VIA[kind], batches=batches_of(kind, cols)) > 20
    root, slots = windowed(agg, keys, outer=False)            # the top stage's order: rows matched on the group key
    pl = P.Plan(root, C.tuples(slots))
    C.check(pl, cols, key=key_slots(keys), via=VIA[kind], batches=batches_of(kind, cols))


def test_having_outer_order_by_limit_offset():
    agg, keys = C.source("merge")
    cols = inputs("merge", 3, n=6000)
    having = P.where(agg, P.gt(C.CNT, P.int_lit(1)), node_type=P.PlanNodeType.HAVING_FILTER_NODE)
    p, g = keys
    stage = P.window_stage(having, [C.wx("rank", 1), C.wx("sum", 2, C.SUMX), C.wx("row_number", 3)], [p], [C.SUMV, g], [False, True])
    tup = C.tuples([(1, I64), (2, F64), (3, I64)])
    rank = P.slot_ref(C.WIN_TUPLE, 1, I64)
    for top in (P.limit(P.sort(stage, [rank, p, g], [True, False, True], tuple_id=6), 20, 5),       # full sort + LIMIT / OFFSET
                P.limit(P.sort(stage, [rank, p, g], [True, True, True], tuple_id=6), -1, 7),        # OFFSET only
                P.limit(stage, 15, 4)):                                                           # LIMIT over the top stage's (total) order
        C.check(P.Plan(top, tup), cols)
    assert C.check(P.Plan(P.sort(stage, [p, g], [True, True], tuple_id=6), tup), cols) < len(C.aggregate_rows(P.Plan(agg, tup), cols)[0])   # (HAVING kept fewer groups)


def test_null_groups_empty_input_scalar_and_one_group():
    # NULL group keys and NULL partitions: a LEFT join's NULL-extended class, NULL g
    agg, keys = C.source("right")
    cols = inputs("right", 5, null_rate=0.3)
    root, slots = windowed(agg, keys)
    C.check(P.Plan(root, C.tuples(slots)), cols, batches=batches_of("right", cols))
    # no input rows
    for kind in ("merge", "inner"):
        agg, keys = C.source(kind)
        empty = [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[:0]) for c in inputs(kind, 6)]
        root, slots = windowed(agg, keys)
        assert C.check(P.Plan(root, C.tuples(slots)), empty, batches=batches_of(kind, empty)) == 0
    # a scalar aggregate under a packet: one default row even without input
    join = P.join(P.scan(1), P.scan(0), [P.eq(C.DK, C.FK)])
    scalar = P.agg(join, C.AGG_TUPLE, [], C.AGGS)
    top = P.packet(P.window_stage(scalar, [C.wx("row_number", 1), C.wx("sum", 2, C.CNT), C.wx("lag", 3, C.SUMV, P.int_lit(1), P.int_lit(-1))]))
    tup = C.tuples([(1, I64), (2, I64), (3, I64)])
    cols = inputs("inner", 7)
    for run in (cols, [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[:0]) for c in cols]):
        got, _ = execute(P.Plan(top, tup), batches_of("inner", run), device=0)
        want_cols, want_rows = C.windows_over(P.Plan(top, tup), C.aggregate_rows(P.Plan(P.packet(scalar), tup), run, "device", batches_of("inner", run)))
        assert C.assert_rows(got, want_cols, want_rows) == 1
    # one group
    agg, keys = C.source("merge")
    one = C.fact(8, 500, n_groups=1, n_keys=-9, null_rate=0.0)
    root, slots = windowed(agg, keys)
    assert C.check(P.Plan(root, C.tuples(slots)), C.store_rows(one)) == 1


@pytest.mark.parametrize("groups", [2047, 2049, 4097, 70_001])
def test_group_counts_across_the_scan_tile_and_the_row_store_floor(groups):
    """the window scan's 2,048-row tiles and the row store's 65,536-row first capacity: exactly `groups` groups (g = 0..groups-1, fk = g % 3)"""
    n = groups * 2
    rng = np.random.default_rng(groups)
    g = np.concatenate([np.arange(groups), rng.integers(0, groups, n - groups)]).astype(np.int32)
    f = C.fact(groups, n, null_rate=0.05, g_nulls=False)
    f[0] = make_column(0, 1, T.INT32, (g % 3).astype(np.int32))
    f[3] = make_column(0, 4, T.INT32, g)
    agg, keys = C.source("merge")
    p, gg = keys
    stage = P.window_stage(agg, [C.wx("row_number", 1), C.wx("rank", 2), C.wx("sum", 3, C.CNT), C.wx("lag", 4, C.SUMV)], [p], [C.SUMV, gg], [False, True],
                           window_frame=None)
    stage = P.window_stage(stage, [C.wx("sum", 5, C.SUMX)], [], [C.CNT], [True])       # (a whole-partition frame: the row oracle's frames are O(rows^2))
    pl = P.Plan(stage, C.tuples([(1, I64), (2, I64), (3, I64), (4, I64), (5, F64)]))
    assert C.check(pl, C.store_rows(f, regions=2), key=key_slots(keys)) == groups


TYPES = [T.INT8, T.INT16, T.INT32, T.INT64, T.UINT8, T.UINT16, T.UINT32, T.UINT64, T.FLOAT, T.DOUBLE, T.BOOL, T.DATE, T.DATETIME, T.TIMESTAMP, T.TIME]


def typed_values(rng, prim, n):
    if prim in (T.FLOAT, T.DOUBLE):
        return rng.choice(np.array([-2.5, -0.0, 0.0, 0.25, 1.5, 1e30, -1e-30, np.inf]), n)
    if prim == T.BOOL:
        return rng.integers(0, 2, n)
    if prim == T.TIME:
        return rng.integers(-(1 << 20), 1 << 20, n)
    if prim in (T.INT8, T.UINT8):
        return rng.integers(0 if prim == T.UINT8 else -128, 128, n)
    if prim in (T.INT16, T.UINT16):
        return rng.integers(0 if prim == T.UINT16 else -30000, 30000, n)
    return rng.integers(0, 1 << 31, n) if prim in (T.INT32, T.UINT32, T.DATE, T.TIMESTAMP) else rng.integers(-(1 << 60), 1 << 60, n) if prim == T.INT64 else rng.integers(0, 1 << 62, n)


@pytest.mark.parametrize("prim", TYPES)
def test_group_keys_and_aggregate_outputs_of_every_type(prim):
    """a group key and MIN / MAX of every type through the row store and the window stage, bit for bit, and the AVG blobs passed through"""
    rng = np.random.default_rng(int(prim) + 100)
    n = 3000
    tup0 = [(1, prim), (2, prim), (3, T.DOUBLE)]
    k, v, x = (P.slot_ref(0, s, t) for s, t in tup0)
    aggs = [P.agg_expr("min", 1, 1, None, v), P.agg_expr("max", 1, 2, None, v), P.agg_expr("avg", 1, 3, 4, x), P.agg_expr("count_star", 1, 5)]
    tuples = {0: tup0, 1: P.agg_tuple_slots(aggs, [prim, prim, T.DOUBLE, I64]), C.WIN_TUPLE: [(1, I64), (2, prim), (3, prim), (4, I64)]}
    keys = np.unique(typed_values(rng, prim, 400))
    cols = [make_column(0, 1, prim, rng.choice(keys, n), rng.random(n) > 0.05), make_column(0, 2, prim, typed_values(rng, prim, n), rng.random(n) > 0.2),
            make_column(0, 3, T.DOUBLE, rng.integers(-40, 40, n) * 0.25, rng.random(n) > 0.1)]
    from oracle import oracle
    partial = oracle.execute(P.Plan(P.agg(P.scan(0), 1, [k], aggs), tuples).serialize(), cols).columns
    mn, mx = P.slot_ref(1, 1, prim), P.slot_ref(1, 2, prim)
    stage = P.window_stage(P.agg(P.scan(0), 1, [k], aggs, merge=True), [C.wx("row_number", 1), C.wx("lag", 2, k),
                                                                       C.wx("lead", 3, mn, P.int_lit(1), mx), C.wx("rank", 4)], [], [k], [True])
    pl = P.Plan(P.sort(stage, [k], [False], tuple_id=3), tuples)
    got, _ = execute(pl, partial, device=0)
    want_cols, want_rows = C.windows_over(pl, C.aggregate_rows(pl, partial))
    C.assert_rows(got, want_cols, want_rows)
    blob = [c for c in got if c.slot_id == 4 and c.tuple_id == 1][0]
    assert blob.values.shape[1] == 16


@pytest.mark.parametrize("mode", ["host_batches", "device_batches", "no_lean"])
def test_host_and_device_batches_and_the_kernel_choice(mode):
    agg, keys = C.source("inner")
    cols = inputs("inner", 9, n=20_000)
    root, slots = windowed(agg, keys)
    pl = P.Plan(root, C.tuples(slots))
    dims, fact = cols[:3], cols[3:]
    if mode == "host_batches":
        b = [dims] + ragged(fact, [0, 1, 777, 9000, 20_000])
        C.check(pl, cols, batches=b)
    elif mode == "device_batches":
        C.check(pl, cols, batches=[to_device(dims), to_device(fact)])
    else:
        C.check(pl, cols, batches=[dims, fact], options={"no_lean": 1})
        agg_m, keys_m = C.source("merge")
        rows = inputs("merge", 9)
        root, slots = windowed(agg_m, keys_m)
        for opts in ({"no_lean": 1}, {"lean_fx": 0}, {}):
            C.check(P.Plan(root, C.tuples(slots)), rows, options=opts)


def test_one_handle_three_requests():
    agg, keys = C.source("left")
    root, slots = windowed(agg, keys)
    pl = P.Plan(root, C.tuples(slots))
    runs = [inputs("left", s) for s in (11, 12, 11)]
    node, st = GpuExecNode(), RuntimeState(device=0)
    node.init(pl)
    node.add_child(ColumnSource(batches_of("left", runs[0])))
    first = None
    try:
        assert node.open(st) == 0, st.error_msg
        for i, cols in enumerate(runs):
            if i:
                node.reset()
                for b in batches_of("left", cols):
                    node.push(b)
                node.finish()
            got, eos, rb = [], False, RowBatch()
            while not eos:
                rc, eos = node.get_next(st, rb)
                assert rc == 0, st.error_msg
                got = got or list(rb.columns)
            C.check(pl, cols, got=got)
            if i == 0:
                first = [c.to_list() for c in got]
            if i == 2:
                assert [c.to_list() for c in got] == first
    finally:
        node.close(st)


@pytest.mark.parametrize("regions", [2, 3])
def test_regions_merged_on_one_gpu_equal_the_single_pass(regions):
    agg, keys = C.source("merge")
    rows = inputs("merge", 13 + regions, n=9000)
    root, slots = windowed(agg, keys)
    pl = P.Plan(root, C.tuples(slots))
    single, _ = execute(pl, rows, device=0)
    n = len(rows[0])
    cuts = np.linspace(0, n, regions + 1).astype(int)
    parts = [[make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b], None if c.valid is None else c.valid[a:b]) for c in rows] for a, b in zip(cuts, cuts[1:])]
    merged = merge_regions(pl, parts, [{}] * regions)
    assert [c.to_list() for c in merged] == [c.to_list() for c in single]
    C.check(pl, rows, got=merged)


def test_repartition_is_refused():
    agg, keys = C.source("merge")
    root, slots = windowed(agg, keys, stages="one")
    with pytest.raises(BkgpuError, match="a window above an aggregate with the repartition merge is outside the GPU path"):
        execute(P.Plan(root, C.tuples(slots)), inputs("merge", 17), device=0, options={"repartition": 1})


def test_c6_star_windows_at_full_size():
    """C6's query with RANK() OVER (PARTITION BY d_year ORDER BY SUM(revenue) DESC) and SUM(SUM(revenue)) OVER (PARTITION BY d_year) at
    bench_configs.py c6's size: the groups against an independent torch computation, the windows against NumPy over the returned groups"""
    import torch
    from baikaldb_b200 import datagen
    from tests.test_gpu_star_fullsize import _gen, dev
    nf, nd, seed = 100_000_000, {"date": 2_556, "part": 1_000_000, "supplier": 100_000}, 6
    date_k = _gen(nd["date"], (1, 1, T.INT32, 4, 11, 0, nd["date"], 1.0), seed)
    part_k = (_gen(nd["part"], (2, 1, T.INT32, 4, 21, 0, nd["part"], 1.0), seed) * datagen.PART_KEY_STRIDE + datagen.PART_KEY_BASE).to(torch.int32)
    year = (1992 + date_k // 365).to(torch.int32)
    brand, cat = _gen(nd["part"], (2, 2, T.INT32, 0, 22, 0, 1000, 1.0), seed), _gen(nd["part"], (2, 3, T.INT32, 0, 23, 0, 25, 1.0), seed)
    supp_k, region = _gen(nd["supplier"], (3, 1, T.INT32, 4, 31, 0, nd["supplier"], 1.0), seed), _gen(nd["supplier"], (3, 2, T.INT32, 0, 32, 0, 5, 1.0), seed)
    fs = [(0, 1, T.INT32, 0, 1, 0, nd["date"], 1.0), (0, 2, T.INT64, 0, 2, 0, nd["part"], 1.0), (0, 3, T.INT32, 0, 3, 0, nd["supplier"], 1.0), (0, 4, T.DOUBLE, 1, 4, 0, 0, 1.0)]
    ft = [_gen(nf, s, seed) for s in fs]
    ft[1] = (ft[1] * datagen.PART_KEY_STRIDE + datagen.PART_KEY_BASE).to(torch.int32)
    batches = [[dev(1, 1, T.INT32, date_k), dev(1, 2, T.INT32, year)], [dev(2, 1, T.INT32, part_k), dev(2, 2, T.INT32, brand), dev(2, 3, T.INT32, cat)],
               [dev(3, 1, T.INT32, supp_k), dev(3, 2, T.INT32, region)], [dev(0, 1, T.INT32, ft[0]), dev(0, 2, T.INT32, ft[1]), dev(0, 3, T.INT32, ft[2]), dev(0, 4, T.DOUBLE, ft[3])]]
    got, _ = execute(queries.c6_star_window(), batches)
    by = {c.name: np.asarray(c.values) for c in got}
    assert [c.name for c in got] == ["1_2", "2_2", "4_1", "4_2", "5_2", "5_1"]   # (window outputs in stage order, bottom-up)
    yr, br, rev, cnt, rnk, ysum = by["1_2"], by["2_2"], by["4_1"], by["4_2"], by["5_1"], by["5_2"]
    # the groups: an independent torch computation over all rows (as tests/test_gpu_star_fullsize.py)
    y = torch.empty(nd["date"], dtype=torch.int64, device="cuda"); y[date_k.long()] = year.long()
    pidx = (part_k.long() - datagen.PART_KEY_BASE) // datagen.PART_KEY_STRIDE
    b = torch.empty(nd["part"], dtype=torch.int64, device="cuda"); b[pidx] = brand.long()
    c = torch.empty(nd["part"], dtype=torch.int64, device="cuda"); c[pidx] = cat.long()
    r = torch.empty(nd["supplier"], dtype=torch.int64, device="cuda"); r[supp_k.long()] = region.long()
    fidx = (ft[1].long() - datagen.PART_KEY_BASE) // datagen.PART_KEY_STRIDE
    keep = (c[fidx] == 12) & (r[ft[2].long()] == 1)
    gk = (y[ft[0].long()] * 1000 + b[fidx])[keep]
    uk, inv = torch.unique(gk, return_inverse=True)
    want_sum = torch.zeros(len(uk), dtype=torch.float64, device="cuda").index_add_(0, inv, ft[3][keep]).cpu().numpy()
    want_cnt = torch.bincount(inv, minlength=len(uk)).cpu().numpy()
    key = yr.astype(np.int64) * 1000 + br
    order = np.argsort(key)
    assert np.array_equal(key[order], uk.cpu().numpy()) and len(key) > 1000
    assert np.array_equal(cnt[order], want_cnt)
    assert np.allclose(rev[order], want_sum, rtol=1e-9, atol=0)
    # the windows over the returned groups: RANK by SUM DESC within the year (ties share a rank), the year's total
    for y0 in np.unique(yr):
        m = yr == y0
        s = rev[m]
        want_rank = np.array([1 + int(np.sum(s > v)) for v in s])
        assert np.array_equal(rnk[m], want_rank)
        assert np.allclose(ysum[m], np.sum(s), rtol=1e-12, atol=0)
    # the outer ORDER BY d_year, rnk, p_brand
    assert np.all(np.diff(yr) >= 0)
    same = np.diff(yr) == 0
    assert np.all(np.diff(rnk)[same] >= 0)
    tie = same & (np.diff(rnk) == 0)
    assert np.all(np.diff(br)[tie] > 0)

"""IN lists the constant pool cannot hold (OP_IN_SET) on the device: against the row oracle for lists it can parse (fewer than 4096
entries), and against numpy's isin with SQL's three-valued logic beyond that — every column type, NULL entries, NOT IN, IN inside OR /
CASE / a GROUP BY key / an aggregate argument, each fragment kind, several sets per plan, a plan run three times, STRING lists through
the dictionary adapter, and 1M entries over 100M device-resident rows."""
import numpy as np
import pytest

from baikaldb_b200 import _lib, plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import ColumnSource, DeviceColumn, GpuExecNode, RowBatch, RuntimeState, execute
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests import window_oracle
from tests.in_set_cases import BulkIn, sql_in
from tests.util import run_both

pytestmark = pytest.mark.gpu

ROWS = 20000
PRIMS = [T.INT32, T.INT64, T.UINT32, T.UINT64, T.DOUBLE, T.DATE, T.DATETIME, T.TIMESTAMP]
LIT = {T.INT32: P.int_lit, T.INT64: P.int_lit, T.UINT32: P.int_lit, T.UINT64: P.int_lit, T.DOUBLE: P.double_lit,
       T.DATE: P.date_lit, T.DATETIME: P.datetime_lit, T.TIMESTAMP: P.timestamp_lit}


def domain(prim, n):
    """4n distinct values of the column's storage type: a list of n of them matches about a quarter of the rows"""
    k = np.arange(4 * n)
    if prim == T.INT32: return (k - 2 * n).astype(np.int32)
    if prim == T.INT64: return (k - 2 * n) * 1_000_003
    if prim == T.UINT32: return (k + 4_000_000_000 - 4 * n).astype(np.uint32)
    if prim == T.UINT64: return np.uint64((1 << 63) - 2 * n) + k.astype(np.uint64)      # across 2^63
    if prim == T.DOUBLE: return (k - 2 * n) / 4.0
    if prim == T.DATE: return (((2024 * 13 + 1) << 5) + k).astype(np.uint32)
    if prim == T.DATETIME: return (np.uint64(2024 * 13 + 1) << np.uint64(46)) + k.astype(np.uint64) * np.uint64(1 << 24)
    return (1_700_000_000 + k).astype(np.uint32)


def table(prim, n, seed):
    rng = np.random.default_rng(seed)
    dom = domain(prim, n)
    x = dom[rng.integers(0, len(dom), ROWS)]
    if prim == T.DOUBLE:
        x[rng.random(ROWS) < 0.02] = np.nan
        x[rng.random(ROWS) < 0.02] = -0.0
        x[rng.random(ROWS) < 0.01] = np.inf
    valid = rng.random(ROWS) > 0.1
    lst = dom[rng.choice(len(dom), n, replace=False)]
    if prim == T.DOUBLE:
        lst[0] = 0.0 if rng.random() < 0.5 else -0.0   # ±0.0 on both sides
    cols = [make_column(0, 1, prim, x, valid), make_column(0, 2, T.INT64, np.arange(ROWS, dtype=np.int64))]
    return cols, x, valid, lst


def lits(prim, lst, has_null):
    out = [LIT[prim](v.item()) for v in lst]
    if has_null:
        out.insert(len(out) // 2, P.null_lit())
    return out


def tuples(prim, aggs, types):
    return {0: [(1, prim), (2, T.INT64)], 1: P.agg_tuple_slots(aggs, types)}


def rows(cols):
    return sorted(zip(*[c.to_list() for c in cols]), key=repr)


def uses_set(plan):
    return "IN_SET" in _lib.explain(plan.serialize())


@pytest.mark.parametrize("has_null", [False, True])
@pytest.mark.parametrize("n", [65, 256, 1000, 4096])
@pytest.mark.parametrize("prim", PRIMS)
def test_in_and_not_in_over_every_type(prim, n, has_null):
    cols, x, valid, lst = table(prim, n, seed=n * 31 + int(prim) * 2 + has_null)
    X, ID = P.slot_ref(0, 1, prim), P.slot_ref(0, 2, T.INT64)
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, ID)]
    # GROUP BY (x IN list): the TRUE, FALSE and NULL groups at once
    grouped = P.Plan(P.agg(P.scan(0), 1, [P.in_(X, *lits(prim, lst, has_null))], aggs), tuples(prim, aggs, [T.INT64, T.INT64]))
    # WHERE x NOT IN list
    negated = P.Plan(P.agg(P.where(P.scan(0), P.not_(P.in_(X, *lits(prim, lst, has_null)))), 1, [], aggs), tuples(prim, aggs, [T.INT64, T.INT64]))
    assert uses_set(grouped) and uses_set(negated)
    ids = np.arange(ROWS)
    hit, known = sql_in(x, valid, lst, has_null)
    want_grouped = sorted([(k, int(m.sum()), int(ids[m].sum())) for k, m in ((1, known & hit), (0, known & ~hit), (None, ~known)) if m.any()], key=repr)
    m = known & ~hit
    want_negated = [(int(m.sum()), int(ids[m].sum()))] if m.any() else []
    got_g, _ = execute(grouped, cols, device=0)
    got_n, _ = execute(negated, cols, device=0)
    assert rows(got_g) == want_grouped
    assert rows(got_n) == want_negated
    if n < 4096:   # (the row oracle parses at most 4096 children per node)
        assert rows(oracle.execute(grouped.serialize(), cols).columns) == want_grouped
        assert rows(oracle.execute(negated.serialize(), cols).columns) == want_negated


@pytest.mark.parametrize("prim", [T.INT64, T.DOUBLE, T.DATE])
def test_in_inside_or_case_and_an_aggregate_argument(prim):
    cols, x, valid, lst = table(prim, 1000, seed=int(prim))
    X, ID = P.slot_ref(0, 1, prim), P.slot_ref(0, 2, T.INT64)
    inl = lambda: P.in_(X, *lits(prim, lst, True))   # noqa: E731
    aggs = [P.agg_expr("count_star", 1, 1),
            P.agg_expr("sum", 1, 2, None, P.case_when(inl(), ID, P.int_lit(-1))),
            P.agg_expr("count", 1, 3, None, P.if_(P.not_(inl()), P.int_lit(1), P.null_lit())),
            P.agg_expr("max", 1, 4, None, P.case_when(P.is_null(inl()), ID, P.int_lit(0)))]
    plan = P.Plan(P.agg(P.where(P.scan(0), P.or_(inl(), P.lt(ID, P.int_lit(500)))), 1, [], aggs), tuples(prim, aggs, [T.INT64] * 4))
    assert uses_set(plan)
    run_both(plan, cols, None)


def test_a_64_entry_list_and_the_same_list_as_a_set_return_the_same_rows():
    cols, x, valid, lst = table(T.INT64, 64, seed=5)
    X = P.slot_ref(0, 1, T.INT64)
    scan_rows = {0: [(1, T.INT64), (2, T.INT64)]}
    short = P.Plan(P.where(P.scan(0), P.in_(X, *lits(T.INT64, lst, False))), scan_rows)
    longer = P.Plan(P.where(P.scan(0), P.in_(X, *lits(T.INT64, lst, False), P.int_lit(-(1 << 62)))), scan_rows)
    assert not uses_set(short) and uses_set(longer)
    a, _ = execute(short, cols, device=0)
    b, _ = execute(longer, cols, device=0)
    assert [c.to_list() for c in a] == [c.to_list() for c in b] and len(a[0]) > 0


# ---- one case per fragment kind, against the row oracle ----
SCAN = [(1, T.INT64), (2, T.INT32), (3, T.DOUBLE), (4, T.INT64)]
K, G, V, ID4 = (P.slot_ref(0, s, t) for s, t in SCAN)


def scan_table(n=30000, seed=3):
    rng = np.random.default_rng(seed)
    return [make_column(0, 1, T.INT64, rng.integers(0, 2000, n), rng.random(n) > 0.1), make_column(0, 2, T.INT32, rng.integers(0, 50, n).astype(np.int32)),
            make_column(0, 3, T.DOUBLE, rng.normal(size=n)), make_column(0, 4, T.INT64, np.arange(n, dtype=np.int64))]


def long_in(e, n=300, step=7, null=False):
    return P.in_(e, *[P.int_lit(i * step) for i in range(n)], *([P.null_lit()] if null else []))


def test_filter_only_rows():
    plan = P.Plan(P.where(P.scan(0), long_in(K)), {0: SCAN})
    assert uses_set(plan)
    run_both(plan, scan_table(), ["0_4"])


def test_order_by_limit_and_full_sort():
    for lim in (100, -1):
        plan = P.Plan(P.sort(P.where(P.scan(0), P.not_(long_in(K, null=False))), [V, ID4], [False, True], limit=lim, tuple_id=0), {0: SCAN})
        assert uses_set(plan)
        run_both(plan, scan_table(), None)
    # an IN set as the ORDER BY key
    plan = P.Plan(P.sort(P.scan(0), [long_in(K, null=True), ID4], [True, True], limit=500, tuple_id=0), {0: SCAN})
    run_both(plan, scan_table(), None)


def test_having_over_groups():
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, V)]
    inner = P.agg(P.where(P.scan(0), long_in(K)), 1, [K], aggs)
    having = P.where(inner, long_in(K, n=100, step=14), node_type=P.PlanNodeType.HAVING_FILTER_NODE)   # (over the group key)
    plan = P.Plan(having, {0: SCAN, 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})
    assert uses_set(plan)
    run_both(plan, scan_table(), ["0_1"], rel=1e-9)


def join_tables(seed=4):
    rng = np.random.default_rng(seed)
    nd, nf = 3000, 60000
    dim = [make_column(1, 1, T.INT32, np.arange(nd, dtype=np.int32)), make_column(1, 2, T.INT64, rng.integers(0, 1000, nd)),
           make_column(1, 3, T.INT32, rng.integers(0, 20, nd).astype(np.int32))]
    fact = [make_column(0, 1, T.INT32, rng.integers(0, nd, nf).astype(np.int32)), make_column(0, 2, T.INT64, rng.integers(0, 1000, nf), rng.random(nf) > 0.05),
            make_column(0, 3, T.INT64, np.arange(nf, dtype=np.int64))]
    return dim, fact, {0: [(1, T.INT32), (2, T.INT64), (3, T.INT64)], 1: [(1, T.INT32), (2, T.INT64), (3, T.INT32)]}


def test_inner_join_child_filter_and_residual():
    dim, fact, tup = join_tables()
    key = P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))
    residual = P.in_(P.add(P.slot_ref(0, 2, T.INT64), P.slot_ref(1, 2, T.INT64)), *[P.int_lit(i * 3) for i in range(400)])
    j = P.join(P.where(P.scan(1), long_in(P.slot_ref(1, 2, T.INT64), n=200, step=3)), P.where(P.scan(0), long_in(P.slot_ref(0, 2, T.INT64), n=400, step=2)),
               [key, residual])
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 3, T.INT64))]
    plan = P.Plan(P.agg(j, 2, [P.slot_ref(1, 3, T.INT32)], aggs), {**tup, 2: P.agg_tuple_slots(aggs, [T.INT64, T.INT64])})
    assert _lib.explain(plan.serialize()).count("in sets: 3,") == 1
    run_both(plan, dim + fact, ["1_3"], batches=[dim, fact], check_scanned=False)


def test_join_rows():
    dim, fact, tup = join_tables(5)
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    plan = P.Plan(P.sort(P.where(j, long_in(P.slot_ref(0, 2, T.INT64), n=100, step=5)), [P.slot_ref(0, 3, T.INT64)], [True], tuple_id=0), tup)
    assert uses_set(plan)
    run_both(plan, dim + fact, None, batches=[dim, fact], check_scanned=False)


def star(fact_pred, dim_pred):
    rng = np.random.default_rng(6)
    nd, ns, nf = 2000, 100, 100000
    cols = [make_column(1, 1, T.INT32, np.arange(nd, dtype=np.int32)), make_column(1, 2, T.INT32, rng.integers(0, 500, nd).astype(np.int32)),
            make_column(2, 1, T.INT32, np.arange(ns, dtype=np.int32)), make_column(2, 2, T.INT32, rng.integers(0, 5, ns).astype(np.int32)),
            make_column(0, 1, T.INT32, rng.integers(0, nd, nf).astype(np.int32)), make_column(0, 2, T.INT32, rng.integers(0, ns, nf).astype(np.int32)),
            make_column(0, 3, T.INT64, rng.integers(0, 3000, nf))]
    tup = {0: [(1, T.INT32), (2, T.INT32), (3, T.INT64)], 1: [(1, T.INT32), (2, T.INT32)], 2: [(1, T.INT32), (2, T.INT32)]}
    dim = P.where(P.scan(1), dim_pred) if dim_pred is not None else P.scan(1)
    j = P.join(dim, P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    j = P.join(P.scan(2), j, [P.eq(P.slot_ref(2, 1, T.INT32), P.slot_ref(0, 2, T.INT32))])
    aggs = [P.agg_expr("count_star", 3, 1), P.agg_expr("sum", 3, 2, None, P.slot_ref(0, 3, T.INT64))]
    root = P.agg(P.where(j, fact_pred) if fact_pred is not None else j, 3, [P.slot_ref(2, 2, T.INT32)], aggs)
    return P.Plan(root, {**tup, 3: P.agg_tuple_slots(aggs, [T.INT64, T.INT64])}), cols


def test_star_dimension_build_time_conjunct_and_fact_predicate():
    dim_pred = P.in_(P.slot_ref(1, 2, T.INT32), *[P.int_lit(i * 2) for i in range(150)])
    fact_pred = long_in(P.slot_ref(0, 3, T.INT64), n=1000, step=2)
    for fp, dp in ((None, dim_pred), (fact_pred, None), (fact_pred, dim_pred)):
        plan, cols = star(fp, dp)
        text = _lib.explain(plan.serialize())
        assert "star:" in text and f"in sets: {(fp is not None) + (dp is not None)}," in text, text
        got, _ = execute(plan, [cols[0:2], cols[2:4], cols[4:]], device=0)
        assert rows(got) == rows(oracle.execute(plan.serialize(), cols).columns)


def test_window_fragment_filter():
    cols = scan_table(20000, seed=9)
    pred = long_in(K, n=500, step=3, null=True)
    fns = [P.window_expr("row_number", 1, 1), P.window_expr("sum", 1, 2, V)]
    plan = P.Plan(P.window_stage(P.where(P.scan(0), pred), fns, [G], [ID4]), {0: SCAN})
    assert uses_set(plan)
    got, _ = execute(plan, cols, device=0)
    # the same window over the rows numpy keeps (tests/window_oracle.py does not evaluate IN)
    k = cols[0]
    keep, known = sql_in(k.values, k.valid, np.arange(500) * 3, True)
    keep &= known
    kept = [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[keep], None if c.valid is None else c.valid[keep]) for c in cols]
    window_oracle.assert_matches(got, P.Plan(P.window_stage(P.scan(0), fns, [G], [ID4]), {0: SCAN}), kept)


def test_sets_in_two_programs_of_one_plan_and_two_in_one_program():
    # WHERE k IN (...) AND v-bucket IN (...) ORDER BY (g IN (...)), id: two sets in the predicate, a third in the sort key's program
    bucket = P.cast_to_signed(P.multiplies(V, P.double_lit(10.0)))
    plan = P.Plan(P.sort(P.where(P.scan(0), long_in(K), P.in_(bucket, *[P.int_lit(i) for i in range(-5, 80)])),
                         [P.in_(G, *[P.int_lit(i) for i in range(0, 100, 2)], *[P.int_lit(1000 + i) for i in range(30)]), ID4], [True, True], tuple_id=0),
                  {0: SCAN})
    text = _lib.explain(plan.serialize())
    assert text.count("IN_SET") >= 3 and "in sets: 3," in text, text
    run_both(plan, scan_table(), None)


def test_three_requests_through_one_opened_plan():
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, V)]
    plan = P.Plan(P.agg(P.where(P.scan(0), long_in(K, n=700, null=True)), 1, [G], aggs), {0: SCAN, 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})
    tables = [scan_table(20000 + 5000 * i, seed=20 + i) for i in range(3)]
    node = GpuExecNode()
    node.init(plan)
    node.add_child(ColumnSource([tables[0]]))
    st = RuntimeState(device=0)
    assert node.open(st) == 0, st.error_msg

    def drain():
        out, eos, rb = [], False, RowBatch()
        while not eos:
            rc, eos = node.get_next(st, rb)
            assert rc == 0, st.error_msg
            out += rows(rb.columns) if rb.columns else []
        return sorted(out, key=repr)

    try:
        for i, cols in enumerate(tables):
            if i:
                node.reset()
                node.push(cols)
                node.finish()
            got = drain()
            want = rows(oracle.execute(plan.serialize(), cols).columns)
            assert [r[0] for r in got] == [r[0] for r in want] and [r[1] for r in got] == [r[1] for r in want]
            assert np.allclose([r[2] for r in got], [r[2] for r in want], rtol=1e-9)
    finally:
        node.close(st)


def test_ten_thousand_strings_through_the_dictionary_adapter():
    pa = pytest.importorskip("pyarrow")
    pc = pytest.importorskip("pyarrow.compute")
    from baikaldb_b200 import dictionary as D
    rng = np.random.default_rng(12)
    words = [f"w{i:06d}".encode() for i in range(30000)]
    s = [words[i] if ok else None for i, ok in zip(rng.integers(0, 30000, 200000), rng.random(200000) > 0.05)]
    wanted = [words[i] for i in rng.choice(30000, 10000, replace=False)] + [b"not in the column"]
    S = P.slot_ref(0, 1, T.STRING)
    aggs = [P.agg_expr("count_star", 1, 1)]
    plan = P.Plan(P.agg(P.where(P.scan(0), P.in_(S, *[P.str_lit(w.decode()) for w in wanted])), 1, [], aggs), {0: [(1, T.STRING)], 1: [(1, T.INT64)]})
    enc = D.encode_strings(plan, [D.StringColumn(0, 1, s)])
    assert uses_set(enc.plan)
    got, _ = execute(enc.plan, enc.columns, device=0)
    arr = pa.array(s, pa.binary())
    want = int(pc.sum(pc.is_in(arr, value_set=pa.array(wanted, pa.binary()))).as_py())
    assert got[0].to_list() == [want]


def test_a_million_entries_over_100m_device_rows_against_torch():
    torch = pytest.importorskip("torch")
    n, s = 100_000_000, 1_000_000
    g = torch.Generator(device="cuda").manual_seed(9)
    grp = torch.randint(0, 1000, (n,), device="cuda", dtype=torch.int32, generator=g)
    f = torch.randint(0, 4 * s, (n,), device="cuda", dtype=torch.int64, generator=g)
    x = torch.rand((n,), device="cuda", dtype=torch.float64, generator=g)
    vals = np.random.default_rng(9).choice(4 * s, s, replace=False).astype(np.int64)
    cols = [DeviceColumn(0, 1, T.INT32, grp.data_ptr(), n, keepalive=grp), DeviceColumn(0, 2, T.INT64, f.data_ptr(), n, keepalive=f),
            DeviceColumn(0, 3, T.DOUBLE, x.data_ptr(), n, keepalive=x)]
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE))]
    plan = P.Plan(P.agg(P.where(P.scan(0), BulkIn(P.slot_ref(0, 2, T.INT64), vals)), 1, [P.slot_ref(0, 1, T.INT32)], aggs),
                  {0: [(1, T.INT32), (2, T.INT64), (3, T.DOUBLE)], 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})
    got, stats = execute(plan, cols, device=0, options={"batch_capacity": 1 << 27})
    assert stats.main_kernel_name.decode() == "k_agg_interp"
    keep = torch.isin(f, torch.from_numpy(vals).cuda())
    cnt = torch.bincount(grp[keep].long(), minlength=1000)
    sm = torch.zeros(1000, dtype=torch.float64, device="cuda").index_add_(0, grp[keep].long(), x[keep])
    by = {c.name: c for c in got}
    k = np.asarray(by["0_1"].values).astype(np.int64)
    assert np.array_equal(np.asarray(by["1_1"].values), cnt.cpu().numpy()[k])
    assert np.allclose(np.asarray(by["1_2"].values), sm.cpu().numpy()[k], rtol=1e-9, atol=0)
    assert int(cnt.sum()) == int(np.asarray(by["1_1"].values).sum()) and len(k) == int((cnt > 0).sum())

"""GPU parity: hash join fused with the aggregate (K4, config C3) vs the row-engine oracle, through the C ABI."""
import numpy as np
import pytest

from baikaldb_b200 import datagen, plan as P, queries
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PrimitiveType as T
from tests.util import LEAN_KERNELS, run_both

pytestmark = pytest.mark.gpu


def test_c3_join_groupby():
    fact, dim = datagen.c3_fact(0, 400_000, 20_000), datagen.c3_dim(0, 20_000, 20_000, n_groups=100)
    got, stats, _ = run_both(queries.c3_join_groupby(), fact + dim, keys=["1_2"], batches=[dim, fact])
    assert len(got[0]) == 100
    # unique build keys: the lean aggregate kernel looks the GROUP BY attribute up through the foreign key itself
    assert stats.main_kernel_name.decode() in LEAN_KERNELS
    # ... or, with the fused probe switched off, reads build columns gathered to probe-row alignment
    _, stats, _ = run_both(queries.c3_join_groupby(), fact + dim, keys=["1_2"], batches=[dim, fact], options={"no_fused_probe": 1})
    assert stats.main_kernel_name.decode() in LEAN_KERNELS
    _, stats, _ = run_both(queries.c3_join_groupby(), fact + dim, keys=["1_2"], batches=[dim, fact], options={"force_generic": 1})
    assert stats.main_kernel_name.decode() == "k_agg_interp"


def test_join_fast_path_sparse_keys_and_unmatched_rows():
    """unique but sparse build keys (packed table instead of the dense array) and probe rows without a partner: the
    fused probe drops them (inner join); the gather path hands such chunks to the general probe; results stay identical"""
    rng = np.random.default_rng(41)
    nd, nf = 5_000, 120_000
    pk = rng.permutation(1 << 24)[:nd].astype(np.int32) * 97          # sparse: range >> 4 * n
    dim = [make_column(1, 1, T.INT32, pk), make_column(1, 2, T.INT32, rng.integers(0, 30, nd))]
    fk = pk[rng.integers(0, nd, nf)]
    fact_all = [make_column(0, 1, T.INT32, fk), make_column(0, 2, T.DOUBLE, rng.random(nf))]
    _, stats, _ = run_both(queries.c3_join_groupby(), fact_all + dim, keys=["1_2"], batches=[dim, fact_all])
    assert stats.main_kernel_name.decode() in LEAN_KERNELS
    fk2 = fk.copy(); fk2[::1000] = 5                                   # 5 is not a build key
    fact_miss = [make_column(0, 1, T.INT32, fk2), make_column(0, 2, T.DOUBLE, fact_all[1].values)]
    _, stats, _ = run_both(queries.c3_join_groupby(), fact_miss + dim, keys=["1_2"], batches=[dim, fact_miss])
    assert stats.main_kernel_name.decode() in LEAN_KERNELS
    _, stats, _ = run_both(queries.c3_join_groupby(), fact_miss + dim, keys=["1_2"], batches=[dim, fact_miss], options={"no_fused_probe": 1})
    assert stats.main_kernel_name.decode() == "k_agg_interp"


@pytest.mark.parametrize("nf", [100_003, 64_001, 2])
def test_join_fused_probe_dense_with_gaps_negative_keys_and_ragged_tail(nf):
    """dense key index with holes (present[] consulted), negative keys (bias), probe keys outside the range, a batch
    length that is not a multiple of four (tail rows probe one by one), unsigned attribute values above 2^31"""
    rng = np.random.default_rng(nf)
    nd = 3_000
    pk = (rng.permutation(4_000)[:nd] - 2_000).astype(np.int32)        # range 4000 > 3000 keys: gaps
    dim = [make_column(1, 1, T.INT32, pk), make_column(1, 2, T.INT32, rng.integers(-7, 7, nd))]
    fk = rng.integers(-2_500, 2_500, nf).astype(np.int32)              # some outside [min, max], some in gaps
    fact = [make_column(0, 1, T.INT32, fk), make_column(0, 2, T.DOUBLE, rng.random(nf))]
    _, stats, _ = run_both(queries.c3_join_groupby(), fact + dim, keys=["1_2"], batches=[dim, fact])
    if nf > 4:
        assert stats.main_kernel_name.decode() in LEAN_KERNELS


def test_c3_streamed_in_several_batches_host_and_build_first_rule():
    fact, dim = datagen.c3_fact(0, 90_000, 5_000), datagen.c3_dim(0, 5_000, 5_000, n_groups=17)
    sl = lambda cols, a, b: [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b]) for c in cols]
    batches = [sl(dim, 0, 1234), sl(dim, 1234, 5_000), sl(fact, 0, 50_000), sl(fact, 50_000, 90_000)]
    run_both(queries.c3_join_groupby(), fact + dim, keys=["1_2"], batches=batches)
    from baikaldb_b200._lib import BkgpuError, ESTATE
    from baikaldb_b200.exec_node import execute
    with pytest.raises(BkgpuError) as e:   # the driver table must be complete before probing (join_node.cpp:920-1022)
        execute(queries.c3_join_groupby(), [sl(dim, 0, 10), sl(fact, 0, 10), sl(dim, 10, 20)])
    assert e.value.code == ESTATE


def test_join_duplicate_build_keys_null_keys_and_residual_conditions():
    """multi-match probes, NULL keys on both sides never match, child filters and a residual (non-equality) join
    condition are evaluated on the joined row; mixed INT32 / INT64 keys meet in INT64 (joiner.cpp:191-200)"""
    rng = np.random.default_rng(31)
    nd, nf = 3_000, 60_000
    dim = [make_column(1, 1, T.INT64, rng.integers(0, 800, nd), rng.random(nd) > 0.05), make_column(1, 2, T.INT32, rng.integers(0, 9, nd)),
           make_column(1, 3, T.DOUBLE, rng.normal(size=nd))]
    fact = [make_column(0, 1, T.INT32, rng.integers(-50, 900, nf), rng.random(nf) > 0.05), make_column(0, 2, T.DOUBLE, rng.random(nf), rng.random(nf) > 0.1),
            make_column(0, 3, T.INT32, rng.integers(0, 100, nf))]
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.multiplies(P.slot_ref(0, 2, T.DOUBLE), P.slot_ref(1, 3, T.DOUBLE))),
            P.agg_expr("max", 2, 3, None, P.slot_ref(0, 3, T.INT32)), P.agg_expr("avg", 2, 4, 5, P.slot_ref(1, 3, T.DOUBLE))]
    outer = P.where(P.scan(1), P.ne(P.slot_ref(1, 2, T.INT32), P.int_lit(4)))
    inner = P.where(P.scan(0), P.lt(P.slot_ref(0, 3, T.INT32), P.int_lit(80)))
    j = P.join(outer, inner, [P.eq(P.slot_ref(0, 1, T.INT32), P.slot_ref(1, 1, T.INT64)),
                              P.gt(P.add(P.slot_ref(0, 3, T.INT32), P.slot_ref(1, 2, T.INT32)), P.int_lit(10))])
    root = P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs)
    pl = P.Plan(root, {0: [(1, T.INT32), (2, T.DOUBLE), (3, T.INT32)], 1: [(1, T.INT64), (2, T.INT32), (3, T.DOUBLE)],
                       2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.INT32, T.DOUBLE])})
    got, _, _ = run_both(pl, fact + dim, keys=["1_2"], batches=[dim, fact])
    assert 4 not in got[0].to_list()


def test_join_without_group_by_and_empty_sides():
    fact, dim = datagen.c3_fact(0, 10_000, 100), datagen.c3_dim(0, 100, 100, n_groups=5)
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE))]
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    pl = P.Plan(P.packet(P.agg(j, 2, [], aggs)), {0: [(1, T.INT32), (2, T.DOUBLE)], 1: [(1, T.INT32), (2, T.INT32)], 2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})
    got, _, _ = run_both(pl, fact + dim, keys=[], batches=[dim, fact])
    assert got[0].to_list() == [10_000]
    empty_dim = [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[:0]) for c in dim]
    got, _, _ = run_both(pl, fact + empty_dim, keys=[], batches=[empty_dim, fact])
    assert got[0].to_list() == [0] and got[1].to_list() == [None]


@pytest.mark.parametrize("nf", [90_001, 400_000])
def test_fused_probe_with_a_fact_side_filter(nf):
    """WHERE on the probe (fact) side below an FK -> PK join: the filter term, the key lookup and the aggregation all run in the
    lean kernel (predicate columns + fused probe + ring queue); some foreign keys have no partner"""
    rng = np.random.default_rng(nf)
    nd = 7_000
    dim = [make_column(1, 1, T.INT32, rng.permutation(9_000)[:nd].astype(np.int32)), make_column(1, 2, T.INT32, rng.integers(0, 60, nd))]
    fact = [make_column(0, 1, T.INT32, rng.integers(0, 9_000, nf)), make_column(0, 2, T.DOUBLE, rng.random(nf)), make_column(0, 3, T.INT32, rng.integers(0, 100, nf))]
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE))]
    inner = P.where(P.scan(0), P.lt(P.slot_ref(0, 3, T.INT32), P.int_lit(37)))
    j = P.join(P.scan(1), inner, [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    pl = P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs), {0: [(1, T.INT32), (2, T.DOUBLE), (3, T.INT32)], 1: [(1, T.INT32), (2, T.INT32)],
                                                                    2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})
    _, stats, _ = run_both(pl, fact + dim, keys=["1_2"], batches=[dim, fact])
    assert stats.main_kernel_name.decode() in LEAN_KERNELS
    run_both(pl, fact + dim, keys=["1_2"], batches=[dim, fact], options={"no_fused_probe": 1})


def _outer_join_tables(seed, nd=2_500, nf=40_000):
    """a dimension with duplicate and NULL keys and keys no fact row refers to; facts with NULL keys and keys without a dimension row"""
    rng = np.random.default_rng(seed)
    dim = [make_column(1, 1, T.INT32, rng.integers(0, 1_200, nd), rng.random(nd) > 0.04), make_column(1, 2, T.INT32, rng.integers(0, 12, nd)),
           make_column(1, 3, T.DOUBLE, rng.normal(size=nd))]
    fact = [make_column(0, 1, T.INT32, rng.integers(400, 1_500, nf), rng.random(nf) > 0.05), make_column(0, 2, T.DOUBLE, rng.random(nf), rng.random(nf) > 0.1),
            make_column(0, 3, T.INT32, rng.integers(0, 100, nf))]
    tuples = {0: [(1, T.INT32), (2, T.DOUBLE), (3, T.INT32)], 1: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE)]}
    return dim, fact, tuples


@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("jt", ["LEFT_JOIN", "RIGHT_JOIN"])
def test_outer_joins_keep_every_preserved_row(jt, residual):
    """LEFT (RIGHT = roles swapped, join_node.cpp:151-156): every row of the preserved table reaches the aggregate — with each partner
    that satisfies the conditions, or once NULL-extended (join_node.cpp:1200-1276, Joiner::construct_null_result_batch):
    COUNT(*) counts the NULL-extended rows, COUNT(fact col) / SUM(fact col) do not"""
    dim, fact, tuples = _outer_join_tables(7 + residual)
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("count", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE)), P.agg_expr("sum", 2, 3, None, P.slot_ref(0, 2, T.DOUBLE)),
            P.agg_expr("min", 2, 4, None, P.slot_ref(0, 3, T.INT32)), P.agg_expr("sum", 2, 5, None, P.slot_ref(1, 3, T.DOUBLE))]
    conds = [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))]
    if residual:
        conds.append(P.gt(P.add(P.slot_ref(0, 3, T.INT32), P.slot_ref(1, 2, T.INT32)), P.int_lit(40)))
    children = (P.scan(1), P.scan(0)) if jt == "LEFT_JOIN" else (P.scan(0), P.scan(1))   # the dimension is the preserved side either way
    j = P.join(children[0], children[1], conds, join_type=getattr(P.JoinType, jt))
    tuples[2] = P.agg_tuple_slots(aggs, [T.INT64, T.INT64, T.DOUBLE, T.INT32, T.DOUBLE])
    pl = P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs), tuples)
    got, _, _ = run_both(pl, fact + dim, keys=["1_2"], batches=[dim, fact])
    by = {c.name: c for c in got}
    assert sum(by["2_1"].to_list()) > sum(by["2_2"].to_list())          # NULL-extended rows exist and count only in COUNT(*)


@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("jt", ["SEMI_JOIN", "ANTI_SEMI_JOIN"])
def test_semi_and_anti_joins_emit_outer_rows_once(jt, residual):
    """SEMI: outer rows with at least one partner, each once whatever the number of partners; ANTI_SEMI: outer rows without one
    (joiner.cpp:655-685) — NULL keys never find a partner"""
    dim, fact, tuples = _outer_join_tables(11 + residual)
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(1, 3, T.DOUBLE)), P.agg_expr("max", 2, 3, None, P.slot_ref(1, 1, T.INT32))]
    conds = [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))]
    if residual:
        conds.append(P.lt(P.slot_ref(0, 3, T.INT32), P.multiplies(P.slot_ref(1, 2, T.INT32), P.int_lit(6))))
    j = P.join(P.scan(1), P.scan(0), conds, join_type=getattr(P.JoinType, jt))
    tuples[2] = P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.INT32])
    for group in ([P.slot_ref(1, 2, T.INT32)], []):
        pl = P.Plan(P.packet(P.agg(j, 2, group, aggs)), tuples)
        got, _, _ = run_both(pl, fact + dim, keys=["1_2"] if group else [], batches=[dim, fact])
    total = {c.name: c for c in got}["2_1"].to_list()[0]
    assert 0 < total < len(dim[0])


def test_outer_join_with_an_empty_probe_side_and_unsupported_shapes():
    dim, fact, tuples = _outer_join_tables(3)
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE))]
    tuples[2] = P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))], join_type=P.JoinType.LEFT_JOIN)
    pl = P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs), tuples)
    no_fact = [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[:0]) for c in fact]
    got, _, _ = run_both(pl, no_fact + dim, keys=["1_2"], batches=[dim, no_fact])     # every dimension row once, NULL-extended
    assert sum({c.name: c for c in got}["2_1"].to_list()) == len(dim[0])
    from baikaldb_b200._lib import BkgpuError, EUNSUPPORTED
    from baikaldb_b200.exec_node import execute
    filtered = P.join(P.where(P.scan(1), P.gt(P.slot_ref(1, 2, T.INT32), P.int_lit(3))), P.scan(0),
                      [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))], join_type=P.JoinType.LEFT_JOIN)
    with pytest.raises(BkgpuError) as e:   # filter-then-join is not the fused predicate's meaning for an outer join: rejected, never wrong
        execute(P.Plan(P.agg(filtered, 2, [P.slot_ref(1, 2, T.INT32)], aggs), tuples), [dim, fact])
    assert e.value.code == EUNSUPPORTED


def test_fused_build_reuses_the_learned_key_range_and_recovers_when_it_no_longer_fits():
    """prepared-statement reuse of C3's plan: the second build skips the min/max pass and trusts the first run's key range (checked by the
    build kernel); dimension keys that leave that range, and duplicate keys, must still give the oracle's rows"""
    from baikaldb_b200.exec_node import ColumnSource, GpuExecNode, RowBatch, RuntimeState
    from oracle import oracle
    from tests.util import assert_same_rows
    rng = np.random.default_rng(21)
    pl = queries.c3_join_groupby()

    def tables(lo, hi, nd, nf, dup=False):
        keys = rng.permutation(np.arange(lo, hi, dtype=np.int64))[:nd]
        if dup:
            keys[: nd // 10] = keys[nd // 10: 2 * (nd // 10)]
        dim = [make_column(1, 1, T.INT32, keys), make_column(1, 2, T.INT32, rng.integers(0, 50, nd))]
        fact = [make_column(0, 1, T.INT32, rng.integers(lo - 5, hi + 5, nf)), make_column(0, 2, T.DOUBLE, rng.random(nf))]
        return dim, fact

    runs = [tables(0, 4000, 3000, 60_000), tables(100, 3900, 3000, 60_000), tables(-7000, 9000, 5000, 60_000), tables(0, 4000, 3000, 60_000, dup=True),
            tables(1_000_000, 1_002_000, 1500, 60_000)]
    node, st = GpuExecNode(), RuntimeState(device=0)
    node.init(pl)
    node.add_child(ColumnSource([runs[0][0], runs[0][1]]))
    try:
        assert node.open(st) == 0, st.error_msg
        for i, (dim, fact) in enumerate(runs):
            if i:
                node.reset(); node.push(dim); node.push(fact); node.finish()
            got, eos, rb = [], False, RowBatch()
            while not eos:
                rc, eos = node.get_next(st, rb)
                assert rc == 0
                got = got or list(rb.columns)
            want = oracle.execute(pl.serialize(), fact + dim)
            assert_same_rows(got, want.columns, ["1_2"])
    finally:
        node.close(st)


def _row_multiset(cols):
    names = sorted(c.name for c in cols)
    by = {c.name: c.to_list() for c in cols}
    n = len(by[names[0]]) if names else 0
    key = lambda t: tuple((0, 0) if v is None else (1, v) for v in t)
    return names, sorted((tuple(by[nm][i] for nm in names) for i in range(n)), key=key)


@pytest.mark.parametrize("jt", ["INNER_JOIN", "LEFT_JOIN", "RIGHT_JOIN"])
@pytest.mark.parametrize("residual", [False, True])
def test_join_that_returns_its_rows(jt, residual):
    """[FILTER ->] JOIN at the top of the fragment (JoinNode::get_next, join_node.cpp:1200-1326): every slot of both tuples comes back, one row
    per pair that satisfies the conditions — duplicate and NULL keys on both sides, several probe batches, LEFT / RIGHT NULL-extension"""
    from baikaldb_b200.exec_node import execute
    from oracle import oracle
    dim, fact, tuples = _outer_join_tables(31 + residual, nd=1_500, nf=20_000)
    conds = [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))]
    if residual:
        conds.append(P.gt(P.add(P.slot_ref(0, 3, T.INT32), P.slot_ref(1, 2, T.INT32)), P.int_lit(55)))
    children = (P.scan(0), P.scan(1)) if jt == "RIGHT_JOIN" else (P.scan(1), P.scan(0))      # the dimension is the outer (preserved) side
    j = P.join(children[0], children[1], conds, join_type=getattr(P.JoinType, jt))
    pl = P.Plan(P.packet(j), {0: tuples[0], 1: tuples[1]})
    want = oracle.execute(pl.serialize(), fact + dim)
    half = len(fact[0]) // 2
    fact_a = [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[:half], None if c.valid is None else c.valid[:half]) for c in fact]
    fact_b = [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[half:], None if c.valid is None else c.valid[half:]) for c in fact]
    got, stats = execute(pl, [dim, fact_a, fact_b], device=0)
    gn, gr = _row_multiset(got)
    wn, wr = _row_multiset(want.columns)
    assert gn == wn and len(gr) == len(wr) > 1000
    assert gr == wr
    if jt != "INNER_JOIN":
        fk = gn.index("0_1")
        assert any(r[fk] is None and r[gn.index("0_3")] is None for r in gr)          # NULL-extended rows exist


def test_join_rows_under_filter_sort_and_limit():
    from baikaldb_b200.exec_node import execute
    from oracle import oracle
    rng = np.random.default_rng(77)
    nd, nf = 800, 30_000
    dim = [make_column(1, 1, T.INT32, np.arange(nd)), make_column(1, 2, T.INT32, rng.integers(0, 9, nd))]
    fact = [make_column(0, 1, T.INT32, rng.integers(0, nd + 50, nf)), make_column(0, 2, T.INT64, rng.permutation(nf))]   # unique sort key
    tuples = {0: [(1, T.INT32), (2, T.INT64)], 1: [(1, T.INT32), (2, T.INT32)]}
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    f = P.where(j, P.ne(P.slot_ref(1, 2, T.INT32), P.int_lit(4)), P.lt(P.mod(P.slot_ref(0, 2, T.INT64), P.int_lit(5)), P.int_lit(3)))
    pl = P.Plan(P.limit(P.sort(f, [P.slot_ref(0, 2, T.INT64)], [False], tuple_id=0), 500, offset=20), tuples)
    run_both(pl, fact + dim, keys=None, batches=[dim, fact], check_scanned=False)                      # ordered comparison, 500 rows
    got, _ = execute(P.Plan(P.limit(f, 77), tuples), [dim, fact], device=0)                           # LIMIT without an order: any 77 joined rows
    assert len(got[0]) == 77
    want = oracle.execute(P.Plan(f, tuples).serialize(), fact + dim)
    _, wr = _row_multiset(want.columns)
    _, gr = _row_multiset(got)
    assert set(gr) <= set(wr)

"""GPU parity: fused scan -> filter -> (GROUP BY) aggregate vs the row-engine oracle, through the C ABI."""
import numpy as np
import pytest

from baikaldb_b200 import datagen, plan as P, queries
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import ColumnSource, GpuExecNode, RowBatch, RuntimeState
from baikaldb_b200.plan import PrimitiveType as T
from tests.util import LEAN_KERNELS, assert_same_rows, run_both
from oracle import oracle

pytestmark = pytest.mark.gpu


def test_c1_count_where():
    cols = datagen.c1_table(0, 1_000_000)
    got, stats, want = run_both(queries.c1_count_where(), cols, keys=[])
    assert got[0].to_list() == [int((cols[0].values < (1 << 19)).sum())]
    assert stats.rows_filtered == want.rows_filtered
    assert stats.main_kernel_name.decode() == "k_count_where_tma"
    got, stats, _ = run_both(queries.c1_count_where(), cols, keys=[], options={"scalar_tma": 0})
    assert stats.main_kernel_name.decode() == "k_agg_scalar_direct" and stats.rows_filtered == want.rows_filtered


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 127, 128, 129, 1000, 2048, 2560, 2561, 65537, 300_003])
@pytest.mark.parametrize("variant", ["lean", "direct", "cas"])
def test_c2_sizes(n, variant):
    """ragged sizes around the 4-rows-per-lane / 128-rows-per-warp boundaries and one CTA's first trip (2048 rows for the general direct
    kernel's 512 threads, 2560 for the lean kernel's 640): the lean kernel (FX by default, the CAS path with lean_fx=0) and the general
    direct kernel"""
    cols = datagen.c2_table(0, n, n_groups=50)
    opts = {"lean": {}, "direct": {"no_lean": 1}, "cas": {"lean_fx": 0}}[variant]
    _, stats, _ = run_both(queries.c2_filter_groupby(), cols, keys=["0_1"], options=opts)
    assert stats.main_kernel_name.decode() in {"lean": LEAN_KERNELS, "direct": ("k_agg_group_direct",), "cas": ("k_agg_group_lean",)}[variant]


def test_lean_int64_key_and_integer_sums():
    rng = np.random.default_rng(12)
    n = 77_777
    cols = [make_column(0, 1, T.INT32, rng.integers(-100, 100, n)), make_column(0, 2, T.INT64, rng.integers(-40, 40, n) * (1 << 35)),
            make_column(0, 3, T.DOUBLE, rng.normal(size=n)), make_column(0, 4, T.INT64, rng.integers(-(1 << 62), 1 << 62, n))]
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE)),
            P.agg_expr("sum", 1, 3, None, P.slot_ref(0, 4, T.INT64)), P.agg_expr("avg", 1, 4, 5, P.slot_ref(0, 3, T.DOUBLE))]
    root = P.agg(P.where(P.scan(0), P.ge(P.slot_ref(0, 1, T.INT32), P.int_lit(-50)), P.ne(P.slot_ref(0, 1, T.INT32), P.int_lit(7))), 1,
                 [P.slot_ref(0, 2, T.INT64)], aggs)
    pl = P.Plan(root, {0: [(1, T.INT32), (2, T.INT64), (3, T.DOUBLE), (4, T.INT64)], 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.INT64, T.DOUBLE])})
    _, stats, _ = run_both(pl, cols, keys=["0_2"])
    assert stats.main_kernel_name.decode() in LEAN_KERNELS


@pytest.mark.parametrize("n", [3, 130, 70_001, 400_000])
@pytest.mark.parametrize("which", ["values", "predicate", "all", "one_value_all_null"])
def test_lean_kernel_with_null_predicate_and_value_columns(n, which):
    """C2's shape with validity bitmaps on the filter and/or value columns (the key stays NULL-free): still the lean kernel —
    a NULL filter operand drops the row, a NULL value adds +0 and skips that aggregate's non-NULL counter; SUM / AVG of a
    group whose inputs are all NULL come back NULL"""
    rng = np.random.default_rng(n)
    cols = datagen.c2_table(0, n, n_groups=40)
    mk = lambda c, valid: make_column(c.tuple_id, c.slot_id, c.prim_type, c.values, valid)
    if which in ("values", "all"):
        cols[2] = mk(cols[2], rng.random(n) > 0.3); cols[3] = mk(cols[3], rng.random(n) > 0.5)
    if which in ("predicate", "all"):
        cols[1] = mk(cols[1], rng.random(n) > 0.2)
    if which == "one_value_all_null":
        cols[3] = mk(cols[3], np.zeros(n, bool)); cols[2] = mk(cols[2], cols[0].values % 7 != 0)   # whole groups without a non-NULL input
    got, stats, _ = run_both(queries.c2_filter_groupby(), cols, keys=["0_1"])
    if n > 4:
        assert stats.main_kernel_name.decode() in LEAN_KERNELS
    _, stats, _ = run_both(queries.c2_filter_groupby(), cols, keys=["0_1"], options={"no_lean_nulls": 1})
    if n > 4:
        assert stats.main_kernel_name.decode() == "k_agg_group_direct"


@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("n", [5, 4_099, 250_000])
def test_lean_kernel_min_max_and_several_aggregates_per_column(n, nulls):
    """MIN / MAX (double, int64, uint64), SUM + MIN + MAX over one column, COUNT(x) alone: the lean kernel's MM instantiation
    (compare-then-CAS extremes), with and without NULLs; the general kernel gives the same rows"""
    rng = np.random.default_rng(n + nulls)
    valid = (lambda: rng.random(n) > 0.3) if nulls else (lambda: None)
    cols = [make_column(0, 1, T.INT32, rng.integers(0, 23, n)), make_column(0, 2, T.INT32, rng.integers(0, 100, n)),
            make_column(0, 3, T.DOUBLE, rng.normal(size=n) * 1e3, valid()), make_column(0, 4, T.INT64, rng.integers(-(1 << 40), 1 << 40, n), valid()),
            make_column(0, 5, T.UINT64, rng.integers(0, 1 << 63, n, dtype=np.uint64) * 2, valid()), make_column(0, 6, T.DOUBLE, rng.random(n), valid())]
    d, i64, u64, e = P.slot_ref(0, 3, T.DOUBLE), P.slot_ref(0, 4, T.INT64), P.slot_ref(0, 5, T.UINT64), P.slot_ref(0, 6, T.DOUBLE)
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("min", 1, 2, None, d), P.agg_expr("max", 1, 3, None, d), P.agg_expr("sum", 1, 4, None, d),
            P.agg_expr("max", 1, 5, None, i64), P.agg_expr("sum", 1, 6, None, i64), P.agg_expr("min", 1, 7, None, u64), P.agg_expr("count", 1, 8, None, e),
            P.agg_expr("avg", 1, 9, 10, d)]
    root = P.agg(P.where(P.scan(0), P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(70))), 1, [P.slot_ref(0, 1, T.INT32)], aggs)
    pl = P.Plan(root, {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE), (4, T.INT64), (5, T.UINT64), (6, T.DOUBLE)],
                       1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE, T.DOUBLE, T.INT64, T.INT64, T.UINT64, T.DOUBLE, T.DOUBLE])})
    _, stats, _ = run_both(pl, cols, keys=["0_1"])
    if n > 4:
        assert stats.main_kernel_name.decode() in LEAN_KERNELS
    _, stats, _ = run_both(pl, cols, keys=["0_1"], options={"no_lean_mm": 1})
    if n > 4:
        assert stats.main_kernel_name.decode() == "k_agg_group_direct"


@pytest.mark.parametrize("k", [0, 1, 10486, 1 << 19, 1038090, 1 << 20])
def test_c2_selectivity(k):  # 0%, ~0%, 1%, 50%, 99%, 100%
    cols = datagen.c2_table(0, 200_000)
    run_both(queries.c2_filter_groupby(k), cols, keys=["0_1"])


def test_c2_generic_kernel_matches():
    cols = datagen.c2_table(0, 100_000)
    _, stats, _ = run_both(queries.c2_filter_groupby(), cols, keys=["0_1"], options={"force_generic": 1})
    assert stats.main_kernel_name.decode() == "k_agg_interp"


@pytest.mark.parametrize("smem_log2", [0, 4, 8, 11])
def test_c2_shared_table_overflow(smem_log2):
    """1000 groups through shared tables of 1 (none) / 16 / 256 / 2048 slots: rows that do not fit go to the global table."""
    cols = datagen.c2_table(0, 150_000)
    run_both(queries.c2_filter_groupby(), cols, keys=["0_1"], options={"smem_capacity_log2": smem_log2})


def test_c2_multi_batch_host_chunks():
    cols = datagen.c2_table(0, 100_000, n_groups=300)
    batches = [[make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b]) for c in cols]
               for a, b in ((0, 1), (1, 40_001), (40_001, 40_001), (40_001, 100_000))]
    run_both(queries.c2_filter_groupby(), cols, keys=["0_1"], batches=batches, options={"chunk_rows": 8192})


def test_empty_input_no_group_by_default_row():
    cols = [make_column(0, 1, T.INT32, np.zeros(0, np.int32))]
    got, _, _ = run_both(queries.c1_count_where(), cols, keys=[])  # under a PACKET node: one row, COUNT = 0
    assert got[0].to_list() == [0]


def test_empty_input_group_by_no_rows():
    cols = datagen.c2_table(0, 0)
    got, _, _ = run_both(queries.c2_filter_groupby(), cols, keys=["0_1"])
    assert len(got[0]) == 0


def _nullable_table(n, seed=7):
    rng = np.random.default_rng(seed)
    key = rng.integers(-3, 4, n).astype(np.int32)
    f = rng.integers(0, 100, n).astype(np.int64)
    a = rng.normal(size=n)
    b = rng.integers(-1000, 1000, n).astype(np.int32)
    return [make_column(0, 1, T.INT32, key, rng.random(n) > 0.2), make_column(0, 2, T.INT64, f, rng.random(n) > 0.1),
            make_column(0, 3, T.DOUBLE, a, rng.random(n) > 0.3), make_column(0, 4, T.INT32, b, rng.random(n) > 0.5)]


def _agg_plan(group, aggs, arg_types, conj=None):
    child = P.where(P.scan(0), *conj) if conj else P.scan(0)
    root = P.agg(child, 1, group, aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.INT64), (3, T.DOUBLE), (4, T.INT32)], 1: P.agg_tuple_slots(aggs, arg_types)})


@pytest.mark.parametrize("generic", [0, 1])
def test_nulls_everywhere(generic):
    """NULL keys form a group; NULL/false predicates drop rows; aggregates skip NULL inputs; SUM/MIN/MAX/AVG of
    nothing is NULL, COUNT is 0 (SURVEY Appendix B 1,5-9)."""
    cols = _nullable_table(50_000)
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("count", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE)),
            P.agg_expr("sum", 1, 3, None, P.slot_ref(0, 3, T.DOUBLE)), P.agg_expr("avg", 1, 4, 5, P.slot_ref(0, 4, T.INT32)),
            P.agg_expr("min", 1, 6, None, P.slot_ref(0, 4, T.INT32)), P.agg_expr("max", 1, 7, None, P.slot_ref(0, 3, T.DOUBLE))]
    pl = _agg_plan([P.slot_ref(0, 1, T.INT32)], aggs, [T.INT64, T.DOUBLE, T.DOUBLE, T.INT32, T.INT32, T.DOUBLE],
                   conj=[P.lt(P.slot_ref(0, 2, T.INT64), P.int_lit(60))])
    got, _, _ = run_both(pl, cols, keys=["0_1"], options={"force_generic": generic})
    assert None in got[0].to_list()  # the NULL group


def test_all_null_aggregate_inputs():
    n = 1000
    cols = [make_column(0, 1, T.INT32, np.arange(n) % 3), make_column(0, 2, T.INT64, np.zeros(n, np.int64)),
            make_column(0, 3, T.DOUBLE, np.ones(n), np.zeros(n, bool)), make_column(0, 4, T.INT32, np.ones(n, np.int32), np.zeros(n, bool))]
    aggs = [P.agg_expr("count", 1, 1, None, P.slot_ref(0, 3, T.DOUBLE)), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE)),
            P.agg_expr("avg", 1, 3, 4, P.slot_ref(0, 4, T.INT32)), P.agg_expr("min", 1, 5, None, P.slot_ref(0, 4, T.INT32))]
    got, _, _ = run_both(_agg_plan([P.slot_ref(0, 1, T.INT32)], aggs, [T.DOUBLE, T.DOUBLE, T.INT32, T.INT32]), cols, keys=["0_1"])
    by = {c.name: c.to_list() for c in got}
    assert by["1_1"] == [0, 0, 0] and by["1_2"] == [None] * 3 and by["1_3"] == [None] * 3 and by["1_5"] == [None] * 3


def test_integer_sum_wraps_and_types():
    """SUM(int32) accumulates in INT64, SUM(uint32) in UINT64, SUM(int64) wraps (expr_value.h:854-856)."""
    n = 4096
    big = np.full(n, np.iinfo(np.int64).max // 1000, np.int64)
    cols = [make_column(0, 1, T.INT32, np.arange(n) % 5 - 2), make_column(0, 2, T.INT64, big),
            make_column(0, 3, T.UINT32, np.full(n, 0xFFFFFFF0, np.uint32)), make_column(0, 4, T.INT32, np.full(n, -(1 << 31), np.int32))]
    aggs = [P.agg_expr("sum", 1, 1, None, P.slot_ref(0, 2, T.INT64)), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.UINT32)),
            P.agg_expr("sum", 1, 3, None, P.slot_ref(0, 4, T.INT32)), P.agg_expr("max", 1, 4, None, P.slot_ref(0, 3, T.UINT32))]
    root = P.agg(P.scan(0), 1, [P.slot_ref(0, 1, T.INT32)], aggs)
    pl = P.Plan(root, {0: [(1, T.INT32), (2, T.INT64), (3, T.UINT32), (4, T.INT32)], 1: P.agg_tuple_slots(aggs, [T.INT64, T.UINT32, T.INT32, T.UINT32])})
    for generic in (0, 1):
        run_both(pl, cols, keys=["0_1"], options={"force_generic": generic})


def test_expression_predicates_and_computed_arguments():
    """OR / IN (with NULL) / NOT / IS NULL / arithmetic / division by zero -> NULL, computed SUM argument,
    computed GROUP BY key (generic interpreter kernel)."""
    cols = _nullable_table(30_000, seed=11)
    s1, s2, s3, s4 = P.slot_ref(0, 1, T.INT32), P.slot_ref(0, 2, T.INT64), P.slot_ref(0, 3, T.DOUBLE), P.slot_ref(0, 4, T.INT32)
    conj = [P.or_(P.lt(s2, P.int_lit(30)), P.in_(s4, P.int_lit(5), P.int_lit(-7), P.null_lit()), P.is_null(s3)),
            P.not_(P.eq(P.mod(s2, P.int_lit(7)), P.int_lit(0)))]
    aggs = [P.agg_expr("count_star", 1, 1),
            P.agg_expr("sum", 1, 2, None, P.multiplies(s3, s4)),
            P.agg_expr("avg", 1, 3, 4, P.divides(s2, P.minus(s4, s4))),  # x / 0 -> NULL for every row
            P.agg_expr("max", 1, 5, None, P.add(s2, s4)),
            P.agg_expr("sum", 1, 6, None, P.uminus(s4))]
    pl = _agg_plan([P.add(s1, P.int_lit(1)), P.gt(s2, P.int_lit(50))], aggs, [T.INT64, T.DOUBLE, T.DOUBLE, T.INT64, T.INT64], conj=conj)
    got, stats, _ = run_both(pl, cols, keys=["-1_0", "-1_1"])
    assert stats.main_kernel_name.decode() == "k_agg_interp"


def test_multi_key_group_by_int64_and_double_keys():
    rng = np.random.default_rng(3)
    n = 40_000
    cols = [make_column(0, 1, T.INT32, rng.integers(0, 4, n)), make_column(0, 2, T.INT64, rng.integers(-2, 2, n) * (1 << 40), rng.random(n) > 0.1),
            make_column(0, 3, T.DOUBLE, rng.integers(0, 3, n) * 0.5), make_column(0, 4, T.INT32, rng.integers(0, 100, n))]
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 4, T.INT32))]
    pl = _agg_plan([P.slot_ref(0, 2, T.INT64), P.slot_ref(0, 3, T.DOUBLE), P.slot_ref(0, 1, T.INT32)], aggs, [T.INT64, T.INT32])
    run_both(pl, cols, keys=["0_2", "0_3", "0_1"])


def test_single_int64_key_direct():
    rng = np.random.default_rng(4)
    n = 60_000
    cols = [make_column(0, 1, T.INT32, rng.integers(0, 4, n)), make_column(0, 2, T.INT64, rng.integers(-50, 50, n) * (1 << 33), rng.random(n) > 0.05),
            make_column(0, 3, T.DOUBLE, rng.random(n)), make_column(0, 4, T.INT32, rng.integers(0, 100, n))]
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE))]
    _, stats, _ = run_both(_agg_plan([P.slot_ref(0, 2, T.INT64)], aggs, [T.INT64, T.DOUBLE]), cols, keys=["0_2"])
    assert stats.main_kernel_name.decode() == "k_agg_group_direct"  # nullable key column: not the lean shape


def test_high_cardinality_global_table():
    rng = np.random.default_rng(5)
    n = 400_000
    cols = [make_column(0, 1, T.INT32, rng.integers(0, 150_000, n)), make_column(0, 2, T.INT64, rng.integers(0, 100, n)),
            make_column(0, 3, T.DOUBLE, rng.random(n)), make_column(0, 4, T.INT32, rng.integers(0, 100, n))]
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE))]
    run_both(_agg_plan([P.slot_ref(0, 1, T.INT32)], aggs, [T.INT64, T.DOUBLE]), cols, keys=["0_1"])


def test_group_table_overflow_is_an_error():
    from baikaldb_b200._lib import BkgpuError, ETOOBIG
    from baikaldb_b200.exec_node import execute
    n = 10_000
    cols = [make_column(0, 1, T.INT32, np.arange(n)), make_column(0, 2, T.INT64, np.zeros(n, np.int64)),
            make_column(0, 3, T.DOUBLE, np.zeros(n)), make_column(0, 4, T.INT32, np.zeros(n, np.int32))]
    aggs = [P.agg_expr("count_star", 1, 1)]
    with pytest.raises(BkgpuError) as ei:
        execute(_agg_plan([P.slot_ref(0, 1, T.INT32)], aggs, [T.INT64]), cols, options={"group_capacity_log2": 10})
    assert ei.value.code == ETOOBIG


def test_removed_options_are_unknown():
    """the peer-memory merge, the pageable-copy switches and output_on_device are gone: setting one is an unknown option, not a no-op"""
    import ctypes
    from baikaldb_b200 import _lib
    L = _lib.lib()
    plan = queries.c2_filter_groupby().serialize()
    h = ctypes.c_void_p()
    _lib.check(L.bkgpu_init(ctypes.byref(h), plan, len(plan), 0, None))
    try:
        for key in ("peer_merge", "no_bounce", "no_stream_copy", "output_on_device"):
            assert L.bkgpu_set_option(h, key.encode(), 1) == _lib.EINVAL, key
            assert "unknown option" in L.bkgpu_last_error(h).decode() and key in L.bkgpu_last_error(h).decode()
        assert L.bkgpu_set_option(h, b"repartition", 1) == _lib.OK
    finally:
        L.bkgpu_close(h)


@pytest.mark.parametrize("n", [1, 4095, 4096, 4097, 70_001, 1_000_003])
@pytest.mark.parametrize("op,c", [("lt", 1 << 19), ("le", 0), ("gt", (1 << 31) - 1), ("ge", -(1 << 31)), ("eq", 77), ("ne", 77)])
def test_count_where_tma_staged_kernel(n, op, c):
    """the TMA-staged variant of C1's scan (csrc/scalar_tma.cu: cp.async.bulk tiles + mbarrier ring): same counts as the oracle at sizes
    around the 4096-row tile, every comparison operator"""
    rng = np.random.default_rng(n % 1000 + len(op))
    vals = rng.integers(0, 1 << 20, n)
    vals[rng.integers(0, n, max(1, n // 50))] = 77
    cols = [make_column(0, 1, T.INT32, vals)]
    aggs = [P.agg_expr("count_star", 1, 1)]
    root = P.agg(P.where(P.scan(0), getattr(P, op)(P.slot_ref(0, 1, T.INT32), P.int_lit(c))), 1, [], aggs)
    pl = P.Plan(P.packet(root), {0: [(1, T.INT32)], 1: P.agg_tuple_slots(aggs, [T.INT64])})
    _, stats, _ = run_both(pl, cols, keys=[], options={"scalar_tma": 1})
    assert stats.main_kernel_name.decode() == "k_count_where_tma"


@pytest.mark.parametrize("variant", ["direct", "generic"])
def test_literal_wider_than_the_column_keeps_its_value(variant):
    """`int32_col < 3000000000`: the comparison runs in INT64 and the literal takes the ARGUMENT's type (Literal::cast_to_col_type,
    include/expr/literal.h:204-210 -> value_to_node_type), it is not narrowed to the column's INT32 first — every non-NULL row passes"""
    rng = np.random.default_rng(3)
    n = 50_000
    cols = [make_column(0, 1, T.INT32, rng.integers(-(1 << 31), 1 << 31, n), rng.random(n) > 0.1), make_column(0, 2, T.INT32, rng.integers(0, 9, n))]
    aggs = [P.agg_expr("count_star", 1, 1)]
    pl = P.Plan(P.agg(P.where(P.scan(0), P.lt(P.slot_ref(0, 1, T.INT32), P.int_lit(3_000_000_000))), 1, [P.slot_ref(0, 2, T.INT32)], aggs),
                {0: [(1, T.INT32), (2, T.INT32)], 1: [(1, T.INT64)]})
    got, _, _ = run_both(pl, cols, keys=["0_2"], options={"force_generic": 1} if variant == "generic" else None)
    assert sum({c.name: c for c in got}["1_1"].to_list()) == int(cols[0].valid.sum())


# ---- the lean kernel at its edges: key-table inserts and overflow, few and many groups, learned cardinality, value shapes, every
# comparison operator of the filter ----
@pytest.mark.parametrize("n_groups", [1, 2, 7, 33, 1000, 1100, 1500, 5000, 40_000])
def test_lean_cardinalities(n_groups):
    """1..40k groups: few groups = every lane of a warp updates the same slot; 5000+ = more groups than the shared table sized before any
    cardinality is known holds (the rest take the global path); the result never depends on which path a row took"""
    cols = datagen.c2_table(0, 300_000, n_groups=n_groups)
    _, stats, _ = run_both(queries.c2_filter_groupby(), cols, keys=["0_1"])
    assert stats.main_kernel_name.decode() in LEAN_KERNELS


@pytest.mark.parametrize("n_groups", [50, 1000, 3000])
def test_lean_second_run_uses_learned_cardinality(n_groups):
    """prepared-statement reuse: the second run sizes the shared table from the first run's group count; same rows every time"""
    cols = datagen.c2_table(0, 200_000, n_groups=n_groups)
    pl = queries.c2_filter_groupby()
    want = oracle.execute(pl.serialize(), cols)
    node, st = GpuExecNode(), RuntimeState(device=0, options={})
    node.init(pl)
    node.add_child(ColumnSource([cols]))
    try:
        assert node.open(st) == 0, st.error_msg
        for run in range(3):
            if run:
                node.reset()
                node.push(cols)
                node.finish()
            got, eos, rb = [], False, RowBatch()
            while not eos:
                rc, eos = node.get_next(st, rb)
                assert rc == 0
                got = got or list(rb.columns)
            assert_same_rows(got, want.columns, ["0_1"])
            # (3000 groups do not fit the lean kernel's shared table: once the cardinality is known the general direct kernel takes over)
            name = node.stats().main_kernel_name.decode()
            assert name in LEAN_KERNELS if (n_groups <= 1000 or run == 0) else name in LEAN_KERNELS + ("k_agg_group_direct",)
    finally:
        node.close(st)


def test_lean_sparse_and_negative_keys():
    rng = np.random.default_rng(5)
    n = 150_000
    keys = rng.choice(np.array([-(1 << 31), -1, 0, 1, (1 << 31) - 1, 123456789, -987654321] + list(rng.integers(-(1 << 31), 1 << 31, 500))), n)
    cols = [make_column(0, 1, T.INT32, keys), make_column(0, 2, T.INT32, rng.integers(0, 1 << 20, n)),
            make_column(0, 3, T.DOUBLE, rng.random(n)), make_column(0, 4, T.DOUBLE, rng.normal(size=n) * 1e3)]
    _, stats, _ = run_both(queries.c2_filter_groupby(), cols, keys=["0_1"])
    assert stats.main_kernel_name.decode() in LEAN_KERNELS


def test_lean_uint32_key_with_all_ones():
    rng = np.random.default_rng(6)
    n = 90_000
    keys = rng.choice(np.array([0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFFF0, 0, 1, 0x80000000], dtype=np.uint32), n)
    cols = [make_column(0, 1, T.UINT32, keys), make_column(0, 2, T.DOUBLE, rng.random(n))]
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 2, T.DOUBLE))]
    pl = P.Plan(P.agg(P.scan(0), 1, [P.slot_ref(0, 1, T.UINT32)], aggs), {0: [(1, T.UINT32), (2, T.DOUBLE)], 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})
    _, stats, _ = run_both(pl, cols, keys=["0_1"])
    assert stats.main_kernel_name.decode() in LEAN_KERNELS


@pytest.mark.parametrize("shape", ["count_only", "one_double", "one_int64", "int64_and_double", "two_int64"])
def test_lean_value_shapes(shape):
    rng = np.random.default_rng(len(shape))
    n = 120_001
    cols = [make_column(0, 1, T.INT32, rng.integers(0, 300, n)), make_column(0, 2, T.INT32, rng.integers(0, 100, n)),
            make_column(0, 3, T.DOUBLE, rng.normal(size=n)), make_column(0, 4, T.INT64, rng.integers(-(1 << 61), 1 << 61, n)),
            make_column(0, 5, T.INT64, rng.integers(-5, 5, n))]
    d, i1, i2 = P.slot_ref(0, 3, T.DOUBLE), P.slot_ref(0, 4, T.INT64), P.slot_ref(0, 5, T.INT64)
    aggs = {"count_only": [P.agg_expr("count_star", 1, 1)],
            "one_double": [P.agg_expr("count_star", 1, 1), P.agg_expr("avg", 1, 2, 3, d)],
            "one_int64": [P.agg_expr("sum", 1, 1, None, i1)],
            "int64_and_double": [P.agg_expr("sum", 1, 1, None, i1), P.agg_expr("sum", 1, 2, None, d), P.agg_expr("count_star", 1, 3)],
            "two_int64": [P.agg_expr("sum", 1, 1, None, i1), P.agg_expr("sum", 1, 2, None, i2)]}[shape]
    types = {"count_only": [T.INT64], "one_double": [T.INT64, T.DOUBLE], "one_int64": [T.INT64], "int64_and_double": [T.INT64, T.DOUBLE, T.INT64],
             "two_int64": [T.INT64, T.INT64]}[shape]
    root = P.agg(P.where(P.scan(0), P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(60))), 1, [P.slot_ref(0, 1, T.INT32)], aggs)
    pl = P.Plan(root, {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE), (4, T.INT64), (5, T.INT64)], 1: P.agg_tuple_slots(aggs, types)})
    _, stats, _ = run_both(pl, cols, keys=["0_1"])
    assert stats.main_kernel_name.decode() in LEAN_KERNELS


@pytest.mark.parametrize("op", ["eq", "ne", "lt", "le", "gt", "ge"])
@pytest.mark.parametrize("c", [-(1 << 31), -7, 0, 41, (1 << 31) - 1])
def test_lean_filter_operators(op, c):
    """every comparison of `int32 column <cmp> constant` at the int32 limits"""
    rng = np.random.default_rng(abs(c) % 1000 + len(op))
    n = 50_000
    f = rng.choice(np.array([-(1 << 31), -(1 << 31) + 1, -8, -7, -6, -1, 0, 1, 40, 41, 42, (1 << 31) - 2, (1 << 31) - 1]), n)
    cols = [make_column(0, 1, T.INT32, rng.integers(0, 64, n)), make_column(0, 2, T.INT32, f), make_column(0, 3, T.DOUBLE, rng.random(n))]
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE))]
    pred = getattr(P, op)(P.slot_ref(0, 2, T.INT32), P.int_lit(c))
    root = P.agg(P.where(P.scan(0), pred, P.ge(P.slot_ref(0, 1, T.INT32), P.int_lit(3))), 1, [P.slot_ref(0, 1, T.INT32)], aggs)
    pl = P.Plan(root, {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE)], 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})
    _, stats, _ = run_both(pl, cols, keys=["0_1"])
    assert stats.main_kernel_name.decode() in LEAN_KERNELS

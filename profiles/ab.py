#!/usr/bin/env python
"""ab.py — A/B of two builds of libbkgpu.so over the aggregate, hash-join, ORDER BY / filter, window and rb_build_agg plans: each build runs the same seeded plans in its own
process (BKGPU_LIB is read when the library is loaded), and the two dumps are compared.

    BKGPU_LIB=/path/a/libbkgpu.so python profiles/ab.py run a.json
    BKGPU_LIB=/path/b/libbkgpu.so python profiles/ab.py run b.json
    python profiles/ab.py compare a.json b.json

Per run the dump keeps the counters kernel_launches, main_kernel_name, main_kernel_launches, main_kernel_bytes, h2d_bytes and d2h_bytes, and
the result columns.  The comparison wants the same counters, the same group keys, integers and bitmap bytes, bit-identical doubles for the
tables of tests/join_key_cases.py (their sums are integer-valued) and 1e-9 relative for other double sums (adds through global atomics are not ordered).  That includes the lean
kernel's FX variant: its fixed-point limbs are exact within a CTA, but the CTAs flush their sums into the global table as double atomics,
so two runs of the same build differ in the last bits."""
import json
import math
import os
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np

from baikaldb_b200 import datagen, plan as P, queries
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PlanNodeType, PrimitiveType as T

CASES = {}


def case(keys, exact=False, ordered=False):
    """keys: the group key columns (None: compare rows, in order when `ordered`, else as a multiset)"""
    def reg(fn):
        CASES[fn.__name__] = (fn, keys, exact, ordered)
        return fn
    return reg


def having(child, *conj):
    return P.where(child, *conj, node_type=PlanNodeType.HAVING_FILTER_NODE)


# ---- each case: (plan, [runs: list of batches], options); runs after the first go through bkgpu_reset of the same plan ----
@case(["1_2"])
def c3():
    fact, dim = datagen.c3_fact(0, 4_000_000, 400_000), datagen.c3_dim(0, 400_000, 400_000, n_groups=1000)
    return queries.c3_join_groupby(), [[dim, fact], [dim, fact]], {}


@case(["1_2"])
def c3_gather_path():
    fact, dim = datagen.c3_fact(0, 4_000_000, 400_000), datagen.c3_dim(0, 400_000, 400_000, n_groups=1000)
    return queries.c3_join_groupby(), [[dim, fact], [dim, fact]], {"no_fused_probe": 1}


@case(["1_2", "2_2"])
def c6_small():
    fact, date, part, supp = datagen.c6_tables(2_000_000, 2_556, 200_000, 20_000)
    return queries.c6_star_groupby(), [[date, part, supp, fact], [date, part, supp, fact]], {}


def outer_tables(seed, nd=2_500, nf=40_000):
    rng = np.random.default_rng(seed)
    dim = [make_column(1, 1, T.INT32, rng.integers(0, 1_200, nd), rng.random(nd) > 0.04), make_column(1, 2, T.INT32, rng.integers(0, 12, nd)),
           make_column(1, 3, T.DOUBLE, rng.normal(size=nd))]
    fact = [make_column(0, 1, T.INT32, rng.integers(400, 1_500, nf), rng.random(nf) > 0.05), make_column(0, 2, T.DOUBLE, rng.random(nf), rng.random(nf) > 0.1),
            make_column(0, 3, T.INT32, rng.integers(0, 100, nf))]
    return dim, fact, {0: [(1, T.INT32), (2, T.DOUBLE), (3, T.INT32)], 1: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE)]}


def left_conds():
    return [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32)), P.gt(P.add(P.slot_ref(0, 3, T.INT32), P.slot_ref(1, 2, T.INT32)), P.int_lit(40))]


@case(["1_2"])
def left_join_residual():
    dim, fact, tup = outer_tables(7, nd=250_000, nf=2_000_000)
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("count", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE)), P.agg_expr("sum", 2, 3, None, P.slot_ref(0, 2, T.DOUBLE)),
            P.agg_expr("min", 2, 4, None, P.slot_ref(0, 3, T.INT32)), P.agg_expr("sum", 2, 5, None, P.slot_ref(1, 3, T.DOUBLE))]
    tup[2] = P.agg_tuple_slots(aggs, [T.INT64, T.INT64, T.DOUBLE, T.INT32, T.DOUBLE])
    j = P.join(P.scan(1), P.scan(0), left_conds(), join_type=P.JoinType.LEFT_JOIN)
    return P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs), tup), [[dim, fact], [dim, fact]], {}


@case(["1_2"])
def full_join_agg_nulls_both_sides():   # rows of both sides without a partner: every gathered column of the chunk holds NULLs
    dim, fact, tup = outer_tables(11, nd=200_000, nf=1_500_000)
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("count", 2, 2, None, P.slot_ref(0, 3, T.INT32)), P.agg_expr("sum", 2, 3, None, P.slot_ref(0, 2, T.DOUBLE)),
            P.agg_expr("sum", 2, 4, None, P.slot_ref(1, 3, T.DOUBLE))]
    tup[2] = P.agg_tuple_slots(aggs, [T.INT64, T.INT64, T.DOUBLE, T.DOUBLE])
    j = P.join(P.scan(1), P.scan(0), left_conds()[:1], join_type=P.JoinType.FULL_JOIN)
    return P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs), tup), [[dim, fact], [dim, fact]], {}


def device_columns(cols):
    """CUDA tensors of the columns (values, and the validity bitmap with 8 bytes of slack)"""
    import torch
    from baikaldb_b200.exec_node import DeviceColumn
    out = []
    for c in cols:
        t = torch.from_numpy(np.ascontiguousarray(c.values).copy()).cuda()
        bm = c.validity_bitmap()
        b = torch.from_numpy(np.concatenate([bm, np.zeros(8, np.uint8)])).cuda() if bm is not None else None
        out.append(DeviceColumn(c.tuple_id, c.slot_id, c.prim_type, t.data_ptr(), len(c), b.data_ptr() if b is not None else 0, (t, b)))
    return out


@case(["1_2"])
def join_device_build_side_in_two_batches():   # the retained build side grows past its first 65,536 rows while keeping them
    dim, fact, tup = outer_tables(13, nd=150_000, nf=1_000_000)
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE)), P.agg_expr("sum", 2, 3, None, P.slot_ref(1, 3, T.DOUBLE))]
    tup[2] = P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE])
    j = P.join(P.scan(1), P.scan(0), left_conds()[:1])
    halves = chunks(dim, [0, 50_000, 150_000])
    return P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs), tup), [[device_columns(h) for h in halves] + [fact]] * 2, {}


@case(None)
def left_join_rows():
    dim, fact, tup = outer_tables(31, nd=1_500, nf=20_000)
    half = len(fact[0]) // 2
    sl = lambda a, b: [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b], None if c.valid is None else c.valid[a:b]) for c in fact]
    j = P.join(P.scan(1), P.scan(0), left_conds(), join_type=P.JoinType.LEFT_JOIN)
    return P.Plan(P.packet(j), tup), [[dim, sl(0, half), sl(half, len(fact[0]))]], {}


@case(None, ordered=True)
def join_rows_sort_limit():
    rng = np.random.default_rng(77)
    nd, nf = 80_000, 3_000_000
    dim = [make_column(1, 1, T.INT32, np.arange(nd)), make_column(1, 2, T.INT32, rng.integers(0, 9, nd))]
    fact = [make_column(0, 1, T.INT32, rng.integers(0, nd + 5_000, nf)), make_column(0, 2, T.INT64, rng.permutation(nf))]   # unique sort key
    tup = {0: [(1, T.INT32), (2, T.INT64)], 1: [(1, T.INT32), (2, T.INT32)]}
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    f = P.where(j, P.ne(P.slot_ref(1, 2, T.INT32), P.int_lit(4)), P.lt(P.mod(P.slot_ref(0, 2, T.INT64), P.int_lit(5)), P.int_lit(3)))
    return P.Plan(P.limit(P.sort(f, [P.slot_ref(0, 2, T.INT64)], [False], tuple_id=0), 5_000, offset=20), tup), [[dim, fact], [dim, fact]], {}


def key_cases():
    from tests import join_key_cases as K
    return K


@case(["0_3", "1_3"], exact=True)
def exact_two_table_gather():
    K = key_cases()
    rng = np.random.default_rng(5)
    d = K.make_dim(rng, 1, T.INT32, T.INT64, 300_000)
    c = K.make_case(rng, [d], 2_000_000, miss=0.0, null=0.0)
    return K.agg_plan([d]), [c.batches(), c.batches()], {}


@case(["0_3", "1_3"], exact=True)
def exact_two_table_misses():
    K = key_cases()
    rng = np.random.default_rng(6)
    d = K.make_dim(rng, 1, T.INT64, T.INT32, 300_000)
    c = K.make_case(rng, [d], 2_000_000)
    return K.agg_plan([d]), [c.batches()], {}


@case(["0_3", "1_3"], exact=True)
def exact_star_duplicate_keys():
    K = key_cases()
    rng = np.random.default_rng(8)
    d1 = K.make_dim(rng, 1, T.INT32, T.INT32, 20_000, null_keys=0.02)
    keys = [int(k) for k in rng.integers(-3_000, 3_000, 9_000)]
    d2 = K.make_dim(rng, 2, T.INT64, T.INT32, 0, keys=keys)
    d3 = K.make_dim(rng, 3, T.UINT32, T.UINT32, 5_000)
    c = K.make_case(rng, [d1, d2, d3], 1_000_000)
    return K.agg_plan([d1, d2, d3]), [c.batches(), c.batches()], {"star_expand_capacity": 4096}


@case(["1_2", "2_2", "0_2"])
def star_duplicate_keys_doubles():
    from tests.test_gpu_star import plan, star, tables
    fact, dims, tup = tables(9, 3, dup=2, nf=2_000_000, nulls=True)
    return plan(star(3), tup), [dims + [fact], dims + [fact]], {}


@case(None, ordered=True)
def having_sort_limit_over_join():
    nd, nf = 50_000, 2_000_000
    fact, dim = datagen.c3_fact(0, nf, nd), datagen.c3_dim(0, nd, nd, n_groups=3_000)
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE))]
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    a = P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs)
    h = having(a, P.gt(P.slot_ref(2, 1, T.INT64), P.int_lit(600)))
    # ordered by the group key: unique, so the order does not hang on the last bits of a sum
    pl = P.Plan(P.limit(P.sort(h, [P.slot_ref(1, 2, T.INT32)], [False], tuple_id=2), 300),
                {0: [(1, T.INT32), (2, T.DOUBLE)], 1: [(1, T.INT32), (2, T.INT32)], 2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])})
    return pl, [[dim, fact], [dim, fact]], {}


@case(["0_1"])
def having_over_aggregate():
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE)), P.agg_expr("avg", 1, 3, 4, P.slot_ref(0, 4, T.DOUBLE))]
    tup = {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE), (4, T.DOUBLE)], 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE])}
    a = P.agg(P.where(P.scan(0), P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(1 << 19))), 1, [P.slot_ref(0, 1, T.INT32)], aggs)
    pl = P.Plan(having(a, P.gt(P.slot_ref(1, 1, T.INT64), P.int_lit(333))), tup)   # (about half of the groups)
    cols = datagen.c2_table(0, 2_000_000, n_groups=3_000)
    return pl, [[cols], [cols]], {}


# ---- aggregates without a join: the kernel choices of csrc/agg_select.cpp ----
@case([])
def c1_tma():
    return queries.c1_count_where(), [[datagen.c1_table(0, 8_000_000)]] * 2, {}


@case([])
def c1_ldg():
    return queries.c1_count_where(), [[datagen.c1_table(0, 8_000_000)]] * 2, {"scalar_tma": 0}


def c2(options, n_groups=1_000):
    return queries.c2_filter_groupby(), [[datagen.c2_table(0, 4_000_000, n_groups=n_groups)]] * 2, options


@case(["0_1"])
def c2_fx():
    return c2({})


@case(["0_1"])
def c2_cas():
    return c2({"lean_fx": 0})


@case(["0_1"])
def c2_no_lean():
    return c2({"no_lean": 1})


@case(["0_1"])
def c2_generic():
    return c2({"force_generic": 1})


@case(["0_1"])
def c2_nulls():
    rng = np.random.default_rng(3)
    n = 4_000_000
    cols = datagen.c2_table(0, n, n_groups=1_000)
    mk = lambda c, valid: make_column(c.tuple_id, c.slot_id, c.prim_type, c.values, valid)
    cols[1], cols[2], cols[3] = mk(cols[1], rng.random(n) > 0.2), mk(cols[2], rng.random(n) > 0.3), mk(cols[3], rng.random(n) > 0.5)
    return queries.c2_filter_groupby(), [[cols]] * 2, {}


@case(["0_1"])
def min_max():
    from tests.test_agg_select import min_max_plan
    rng = np.random.default_rng(4)
    n = 4_000_000
    cols = [make_column(0, 1, T.INT32, rng.integers(0, 23, n)), make_column(0, 2, T.INT32, rng.integers(0, 100, n)),
            make_column(0, 3, T.DOUBLE, rng.normal(size=n) * 1e3), make_column(0, 4, T.INT64, rng.integers(-(1 << 40), 1 << 40, n)),
            make_column(0, 5, T.UINT64, rng.integers(0, 1 << 63, n, dtype=np.uint64) * 2), make_column(0, 6, T.DOUBLE, rng.random(n))]
    return min_max_plan(), [[cols]] * 2, {}


@case(["0_2"])
def int64_key():
    from tests.test_agg_select import int64_key_plan
    rng = np.random.default_rng(5)
    n = 4_000_000
    cols = [make_column(0, 1, T.INT32, rng.integers(-100, 100, n)), make_column(0, 2, T.INT64, rng.integers(-40, 40, n) * (1 << 35)),
            make_column(0, 3, T.DOUBLE, rng.normal(size=n)), make_column(0, 4, T.INT64, rng.integers(-(1 << 62), 1 << 62, n))]
    return int64_key_plan(), [[cols]] * 2, {}


@case(["0_1"])
def c2_smem_log2_0():   # 1,000 groups through the shared-table capacities of tests/test_gpu_agg.py::test_c2_shared_table_overflow
    return c2({"smem_capacity_log2": 0})


@case(["0_1"])
def c2_smem_log2_4():   # 1,000 groups through the shared-table capacities of tests/test_gpu_agg.py::test_c2_shared_table_overflow
    return c2({"smem_capacity_log2": 4})


@case(["0_1"])
def c2_smem_log2_8():   # 1,000 groups through the shared-table capacities of tests/test_gpu_agg.py::test_c2_shared_table_overflow
    return c2({"smem_capacity_log2": 8})


@case(["0_1"])
def c2_smem_log2_11():   # 1,000 groups through the shared-table capacities of tests/test_gpu_agg.py::test_c2_shared_table_overflow
    return c2({"smem_capacity_log2": 11})


@case(["0_1"])
def c2_groups_past_the_fused_buffer():   # 200,000 groups: more than the fused extraction holds, so k_extract reads them back (the first run regrows its buffers)
    return c2({}, n_groups=200_000)


@case(["0_1"])
def hll_grouped():   # hll_add_agg per group: the arena's counters and blocks come back after the extraction
    from tests import hll_cases
    rng = np.random.default_rng(21)
    n = 1_000_000
    cols = [make_column(0, 1, T.INT32, rng.integers(0, 300, n).astype(np.int32)), make_column(0, 2, T.INT64, rng.integers(0, 50_000, n), rng.random(n) > 0.1),
            make_column(0, 3, T.DOUBLE, rng.normal(size=n))]
    return hll_cases.scan_plan(T.INT64, extra=True), [chunks(cols, [0, 400_000, n])] * 2, {}


@case([])
def scalar_sum():
    from tests.test_agg_select import scalar_sum_plan
    return scalar_sum_plan(), [[datagen.c2_table(0, 4_000_000)]] * 2, {}


# ---- ORDER BY / top-k / filter-only, the window stage, rb_build_agg: sort.cu, window.cu, rb.cu ----
def chunks(cols, cuts):
    return [[make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b], None if c.valid is None else c.valid[a:b]) for c in cols]
            for a, b in zip(cuts, cuts[1:])]


@case(None, ordered=True)
def filter_limit_offset_host_chunks():
    rng = np.random.default_rng(19)
    n = 600_000
    cols = [make_column(0, 1, T.INT64, rng.integers(0, 100, n)), make_column(0, 2, T.INT32, np.arange(n, dtype=np.int32), rng.random(n) > 0.2)]
    conj = P.and_(P.gt(P.slot_ref(0, 1, T.INT64), P.int_lit(90)), P.not_(P.is_null(P.slot_ref(0, 2, T.INT32))))
    pl = P.Plan(P.limit(P.where(P.scan(0), conj), 30_000, 17), {0: [(1, T.INT64), (2, T.INT32)]})
    batches = chunks(cols, [0, 250_000, 250_001, 600_000])
    return pl, [batches, batches], {"chunk_rows": 40_000}   # host columns cross the staging buffers in 40k-row chunks


@case(None, ordered=True)
def full_sort_two_keys_nulls():
    rng = np.random.default_rng(17)
    n = 700_000
    cols = [make_column(0, 1, T.INT64, rng.integers(0, 50, n), rng.random(n) > 0.05), make_column(0, 2, T.INT32, rng.integers(-5, 5, n), rng.random(n) > 0.1),
            make_column(0, 3, T.DOUBLE, rng.normal(size=n))]
    pl = P.Plan(P.sort(P.scan(0), [P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 2, T.INT32)], [True, False], [False, True], tuple_id=0),
                {0: [(1, T.INT64), (2, T.INT32), (3, T.DOUBLE)]})
    return pl, [chunks(cols, [0, 300_000, n])] * 2, {}


@case(None, ordered=True)
def topk_null_keys():
    rng = np.random.default_rng(5)
    n = 2_000_000
    cols = [make_column(0, 1, T.INT64, rng.integers(-1000, 1000, n), rng.random(n) > 0.01), make_column(0, 2, T.INT32, np.arange(n, dtype=np.int32))]
    pl = P.Plan(P.sort(P.scan(0), [P.slot_ref(0, 1, T.INT64)], [True], [True], limit=700, tuple_id=0), {0: [(1, T.INT64), (2, T.INT32)]})
    return pl, [[cols], chunks(cols, [0, 1_000_000, n])], {}


@case(None, ordered=True)
def window_stack_then_order_by():
    from tests.test_gpu_window import FRAMES, SCAN, K, V, X, U, table
    cols = table(19, 300_000, n_keys=250)
    s0 = P.window_stage(P.scan(0), [P.window_expr("row_number", 1, 1), P.window_expr("lag", 1, 2, X)], [K], [V])
    s1 = P.window_stage(s0, [P.window_expr("rank", 1, 3)], [U], [X], [False])
    s2 = P.window_stage(s1, [P.window_expr("sum", 1, 4, X), P.window_expr("count", 1, 5, X)], [U], [X], [False], window_frame=FRAMES["rows_bounded"])
    out = [(1, T.INT64), (2, T.DOUBLE), (3, T.INT64), (4, T.DOUBLE), (5, T.INT64)]
    pl = P.Plan(P.limit(P.sort(s2, [P.slot_ref(1, 1, T.INT64), P.slot_ref(1, 4, T.DOUBLE)], [False, True], tuple_id=2), 50_000, 100), {0: SCAN, 1: out})
    return pl, [[cols], [cols]], {}


@case(None, ordered=True)
def window_limit_offset():   # no query ORDER BY: the window rows leave through the stage's permutation after LIMIT / OFFSET
    from tests.test_gpu_window import SCAN, K, V, X, table
    st = P.window_stage(P.scan(0), [P.window_expr("row_number", 1, 1), P.window_expr("sum", 1, 2, X)], [K], [V])
    pl = P.Plan(P.limit(st, 40_000, 1_234), {0: SCAN, 1: [(1, T.INT64), (2, T.DOUBLE)]})
    cols = table(29, 300_000, n_keys=250)
    return pl, [[cols], [cols]], {}


@case(None, ordered=True)
def order_by_over_group_by():   # no LIMIT: the post fragment radix-sorts every group
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE))]
    tup = {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE), (4, T.DOUBLE)], 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE])}
    a = P.agg(P.scan(0), 1, [P.slot_ref(0, 1, T.INT32)], aggs)
    pl = P.Plan(P.sort(a, [P.slot_ref(0, 1, T.INT32)], [False], tuple_id=1), tup)   # (the group key: unique, so the order is fixed)
    cols = datagen.c2_table(0, 2_000_000, n_groups=50_000)
    return pl, [[cols], [cols]], {}


@case(["0_1"])
def rb_compaction():
    from tests import rb_cases
    rng = np.random.default_rng(12)
    n, g = 300_000, 10
    cols = [make_column(0, 1, T.INT32, rng.integers(0, g, n).astype(np.int32)), make_column(0, 2, T.INT64, rng.integers(0, 150, n)),
            make_column(0, 3, T.DOUBLE, rng.integers(0, 1000, n).astype(np.float64))]
    return rb_cases.scan_plan(T.INT64, extra=True), [chunks(cols, list(range(0, n, 70_000)) + [n])] * 2, {"rb_pair_capacity": 4096}


# ---- run ----
def execute_runs(pl, runs, options):
    from baikaldb_b200._lib import BkgpuError
    from baikaldb_b200.exec_node import ColumnSource, GpuExecNode, RowBatch, RuntimeState
    node, st = GpuExecNode(), RuntimeState(device=0, options=dict(options))
    node.init(pl)
    node.add_child(ColumnSource(runs[0]))
    out = []
    try:
        if node.open(st) < 0:
            raise BkgpuError(st.error_code, st.error_msg)
        for i, batches in enumerate(runs):
            if i:
                node.reset()
                for b in batches:
                    node.push(b)
                node.finish()
            cols, eos, rb = {}, False, RowBatch()
            while not eos:
                rc, eos = node.get_next(st, rb)
                if rc < 0:
                    raise BkgpuError(rc, st.error_msg)
                for c in rb.columns:   # (a BITMAP or an HLL sketch arrives as its serialized bytes, an AVG intermediate {double sum; int64 count} as 16 bytes)
                    unpack = (lambda v: v.hex()) if c.prim_type in (T.BITMAP, T.HLL) else (lambda v: list(struct.unpack("<dq", v)))
                    cols.setdefault(c.name, []).extend([unpack(v) if isinstance(v, bytes) else v for v in c.to_list()])
            s = node.stats()
            out.append({"kernel_launches": s.kernel_launches, "main_kernel_name": s.main_kernel_name.decode(), "main_kernel_launches": s.main_kernel_launches,
                        "main_kernel_bytes": s.main_kernel_bytes, "h2d_bytes": s.h2d_bytes, "d2h_bytes": s.d2h_bytes, "columns": cols})
    finally:
        node.close(st)
    return out


def run(path):
    import torch
    from baikaldb_b200 import _lib
    dump = {"version": _lib.lib().bkgpu_version().decode(), "gpu": torch.cuda.get_device_name(0), "cases": {}}
    for name, (fn, _, _, _) in CASES.items():
        pl, runs, options = fn()
        dump["cases"][name] = execute_runs(pl, runs, options)
        print(name, [(r["kernel_launches"], r["main_kernel_name"]) for r in dump["cases"][name]], flush=True)
    json.dump(dump, open(path, "w"))


def same_value(a, b, exact):
    if isinstance(a, list) and isinstance(b, list):
        return len(a) == len(b) and all(same_value(x, y, exact) for x, y in zip(a, b))
    if a is None or b is None or not isinstance(a, float):
        return a == b
    if exact or a == b:
        return a == b
    return math.isclose(a, b, rel_tol=1e-9, abs_tol=0.0)


COUNTERS = ("kernel_launches", "main_kernel_name", "main_kernel_launches", "main_kernel_bytes", "h2d_bytes", "d2h_bytes")


def compare(path_a, path_b):
    A, B = json.load(open(path_a)), json.load(open(path_b))
    print("A:", A["version"], "\nB:", B["version"], "\nGPU:", A["gpu"], "/", B["gpu"])
    bad = 0
    for name, (_, keys, exact, ordered) in CASES.items():
        for i, (ra, rb) in enumerate(zip(A["cases"][name], B["cases"][name])):
            problems = [f"{k} {ra[k]} != {rb[k]}" for k in COUNTERS if ra[k] != rb[k]]
            ca, cb = ra["columns"], rb["columns"]
            names = sorted(ca)
            if names != sorted(cb):
                problems.append(f"columns {names} != {sorted(cb)}")
            else:
                rows_a = list(zip(*(ca[n] for n in names)))
                rows_b = list(zip(*(cb[n] for n in names)))
                if keys is not None:   # by group key
                    kix = [names.index(k) for k in keys]
                    ga = {tuple(r[j] for j in kix): r for r in rows_a}
                    gb = {tuple(r[j] for j in kix): r for r in rows_b}
                    if set(ga) != set(gb) or len(ga) != len(rows_a) or len(gb) != len(rows_b):
                        problems.append("group keys differ")
                    else:
                        pairs = [(ga[k], gb[k]) for k in ga]
                else:
                    if not ordered:
                        order = lambda t: tuple((0, 0) if v is None else (1, v) for v in t)
                        rows_a, rows_b = sorted(rows_a, key=order), sorted(rows_b, key=order)
                    if len(rows_a) != len(rows_b):
                        problems.append(f"{len(rows_a)} rows != {len(rows_b)}")
                    pairs = list(zip(rows_a, rows_b))
                if not problems:
                    diff = [(names[j], x[j], y[j]) for x, y in pairs for j in range(len(names)) if not same_value(x[j], y[j], exact)]
                    if diff:
                        problems.append(f"{len(diff)} values differ, first {diff[:3]}")
            n = len(next(iter(ca.values()), []))
            print(f"{name}[{i}]: {n} rows, launches {ra['kernel_launches']}, {ra['main_kernel_name']}, h2d {ra['h2d_bytes']}, d2h {ra['d2h_bytes']}: "
                  + ("same" if not problems else "DIFFERENT: " + "; ".join(problems)))
            bad += bool(problems)
    print("all cases agree" if not bad else f"{bad} runs differ")
    return 1 if bad else 0


if __name__ == "__main__":
    if sys.argv[1] == "run":
        run(sys.argv[2])
    else:
        sys.exit(compare(sys.argv[2], sys.argv[3]))

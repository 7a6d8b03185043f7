"""GPU parity of the cross-region merge: a table split into 2, 3 or 5 regions, one plan handle per region on cuda:0, each region's partial
state exported (bkgpu_partial_export: k_partial_export_rows, or the top-k rows of sort_partial_export) into its slice of one device
buffer and folded by one handle (bkgpu_partial_merge: k_partial_merge_rows / merge_group, or sort_partial_merge).  The merged result is
compared with the plain reference of the whole table, bit for bit: tests/agg_type_cases.py's for aggregates (double sums whose value
depends on the order of addition within their "approx" bound, either sign of zero for MIN / MAX over mixed zeros), the row oracle with
rel=0 for joins, tests/region_merge_cases.py's stable sort (checked against the oracle on the CPU) for top-k.

Regions (tests/region_merge_cases.py): an empty region, a region of one row, a region holding only NULL-key (or NULL-value) rows, a group
whose rows all sit in one region, a group whose values are NULL in one region and present in another, ragged sizes.  The multi-GPU path
runs the same export and merge kernels, with the merging rank's own rows already in its table."""
import ctypes
import math
from collections import Counter

import numpy as np
import pytest
import torch

from baikaldb_b200 import _lib, plan as P
from baikaldb_b200._lib import BkgpuError
from baikaldb_b200.column import Column, make_column
from baikaldb_b200.plan import PlanNodeType, PrimitiveType as T
from oracle import oracle
from tests import join_key_cases as J
from tests.agg_type_cases import (AT, AVG_FNS, DIRECT, FNS, FX, FX_OPEN, INTERP, OPTIONS, SCALAR, SIGNED_ZERO, TYPES, Table, agg_plan,
                                  assert_matches, key_image, key_table, main_fns, reference, tname, value_table, zero_table)
from tests.region_merge_cases import (BIG, BIG_CASES, REGION_COUNTS, TOPK_KO, big_table, contiguous, role_layout, take, topk_cases, topk_plan,
                                      topk_reference, topk_table)
from tests.util import assert_same_rows, export_and_merge, merge_regions, open_node, partial_capacity

pytestmark = pytest.mark.gpu
N = 40_007
SUMS = ("count_star", "sum", "avg")   # FX's shape: every value column feeds one SUM lane


# ---------------------------------------------------------------- aggregates
def images(t: Table) -> list:
    return [key_image(t.kt, t.key_arr[i], t.key_valid is None or bool(t.key_valid[i])) if t.grouped else () for i in range(t.n)]


def agg_layout(t: Table, regions: int):
    """the role layout of `t`'s rows (region_merge_cases.role_layout).  The lonely group is the rarest present key with two rows or
    more.  Where `t` has NULL values, one group that has rows in the first and the last non-empty region loses its values in the first:
    NULL there, present in the other.  Returns the row indices of each region"""
    n, img = t.n, images(t)
    if t.grouped and t.key_valid is not None:
        null_rows = ~t.key_valid
    elif t.v_valid is not None:
        null_rows = ~t.v_valid
    else:
        null_rows = np.zeros(n, bool)
    lonely = np.zeros(n, bool)
    if t.grouped:
        counts = Counter(k for k, dead in zip(img, null_rows) if not dead and not k[0])
        pick = min((c, k) for k, c in counts.items() if c >= 2)[1]
        lonely = np.array([k == pick for k in img]) & ~null_rows
    parts = role_layout(n, regions, null_rows, lonely)
    if t.grouped and t.v_valid is not None:
        full = [p for p in parts if len(p) > 1 and not null_rows[p].all()]
        first, last = set(img[i] for i in full[0]), set(img[i] for i in full[-1])
        both = sorted(k for k in first & last if not k[0] and k != img[np.flatnonzero(lonely)[0]])
        assert both, "no group has rows in two regions"
        g = both[len(both) // 2]
        for i in full[0]:
            if img[i] == g:
                t.v_valid[i] = False
    return parts


def run_merged(plan, t: Table, fns, kernels, parts, want=None, passes=None, merger=0, groups=None):
    """`plan` over each region of `parts` on its own handle, region r pinned to kernels[r % len(kernels)]; the merged result against
    the reference of the whole table.  The largest region must have run the kernel it was pinned to.  `groups`: the number of groups
    each region's export must hold"""
    want = want if want is not None else reference(t, fns, passes)
    names = [kernels[r % len(kernels)] for r in range(len(parts))]
    stats, headers = [], []
    got = merge_regions(plan, [take(t.columns(), ix) for ix in parts], [OPTIONS[k] for k in names], merger, stats, headers)
    if groups is not None:
        assert headers == groups, (headers, groups)
    big = int(np.argmax([len(ix) for ix in parts]))
    if len(parts[big]):
        assert stats[big].main_kernel_name.decode() == names[big], (stats[big].main_kernel_name, names[big])
    assert_matches(got, want, t.kt if t.grouped else None, what=f"merge of {len(parts)} regions")
    return got


@pytest.mark.parametrize("nulls", [False, True], ids=["no_null_keys", "null_keys"])
@pytest.mark.parametrize("kt", TYPES, ids=tname)
def test_key_types(kt, nulls):
    """every key type (its edges, +-0.0 and NaN payloads of FLOAT / DOUBLE as separate groups, the EMPTY_KEY image as the hottest key),
    through the interpreter and the direct kernel in alternate regions"""
    i = TYPES.index(kt)
    rng = np.random.default_rng(20_000 + 2 * int(kt) + nulls)
    t = key_table(rng, kt, N, key_nulls=0.05 if nulls else 0.0, value_nulls=0.1)
    parts = agg_layout(t, REGION_COUNTS[(i + nulls) % 3])
    run_merged(agg_plan(t), t, FNS, [INTERP, DIRECT], parts, merger=i % len(parts))


@pytest.mark.parametrize("kernel", [INTERP, DIRECT, SCALAR])
@pytest.mark.parametrize("vt", TYPES, ids=tname)
def test_argument_types(vt, kernel):
    """COUNT(*), COUNT, SUM, MIN, MAX and AVG of every value type (agg_type_cases.value_table: edges, SUM of only -0.0, of mixed +-0.0,
    NaN and Inf, all-NULL groups, the largest finite values, denormals), every region pinned to `kernel`"""
    i = TYPES.index(vt)
    rng = np.random.default_rng(21_000 + 4 * int(vt) + [INTERP, DIRECT, SCALAR].index(kernel))
    t = value_table(rng, vt, N, grouped=kernel != SCALAR)
    parts = agg_layout(t, REGION_COUNTS[i % 3])
    run_merged(agg_plan(t, main_fns(vt)), t, main_fns(vt), [kernel], parts)
    run_merged(agg_plan(t, AVG_FNS), t, AVG_FNS, [kernel], parts, merger=len(parts) - 1)


@pytest.mark.parametrize("kt", [T.INT64, T.DOUBLE, T.UINT8, T.DATETIME, T.FLOAT, T.BOOL], ids=tname)
def test_two_keys(kt):
    """GROUP BY key, 0_2 WHERE 0_2 < 6: two key expressions and the NULL flags, several words per exported key"""
    rng = np.random.default_rng(22_000 + int(kt))
    t = key_table(rng, kt, N, key_nulls=0.05, value_nulls=0.1)
    parts = agg_layout(t, 3)
    plan = agg_plan(t, predicate=P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(6)), extra_keys=[P.slot_ref(0, 2, T.INT32)])
    stats = []
    got = merge_regions(plan, [take(t.columns(), ix) for ix in parts], [OPTIONS[INTERP], OPTIONS[DIRECT], OPTIONS[INTERP]], 1, stats)
    by = {c.name: c for c in got}
    second = by["0_2"].values
    assert sorted(set(second.tolist())) == list(range(6))
    for f in range(6):
        m = second == f
        rows = [Column(c.tuple_id, c.slot_id, c.prim_type, c.values[m], None if c.valid is None else c.valid[m]) for c in got]
        assert_matches(rows, reference(t, FNS, passes=lambda i: t.filt[i] == f), kt, what=f"0_2 = {f}")


def test_kernels_mixed_across_regions():
    """FX in one region, the interpreter in another, the direct kernel in a third: FX's limbs, the interpreter's and the direct
    kernel's double lanes meet as doubles"""
    rng = np.random.default_rng(23_000)
    t = key_table(rng, T.INT64, N)   # (NULL-free keys and values: FX's shape)
    parts = [np.arange(a, b) for a, b in contiguous(N, 3)]
    run_merged(agg_plan(t, SUMS), t, SUMS, [FX, INTERP, DIRECT], parts)
    run_merged(agg_plan(t, SUMS), t, SUMS, [DIRECT, FX, INTERP], parts, merger=2)


@pytest.mark.parametrize("what,mix", [(w, m) for m in ("interp_direct", "fx") for w in SIGNED_ZERO if (w, m) != ("minus_zero_nulls", "fx")])
def test_sum_of_signed_zeros(what, mix, request):
    """the reference's merge takes the first non-NULL SUM and adds the rest (AggFnCall::merge): -0.0 in every region gives -0.0, +0.0 in
    any region gives +0.0.  "fx": FX in the first region (NULL-free batches), whose SUM over only -0.0 comes out +0.0 (the recorded gap)"""
    if mix == "fx" and what == "minus_zero":
        request.applymarker(FX_OPEN)
    rng = np.random.default_rng(24_000 + list(SIGNED_ZERO).index(what))
    t = zero_table(rng, T.DOUBLE, what, N, nulls=mix != "fx")
    if mix == "fx":   # (every row passes: a filter that dropped a group's +-1.5 or +0.0 rows would leave it -0.0 only, the gap again)
        everything = P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(100))
        run_merged(agg_plan(t, SUMS, predicate=everything), t, SUMS, [FX, INTERP, DIRECT], [np.arange(a, b) for a, b in contiguous(N, 3)],
                   passes=lambda i: True)
    else:
        run_merged(agg_plan(t), t, FNS, [INTERP, DIRECT], agg_layout(t, 5))


@pytest.mark.parametrize("kernel", [SCALAR, INTERP])
def test_scalar_with_empty_and_filtered_regions(kernel):
    """the scalar aggregate: every region empty, and every row filtered out, give the blank row (COUNT 0, everything else NULL); SUM,
    MIN and MAX over only -0.0 stay -0.0 beside a region whose rows are all filtered out and an empty one (export skips the single
    group a region's rows never reached)"""
    rng = np.random.default_rng(25_000)
    t = value_table(rng, T.DOUBLE, N, grouped=False)
    none = np.zeros(0, np.int64)
    run_merged(agg_plan(t), t, FNS, [kernel], [none, none, none], want=reference(t, FNS, passes=lambda i: False), groups=[0, 0, 0])
    everything_out = agg_plan(t, predicate=P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(0)))
    run_merged(everything_out, t, FNS, [kernel], [np.arange(a, b) for a, b in contiguous(N, 3)], want=reference(t, FNS, passes=lambda i: False),
               groups=[0, 0, 0])
    z = zero_table(rng, T.DOUBLE, "minus_zero", N, grouped=False, nulls=False)
    spans = contiguous(N, 5)
    z.filt[spans[3][0]:spans[3][1]] = 50 + z.filt[spans[3][0]:spans[3][1]] % 50   # region 3: every row fails 0_2 < 50
    want = reference(z, FNS)
    assert want[()][f"{AT}_3"].value == -0.0 and math.copysign(1, want[()][f"{AT}_3"].value) < 0
    run_merged(agg_plan(z), z, FNS, [kernel], [np.arange(a, b) for a, b in spans], want=want, merger=1,
               groups=[int((z.filt[a:b] < 50).any()) for a, b in spans])


# ---------------------------------------------------------------- post fragments above the merged aggregate
@pytest.mark.parametrize("vt", [T.INT8, T.FLOAT, T.BOOL, T.UINT16], ids=tname)
def test_having_and_order_by_after_the_merge(vt):
    """HAVING COUNT(*) > c, ORDER BY MIN(v) DESC, key LIMIT 20 over the merged groups.  c is the largest count any group has in any one
    region, so every group that passes passes only on its merged count"""
    rng = np.random.default_rng(26_000 + int(vt))
    t = key_table(rng, T.INT32, N, vt=vt, value_nulls=0.05, n_random=200)
    parts = agg_layout(t, 3)
    img = images(t)
    c = max(max(Counter(img[i] for i in ix if t.filt[i] < 50).values()) for ix in parts if len(ix))
    a = agg_plan(t, main_fns(vt))
    having = P.where(a.root, P.gt(P.slot_ref(AT, 1, T.INT64), P.int_lit(c)), node_type=PlanNodeType.HAVING_FILTER_NODE)
    plan = P.Plan(P.limit(P.sort(having, [P.slot_ref(AT, 4, vt), P.slot_ref(0, 1, T.INT32)], [False, True], tuple_id=AT), 20), a.tuples)
    ref = {k: r for k, r in reference(t, main_fns(vt)).items() if r[f"{AT}_1"].value > c}
    assert len(ref) >= 20, (c, len(ref))
    order = sorted(ref, key=lambda k: (-(ref[k][f"{AT}_4"].value if ref[k][f"{AT}_4"].kind != "null" else -math.inf), k[1]))[:20]
    got = merge_regions(plan, [take(t.columns(), ix) for ix in parts], [OPTIONS[DIRECT], OPTIONS[INTERP], OPTIONS[DIRECT]])
    by = {x.name: x for x in got}
    assert [key_image(T.INT32, x, True) for x in by["0_1"].values] == order
    assert_matches(got, {k: ref[k] for k in order}, T.INT32)


# ---------------------------------------------------------------- joins
def _join_regions(case: J.Case, plan, keys):
    want = oracle.execute(plan.serialize(), case.all_columns()).columns
    for r in REGION_COUNTS:   # every region: all dimension rows, its own slice of the fact table
        regions = [case.dim_columns() + [take(case.fact_columns(), span)] for span in contiguous(case.n, r)]
        got = merge_regions(plan, regions, [{}] * r, merger=r - 1)
        assert_same_rows(got, want, keys, rel=0)


def test_two_table_join_aggregate():
    rng = np.random.default_rng(27_000)
    dim = J.make_dim(rng, 1, T.INT64, T.INT32, 300)
    case = J.make_case(rng, [dim], N)
    _join_regions(case, J.agg_plan([dim]), J.group_keys([dim]))
    _join_regions(case, J.agg_plan([dim], grouped=False), None)
    _join_regions(case, J.fused_plan(dim), ["1_3"])


def test_star_join_aggregate():
    rng = np.random.default_rng(27_001)
    pairs = [J.PAIRS[1], J.PAIRS[8], J.PAIRS[13]]
    dims = [J.make_dim(rng, d, dk, fk, 150 + 100 * d, null_keys=0.03) for d, (dk, fk) in enumerate(pairs, start=1)]
    case = J.make_case(rng, dims, N)
    _join_regions(case, J.agg_plan(dims), J.group_keys(dims))
    _join_regions(case, J.agg_plan(dims, grouped=False), None)


# ---------------------------------------------------------------- top-k
def assert_topk(got, keys, valid, want_rows, what):
    by = {c.name: c for c in got}
    assert np.array_equal(by["0_2"].values, want_rows), (what, by["0_2"].values[:8], want_rows[:8])
    kv = by["0_1"].valid if by["0_1"].valid is not None else np.ones(len(want_rows), bool)
    assert np.array_equal(kv, valid[want_rows]), what
    assert by["0_1"].values[kv].tobytes() == keys[want_rows][kv].tobytes(), what   # (bits: a -0.0 comes back -0.0)


def topk_regions(cols, spans):
    """each region's rows, its region_base the global number of its first row"""
    return [take(cols, s) for s in spans], [{"region_base": s[0]} for s in spans]


@pytest.mark.parametrize("kind", list(TOPK_KO))
@pytest.mark.parametrize("kt", TYPES, ids=tname)
def test_topk(kt, kind):
    """ORDER BY key ASC / DESC, NULLS FIRST / LAST, LIMIT k OFFSET o: the merged rows are rows [o, o + k) of a stable sort of the whole
    table, equal keys (-0.0 with +0.0) in global arrival order"""
    cols, keys, valid = topk_table(kt, kind)
    for i, (_, _, asc, nf, k, o) in enumerate(c for c in topk_cases() if c[:2] == (kt, kind)):
        spans = contiguous(len(keys), REGION_COUNTS[i % 3])
        batches, opts = topk_regions(cols, spans)
        got = merge_regions(topk_plan(kt, asc, nf, k, o), batches, opts, merger=i % len(spans))
        assert_topk(got, keys, valid, topk_reference(keys, valid, asc, nf, k, o), (asc, nf, k, o))


def test_topk_sampled_region():
    """one region of BIG rows, whose selection samples before it collects, beside a small one; keys repeat across both"""
    cols, keys, valid = big_table()
    spans = [(0, BIG), (BIG, len(keys))]
    for asc, nf, k, o in BIG_CASES:
        batches, opts = topk_regions(cols, spans)
        got = merge_regions(topk_plan(T.INT64, asc, nf, k, o), batches, opts, merger=1)
        assert_topk(got, keys, valid, topk_reference(keys, valid, asc, nf, k, o), (asc, nf, k, o))


# ---------------------------------------------------------------- refusals and limits
def _code(fn, *args, handle=None):
    with pytest.raises(BkgpuError) as e:
        _lib.check(fn(*args), handle)
    return e.value.code


def test_plans_without_a_partial_state_are_refused():
    """ORDER BY two keys with a LIMIT, LIMIT + OFFSET beyond 4096, ORDER BY without a LIMIT: no top-k state, capacity 0, export and
    merge refused"""
    cols, _, _ = topk_table(T.INT64, "dense")
    cols = cols + [make_column(0, 3, T.INT32, np.arange(len(cols[0].values), dtype=np.int32) % 7)]
    tuples = {0: [(1, T.INT64), (2, T.INT32), (3, T.INT32)]}
    k1, k3 = P.slot_ref(0, 1, T.INT64), P.slot_ref(0, 3, T.INT32)
    plans = [P.Plan(P.limit(P.sort(P.scan(0), [k3, k1], [True, False], tuple_id=0), 10), tuples),
             P.Plan(P.limit(P.sort(P.scan(0), [k1], [True], tuple_id=0), 4000, 97), tuples),
             P.Plan(P.sort(P.scan(0), [k1], [False], tuple_id=0), tuples)]
    L = _lib.lib()
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    for pl in plans:
        node, st = open_node(pl, cols)
        try:
            assert partial_capacity(node) == 0
            h, ptr = node.handle(), ctypes.c_void_p(buf.data_ptr())
            assert _code(L.bkgpu_partial_export, h, ptr, 64, handle=h) == _lib.EUNSUPPORTED
            assert _code(L.bkgpu_partial_merge, h, ptr, 0, 1, handle=h) == _lib.EUNSUPPORTED
        finally:
            node.close(st)


def test_bytes_per_rank_must_equal_the_capacity():
    rng = np.random.default_rng(28_000)
    t = key_table(rng, T.INT64, 5_003)
    cols, _, _ = topk_table(T.INT32, "dense", n=5_003)
    L = _lib.lib()
    for plan, region_cols in ((agg_plan(t), t.columns()), (topk_plan(T.INT32, True, True, 100, 3), cols)):
        nodes = [open_node(plan, take(region_cols, s)) for s in contiguous(5_003, 2)]
        try:
            nbytes = partial_capacity(nodes[0][0])
            buf = torch.zeros(2 * nbytes + 64, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            for r, (node, _) in enumerate(nodes):
                _lib.check(L.bkgpu_partial_export(node.handle(), ctypes.c_void_p(buf.data_ptr() + r * nbytes), nbytes), node.handle())
            h = nodes[0][0].handle()
            for wrong in (nbytes + 8, nbytes - 8):
                assert _code(L.bkgpu_partial_merge, h, ctypes.c_void_p(buf.data_ptr()), wrong, 2, handle=h) == _lib.EINVAL
            assert _code(L.bkgpu_partial_export, h, ctypes.c_void_p(buf.data_ptr()), nbytes - 8, handle=h) == _lib.EINVAL
        finally:
            for node, st in nodes:
                node.close(st)


def _int_table(keys, seed) -> Table:
    """INT32 keys, INT64 values, every row passing the filter"""
    rng = np.random.default_rng(seed)
    v = [int(x) for x in rng.integers(-1000, 1000, len(keys))]
    return Table(T.INT32, T.INT64, [int(k) for k in keys], None, np.zeros(len(keys), np.int32), v, None, list(v))


def test_partial_capacity_edge():
    """partial_capacity 500: regions of exactly 500 groups merge; a region of 501 fails its export with ETOOBIG, and a merge over what that
    export left in the buffer (a header of 501 groups) fails as well rather than returning the other regions' groups alone"""
    fns = ("count_star", "sum", "min")
    keys = np.concatenate([np.arange(500).repeat(3), np.arange(250, 750).repeat(2), np.arange(100, 600)])
    t = _int_table(keys, 29_000)
    spans = [(0, 1500), (1500, 2500), (2500, 3000)]
    plan = agg_plan(t, fns)
    headers = []
    got = merge_regions(plan, [take(t.columns(), s) for s in spans], [{"partial_capacity": 500}] * 3, headers=headers)
    assert headers == [500, 500, 500]
    assert_matches(got, reference(t, fns), T.INT32)
    over = _int_table(np.concatenate([np.arange(500), np.arange(1000, 1501)]), 29_001)
    L = _lib.lib()
    nodes = [open_node(agg_plan(over, fns), take(over.columns(), s), {"partial_capacity": 500}) for s in ((0, 500), (500, 1001))]
    try:
        nbytes = partial_capacity(nodes[0][0])
        buf = torch.zeros(2 * nbytes, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        h0, h1 = nodes[0][0].handle(), nodes[1][0].handle()
        _lib.check(L.bkgpu_partial_export(h0, ctypes.c_void_p(buf.data_ptr()), nbytes), h0)
        assert _code(L.bkgpu_partial_export, h1, ctypes.c_void_p(buf.data_ptr() + nbytes), nbytes, handle=h1) == _lib.ETOOBIG
        assert _code(L.bkgpu_partial_merge, h0, ctypes.c_void_p(buf.data_ptr()), nbytes, 2, handle=h0) == _lib.ETOOBIG
    finally:
        for node, st in nodes:
            node.close(st)


def test_union_beyond_the_group_table():
    """group_capacity_log2 = 10 (1024 slots): three regions of 700 groups each fit, but 2100 distinct groups do not fit the merging
    table (ETOOBIG, no partial answer); three regions of 700 groups whose union is 900 merge"""
    fns = ("count_star", "sum", "max")
    opts = {"group_capacity_log2": 10}
    disjoint = _int_table(np.concatenate([np.arange(r * 700, (r + 1) * 700) for r in range(3)]), 30_000)
    nodes = [open_node(agg_plan(disjoint, fns), take(disjoint.columns(), (r * 700, (r + 1) * 700)), opts) for r in range(3)]
    try:
        with pytest.raises(BkgpuError) as e:
            export_and_merge(nodes)
        assert e.value.code == _lib.ETOOBIG, e.value
    finally:
        for node, st in nodes:
            node.close(st)
    overlap = _int_table(np.concatenate([np.arange(r * 100, r * 100 + 700) for r in range(3)]), 30_001)
    got = merge_regions(agg_plan(overlap, fns), [take(overlap.columns(), (r * 700, (r + 1) * 700)) for r in range(3)], [opts] * 3)
    assert_matches(got, reference(overlap, fns), T.INT32)


# ---------------------------------------------------------------- reuse
def test_reset_and_merge_again():
    """export -> merge -> bkgpu_reset -> new rows -> export -> merge on the same handles: the second result is the second table's alone"""
    rng = np.random.default_rng(31_000)
    t1 = key_table(rng, T.INT64, N, key_nulls=0.05, value_nulls=0.1)
    t2 = key_table(rng, T.INT64, N, key_nulls=0.02, value_nulls=0.3, n_random=20)
    spans = contiguous(N, 5)
    cols1, keys1, valid1 = topk_table(T.DOUBLE, "dense", seed=0)
    cols2, keys2, valid2 = topk_table(T.DOUBLE, "dense", seed=1)
    # aggregate
    kernels = [INTERP, DIRECT]
    nodes = [open_node(agg_plan(t1), take(t1.columns(), s), OPTIONS[kernels[r % 2]]) for r, s in enumerate(spans)]
    try:
        assert_matches(export_and_merge(nodes, merger=2), reference(t1), T.INT64, what="first run")
        for (node, _), s in zip(nodes, spans):
            node.reset()
            node.push(take(t2.columns(), s))
            node.finish()
        assert_matches(export_and_merge(nodes, merger=2), reference(t2), T.INT64, what="second run")
    finally:
        for node, st in nodes:
            node.close(st)
    # top-k
    tspans = contiguous(len(keys1), 5)
    plan = topk_plan(T.DOUBLE, False, True, 1000, 100)
    nodes = [open_node(plan, take(cols1, s), {"region_base": s[0]}) for s in tspans]
    try:
        assert_topk(export_and_merge(nodes, merger=4), keys1, valid1, topk_reference(keys1, valid1, False, True, 1000, 100), "first run")
        for (node, _), s in zip(nodes, tspans):
            node.reset()
            node.push(take(cols2, s))
            node.finish()
        assert_topk(export_and_merge(nodes, merger=4), keys2, valid2, topk_reference(keys2, valid2, False, True, 1000, 100), "second run")
    finally:
        for node, st in nodes:
            node.close(st)

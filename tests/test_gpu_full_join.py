"""GPU: FULL OUTER joins under an aggregate and as returned rows, against Acero's FULL_OUTER hashjoin (tests/full_join_cases.py) — duplicate
and NULL keys on both sides, residual conditions, reconciliation filters above the join, empty and fully (un)matched sides, ragged probe
batches, pair counts beyond the first buffer, every integer key type, and one 10M x 1M join against torch."""
import math

import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import ColumnSource, GpuExecNode, RowBatch, RuntimeState, execute
from baikaldb_b200.plan import PrimitiveType as T
from tests import full_join_cases as F
from tests import join_key_cases as K
from tests.util import REL_TOL

pytestmark = pytest.mark.gpu

FULL = P.JoinType.FULL_JOIN
IS_NULL_EITHER = [("or", ("is_null", F.col(1, 1)), ("is_null", F.col(0, 1)))]
ARG_PRIM = {(1, 1): T.INT32, (1, 2): T.INT32, (1, 3): T.DOUBLE, (1, 4): T.INT64, (0, 1): T.INT32, (0, 2): T.DOUBLE, (0, 3): T.INT32, (0, 4): T.INT64}
AGGS = [("count_star", None), ("count", F.col(0, 2, T.DOUBLE)), ("sum", F.col(0, 2, T.DOUBLE)), ("min", F.col(0, 3)), ("max", F.col(1, 3, T.DOUBLE)),
        ("avg", F.col(1, 3, T.DOUBLE)), ("sum", F.col(0, 4, T.INT64))]


def cut(cols, a, b):
    return [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[a:b], None if c.valid is None else c.valid[a:b]) for c in cols]


def ragged(probe, sizes):
    out, a = [], 0
    for s in sizes:
        out.append(cut(probe, a, a + s)); a += s
    return out + [cut(probe, a, len(probe[0]))]


def join_node(residual):
    return P.join(P.scan(1), P.scan(0), [F.to_plan(F.ON)] + [F.to_plan(c) for c in residual], join_type=FULL)


def agg_plan(residual, above, group, aggs, tuples=None):
    fns, types = [], []
    for i, (name, arg) in enumerate(aggs):
        s = i + 1
        if name == "avg":
            fns.append(P.agg_expr("avg", 2, s, 20 + s, F.to_plan(arg)))
        else:
            fns.append(P.agg_expr(name, 2, s, None, *([] if arg is None else [F.to_plan(arg)])))
        types.append(T.INT64 if arg is None or name == "count" else arg[3])
    j = join_node(residual)
    root = P.agg(P.where(j, *[F.to_plan(c) for c in above]) if above else j, 2, [F.to_plan(g) for g in group], fns)
    return P.Plan(root, {**(tuples or F.TUPLES), 2: P.agg_tuple_slots(fns, types)})


def gpu_groups(cols, group, aggs):
    by = {c.name: c.to_list() for c in cols}
    gnames = [f"{g[1]}_{g[2]}" for g in group]
    n = len(cols[0]) if cols else 0
    out = {}
    for r in range(n):
        vals = []
        for i, (name, _) in enumerate(aggs):
            v = by[f"2_{i + 1}" if f"2_{i + 1}" in by else f"2_{21 + i}"][r]
            if isinstance(v, bytes):   # AVG's {double sum; int64 count}
                s, c = np.frombuffer(v, np.float64, 1)[0], np.frombuffer(v, np.int64, 1, 8)[0]
                v = None if c == 0 else float(s) / int(c)
            vals.append(v)
        out[tuple(by[g][r] for g in gnames)] = vals
    return out


def assert_groups(got, want):
    assert set(got) == set(want), (sorted(set(got) - set(want), key=str)[:5], sorted(set(want) - set(got), key=str)[:5])
    for k in want:
        for x, y in zip(got[k], want[k]):
            if x is None or y is None:
                assert x is None and y is None, (k, got[k], want[k])
            elif isinstance(y, float) or isinstance(x, float):
                assert math.isclose(x, y, rel_tol=REL_TOL, abs_tol=1e-9), (k, got[k], want[k])
            else:
                assert x == y, (k, got[k], want[k])


def check_agg(build, probe, residual, above, group, aggs=AGGS, batches=None, options=None):
    got, stats = execute(agg_plan(residual, above, group, aggs), batches or [build, probe], device=0, options=options)
    rows = F.acero_full_join(F.arrow_table(build), F.arrow_table(probe), "1_1", "0_1", residual, above).to_pylist()
    want = F.aggregate(rows, [f"{g[1]}_{g[2]}" for g in group], [(n, None if a is None else f"{a[1]}_{a[2]}") for n, a in aggs])
    assert_groups(gpu_groups(got, group, aggs), want)
    return stats


def check_rows(build, probe, residual, above, batches=None, options=None):
    j = join_node(residual)
    child = P.where(j, *[F.to_plan(c) for c in above]) if above else j
    names = [c.name for c in build + probe]
    want = F.acero_full_join(F.arrow_table(build), F.arrow_table(probe), "1_1", "0_1", residual, above).to_pylist()
    got, _ = execute(P.Plan(P.packet(child), F.TUPLES), batches or [build, probe], device=0, options=options)
    assert F.multiset(F.rows_of(got), names) == F.multiset(want, names)
    # ORDER BY probe row id, build row id (NULLs first) + LIMIT / OFFSET: the exact rows in order
    keys = [P.slot_ref(0, 4, T.INT64), P.slot_ref(1, 4, T.INT64)]
    got, _ = execute(P.Plan(P.limit(P.sort(child, keys, [True, True], tuple_id=0), 60, offset=7), F.TUPLES), batches or [build, probe], device=0, options=options)
    order = sorted(want, key=lambda r: F.row_key(r, ["0_4", "1_4"]))[7:67]
    assert [F.row_key(r, names) for r in F.rows_of(got)] == [F.row_key(r, names) for r in order]
    return want


@pytest.mark.parametrize("residual", [[], [("gt", ("add", F.col(0, 3), F.col(1, 2)), ("int", 9))], [("gt", F.col(0, 3), ("int", 5))]],
                         ids=["keys", "both-tuples", "one-sided"])
@pytest.mark.parametrize("above", [[], IS_NULL_EITHER, [("or", ("is_null", F.col(0, 4)), ("lt", F.col(0, 3), ("int", 4)))],
                                   [("gt", ("ifnull", F.col(1, 2), ("int", 4)), ("int", 3))]], ids=["none", "is-null", "or", "ifnull"])
def test_full_join_aggregate(residual, above):
    rng = np.random.default_rng(len(residual) * 7 + len(str(above)))
    build, probe = F.random_tables(rng, 3_000, 40_000, key_range=2_400)
    batches = [build] + ragged(probe, [1, 9_999, 13_001])          # matched[] spans the probe batches
    check_agg(build, probe, residual, above, [F.col(1, 2)], batches=batches)
    check_agg(build, probe, residual, above, [F.col(0, 3)], batches=batches)   # a probe-side key: the build rows' NULL group
    check_agg(build, probe, residual, above, [F.col(1, 2), F.col(0, 3)], [("count_star", None), ("sum", F.col(1, 4, T.INT64))], batches=batches)


def test_full_join_aggregate_general_kernel_and_no_group():
    rng = np.random.default_rng(5)
    build, probe = F.random_tables(rng, 2_000, 30_000, key_range=1_500)
    stats = check_agg(build, probe, [], IS_NULL_EITHER, [F.col(1, 2)], options={"force_generic": 1})
    assert stats.main_kernel_name.decode() == "k_agg_interp"
    check_agg(build, probe, [("lt", F.col(1, 2), ("int", 6))], [], [])


@pytest.mark.parametrize("case", ["empty-build", "empty-probe", "all-matched", "none-matched"])
def test_full_join_edges(case):
    rng = np.random.default_rng(17)
    build, probe = F.random_tables(rng, 1_000, 8_000, key_range=1_000, null_frac=0.0)
    if case == "empty-build":
        build = cut(build, 0, 0)
    elif case == "empty-probe":
        probe = cut(probe, 0, 0)
    elif case == "all-matched":
        keys = np.arange(1_000, dtype=np.int32)
        build[0] = make_column(1, 1, T.INT32, keys)
        probe[0] = make_column(0, 1, T.INT32, np.concatenate([keys, rng.integers(0, 1_000, 7_000)]).astype(np.int32))
    else:
        probe[0] = make_column(0, 1, T.INT32, rng.integers(5_000, 9_000, 8_000))
    for above in ([], IS_NULL_EITHER):
        check_agg(build, probe, [], above, [F.col(1, 2)])
        check_agg(build, probe, [], above, [])
        check_rows(build, probe, [], above)


def test_pairs_beyond_the_first_buffer_are_rerun():
    """few keys, many duplicates on both sides: a probe batch joins to far more pairs than it has rows (the first guess), so the pair pass
    runs again with the buffer grown to the count"""
    rng = np.random.default_rng(23)
    build, probe = F.random_tables(rng, 400, 6_000, key_range=12, null_frac=0.05)
    want = check_rows(build, probe, [("gt", F.col(0, 3), ("int", 2))], [])
    assert len(want) > 4 * 6_000
    check_agg(build, probe, [("gt", F.col(0, 3), ("int", 2))], [], [F.col(1, 2)])


@pytest.mark.parametrize("residual", [[], [("gt", ("add", F.col(0, 3), F.col(1, 2)), ("int", 9))]], ids=["keys", "residual"])
@pytest.mark.parametrize("above", [[], IS_NULL_EITHER], ids=["none", "is-null"])
def test_full_join_rows(residual, above):
    rng = np.random.default_rng(41 + len(residual) + 2 * len(above))
    build, probe = F.random_tables(rng, 1_500, 20_000, key_range=1_800)
    want = check_rows(build, probe, residual, above, batches=[build] + ragged(probe, [7_777, 3]))
    assert any(r["1_1"] is None and r["1_4"] is None for r in want) and any(r["0_4"] is None for r in want)


def test_same_plan_twice_through_reset():
    rng = np.random.default_rng(3)
    build, probe = F.random_tables(rng, 2_000, 25_000, key_range=2_000)
    pl = agg_plan([("gt", F.col(0, 3), ("int", 3))], IS_NULL_EITHER, [F.col(1, 2)], AGGS)
    node, st = GpuExecNode(), RuntimeState(device=0)
    node.init(pl)
    node.add_child(ColumnSource([build, probe]))
    results = []
    try:
        assert node.open(st) == 0, st.error_msg
        for i in range(2):
            if i:
                node.reset(); node.push(build); node.push(probe); node.finish()
            got, eos, rb = [], False, RowBatch()
            while not eos:
                rc, eos = node.get_next(st, rb)
                assert rc == 0
                got = got or list(rb.columns)
            results.append(gpu_groups(got, [F.col(1, 2)], AGGS))
    finally:
        node.close(st)
    assert_groups(results[1], results[0])
    rows = F.acero_full_join(F.arrow_table(build), F.arrow_table(probe), "1_1", "0_1", [("gt", F.col(0, 3), ("int", 3))], IS_NULL_EITHER).to_pylist()
    assert_groups(results[0], F.aggregate(rows, ["1_2"], [(n, None if a is None else f"{a[1]}_{a[2]}") for n, a in AGGS]))


@pytest.mark.parametrize("pair", K.PAIRS, ids=K.pair_id)
def test_every_integer_key_type(pair):
    """dimension key type dk, fact key type fk: keys compared in their cast type, NULLs on both sides, duplicate and unmatched keys"""
    dk, fk = pair
    rng = np.random.default_rng(abs(hash(K.pair_id(pair))) % 2**32)
    keys = K.unique_keys(rng, dk, fk, 300)
    nd = len(keys)
    dkeys = keys + keys[: nd // 5]                                   # duplicate build keys
    dvalid = rng.random(len(dkeys)) > 0.05
    shared = [k for k in keys if K.in_range(fk, k)]
    fkeys = [shared[i] for i in rng.integers(0, len(shared), 2_000)] + K.misses_for(rng, keys, fk)[:300]
    fvalid = rng.random(len(fkeys)) > 0.05
    dtype = lambda t: np.dtype(K.storage_dtype(t))
    build = [make_column(1, 1, dk, np.array(dkeys, dtype=object).astype(dtype(dk)), dvalid),
             make_column(1, 2, T.INT64, np.array([K.attr64(k) for k in dkeys], dtype=np.int64)), make_column(1, 3, T.INT32, np.array([k % 7 for k in dkeys], dtype=np.int32))]
    probe = [make_column(0, 1, T.INT64, np.arange(len(fkeys))), make_column(0, 10, fk, np.array(fkeys, dtype=object).astype(dtype(fk)), fvalid)]
    tuples = {1: [(1, dk), (2, T.INT64), (3, T.INT32)], 0: [(1, T.INT64), (10, fk)]}
    aggs = [("count_star", None), ("sum", F.col(0, 1, T.INT64)), ("sum", F.col(1, 2, T.INT64)), ("min", F.col(1, 2, T.INT64))]
    fns = [P.agg_expr("count_star", 2, 1)] + [P.agg_expr(n, 2, i + 2, None, F.to_plan(a)) for i, (n, a) in enumerate(aggs[1:])]
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, dk), P.slot_ref(0, 10, fk))], join_type=FULL)
    pl = P.Plan(P.agg(j, 2, [P.slot_ref(1, 3, T.INT32)], fns), {**tuples, 2: P.agg_tuple_slots(fns, [T.INT64, T.INT64, T.INT64, T.INT64])})
    got, _ = execute(pl, [build, probe], device=0)
    rows = F.acero_full_join(F.arrow_table(build), F.arrow_table(probe), "1_1", "0_10", [], []).to_pylist()
    want = F.aggregate(rows, ["1_3"], [(n, None if a is None else f"{a[1]}_{a[2]}") for n, a in aggs])
    assert_groups(gpu_groups(got, [F.col(1, 3)], aggs), want)


def test_ten_million_by_one_million_against_torch():
    """GROUP BY a dimension attribute, COUNT(*), SUM(x): the partner of every fact row through a key -> row map in torch"""
    import torch
    nf, nd = 10_000_000, 1_000_000
    g = torch.Generator().manual_seed(11)
    key = torch.randperm(nd, generator=g).to(torch.int32)
    attr = (key % 97).to(torch.int32)
    fk = torch.randint(nd // 10, nd + nd // 20, (nf,), generator=g, dtype=torch.int32)
    x = torch.randint(-1000, 1000, (nf,), generator=g).double() / 8
    fvalid, dvalid = torch.rand(nf, generator=g) > 1e-4, torch.rand(nd, generator=g) > 1e-4
    build = [make_column(1, 1, T.INT32, key.numpy(), dvalid.numpy()), make_column(1, 2, T.INT32, attr.numpy())]
    probe = [make_column(0, 1, T.INT32, fk.numpy(), fvalid.numpy()), make_column(0, 2, T.DOUBLE, x.numpy())]
    aggs = [("count_star", None), ("sum", F.col(0, 2, T.DOUBLE))]
    tuples = {0: [(1, T.INT32), (2, T.DOUBLE)], 1: [(1, T.INT32), (2, T.INT32)]}
    got, _ = execute(agg_plan([], [], [F.col(1, 2)], aggs, tuples), [build] + ragged(probe, [4_000_000]), device=0)
    row_of = torch.full((nd,), -1, dtype=torch.int64)
    row_of[key[dvalid].long()] = torch.arange(nd)[dvalid]
    ok = fvalid & (fk < nd)
    partner = torch.full((nf,), -1, dtype=torch.int64)
    partner[ok] = row_of[fk[ok].long()]
    hit = partner >= 0
    matched = torch.zeros(nd, dtype=torch.bool); matched[partner[hit]] = True
    grp = torch.full((nf,), 97, dtype=torch.int64)   # 97 = the NULL group
    grp[hit] = attr[partner[hit]].long()
    cnt = torch.bincount(grp, minlength=98) + torch.bincount(attr[~matched].long(), minlength=98)
    sm = torch.zeros(98, dtype=torch.float64).index_add_(0, grp, x)
    want = {(None if a == 97 else a,): [int(cnt[a]), float(sm[a])] for a in range(98)}
    assert_groups(gpu_groups(got, [F.col(1, 2)], aggs), want)

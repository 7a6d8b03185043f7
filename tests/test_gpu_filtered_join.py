"""GPU parity: LEFT / RIGHT / SEMI / ANTI_SEMI joins over filtered children against the row oracle (whose meaning
tests/test_filtered_join_plan.py pins against Acero's filter -> hashjoin), and one 10M x 1M case against torch."""
import numpy as np
import pytest

from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.exec_node import ColumnSource, GpuExecNode, RowBatch, RuntimeState, execute
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests import filtered_join_cases as C
from tests import full_join_cases as F
from tests.date_fn_cases import date_image
from tests.full_join_cases import col
from tests.util import assert_same_rows, ragged, run_both

pytestmark = pytest.mark.gpu


def pairs(jt, build, probe, bf=(), pf=(), residual=(), batches=None):
    """the joined rows as row ids, GPU against the oracle; returns the oracle's {(row ids...): count}"""
    got, _, want = run_both(C.pairs_plan(jt, bf, pf, residual), build + probe, keys=C.group_names(jt), batches=batches or [build, probe])
    return C.counted(want.columns, C.group_names(jt))


def small_tables():
    """build rows (id: key, 1_2): 0: 1, 5   1: 1, 1   2: 2, 5   3: 3, 1   4: NULL, 5   5: NULL, 1   6: 4, 5; probe keys 1 (0_2 NULL), 3, 3, NULL"""
    kv = np.array([True, True, True, True, False, False, True])
    build = [make_column(1, 1, T.INT32, np.array([1, 1, 2, 3, 0, 0, 4]), kv), make_column(1, 2, T.INT32, np.array([5, 1, 5, 1, 5, 1, 5])),
             make_column(1, 3, T.DOUBLE, np.arange(7) / 4.0), make_column(1, 4, T.INT64, np.arange(7))]
    probe = [make_column(0, 1, T.INT32, np.array([1, 3, 3, 0]), np.array([True, True, True, False])),
             make_column(0, 2, T.DOUBLE, np.array([0.0, 2.5, -1.0, 4.0]), np.array([False, True, True, True])),
             make_column(0, 3, T.INT32, np.array([1, 2, 3, 4])), make_column(0, 4, T.INT64, np.arange(4))]
    return build, probe


def test_build_rows_that_fail_their_filter_vanish():
    """1_2 > 3 keeps build rows 0, 2, 4 (NULL key), 6: rows 1 and 3 have partners but fail, row 5 (NULL key) fails — none of them is emitted"""
    build, probe = small_tables()
    keep = [("gt", col(1, 2), ("int", 3))]
    assert set(pairs("SEMI_JOIN", build, probe, keep)) == {(0,)}
    assert set(pairs("ANTI_SEMI_JOIN", build, probe, keep)) == {(2,), (4,), (6,)}
    # a probe filter that is NULL for the only probe row with key 1 (0_2 NULL): that row joins nothing
    assert not pairs("SEMI_JOIN", build, probe, keep, [("gt", col(0, 2, T.DOUBLE), ("int", 0))])
    assert set(pairs("ANTI_SEMI_JOIN", build, probe, keep, [("gt", col(0, 2, T.DOUBLE), ("int", 0))])) == {(0,), (2,), (4,), (6,)}
    left = pairs("LEFT_JOIN", build, probe, pf=[("gt", col(0, 2, T.DOUBLE), ("int", 0))])
    assert left[(3, 1)] == 1 and left[(0, None)] == 1 and left[(1, None)] == 1 and (3, 2) not in left


@pytest.mark.parametrize("seed", range(12))
def test_random_filtered_joins(seed):
    """duplicate and NULL keys on both sides, filters that are NULL, residual conditions, a probe side in ragged batches"""
    rng = np.random.default_rng(1000 + seed)
    jt, bf, pf, residual = C.random_case(rng, seed)
    build, probe = F.random_tables(rng, 3_000, 40_000, key_range=2_500, null_frac=0.1)
    want = pairs(jt, build, probe, bf, pf, residual, batches=[build] + ragged(probe, [12_345, 3, 8_000]))
    assert want


@pytest.mark.parametrize("jt", ["LEFT_JOIN", "RIGHT_JOIN", "SEMI_JOIN", "ANTI_SEMI_JOIN"])
def test_everything_filtered_away_and_an_empty_probe_side(jt):
    rng = np.random.default_rng(5)
    build, probe = F.random_tables(rng, 500, 4_000, key_range=400)
    none_p = [("gt", col(0, 3), ("int", 1000))]
    n_out = sum(pairs(jt, build, probe, pf=none_p).values())
    assert n_out == (0 if jt == "SEMI_JOIN" else 500)                # no probe row: every build row is unmatched
    empty = [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[:0]) for c in probe]
    assert sum(pairs(jt, build, empty, pf=[("lt", col(0, 3), ("int", 7))]).values()) == (0 if jt == "SEMI_JOIN" else 500)
    if "SEMI" in jt:
        assert not pairs(jt, build, probe, bf=[("gt", col(1, 2), ("int", 100))])   # no build row
        kept = int((build[1].values > 3).sum())
        assert sum(pairs(jt, build, empty, bf=[("gt", col(1, 2), ("int", 3))]).values()) == (0 if jt == "SEMI_JOIN" else kept)


def test_a_long_in_list_and_a_date_function_in_child_filters():
    """WHERE k IN (1000 values) AND MONTH(d) <= 6 in the probe child, YEAR(d) >= 1995 in the build child (an uncorrelated IN / EXISTS subquery)"""
    rng = np.random.default_rng(17)
    nb, np_ = 4_000, 60_000

    def days(n):   # (DATE images, their year, their month)
        y, m, d = rng.integers(1990, 2000, n), rng.integers(1, 13, n), rng.integers(1, 29, n)
        return np.array([date_image(int(a), int(b), int(c)) for a, b, c in zip(y, m, d)], dtype=np.uint32), y, m
    bd, by, _ = days(nb)
    pd, _, pm = days(np_)
    # slots 4: YEAR / MONTH of the DATE column, precomputed for the oracle (which has no date functions)
    build = [make_column(1, 1, T.INT32, rng.integers(0, 3_000, nb), rng.random(nb) > 0.05), make_column(1, 2, T.INT32, rng.integers(0, 20, nb)),
             make_column(1, 3, T.DATE, bd), make_column(1, 4, T.INT64, by)]
    probe = [make_column(0, 1, T.INT32, rng.integers(0, 3_500, np_), rng.random(np_) > 0.05), make_column(0, 2, T.DATE, pd),
             make_column(0, 3, T.INT32, rng.integers(0, 4_000, np_)), make_column(0, 4, T.INT64, pm)]
    tuples = {1: [(1, T.INT32), (2, T.INT32), (3, T.DATE), (4, T.INT64)], 0: [(1, T.INT32), (2, T.DATE), (3, T.INT32), (4, T.INT64)]}
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("max", 2, 2, None, P.slot_ref(1, 1, T.INT32))]
    in_list = P.in_(P.slot_ref(0, 3, T.INT32), *[P.int_lit(i * 3) for i in range(1000)])
    on = [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))]

    def plan(jt, year, month):
        probe_f = P.where(P.scan(0), in_list, P.le(month, P.int_lit(6)))
        build_f = P.where(P.scan(1), P.ge(year, P.int_lit(1995))) if jt != "LEFT_JOIN" else P.scan(1)
        return P.Plan(P.agg(P.join(build_f, probe_f, on, join_type=getattr(P.JoinType, jt)), 2, [P.slot_ref(1, 2, T.INT32)], aggs),
                      {**tuples, 2: P.agg_tuple_slots(aggs, [T.INT64, T.INT32])})
    for jt in ("SEMI_JOIN", "ANTI_SEMI_JOIN", "LEFT_JOIN"):
        got, _ = execute(plan(jt, P.common("year", P.slot_ref(1, 3, T.DATE)), P.common("month", P.slot_ref(0, 2, T.DATE))), [build, probe], device=0)
        want = oracle.execute(plan(jt, P.slot_ref(1, 4, T.INT64), P.slot_ref(0, 4, T.INT64)).serialize(), build + probe).columns
        assert_same_rows(got, want, ["1_2"])
        assert 0 < sum({c.name: c for c in got}["2_1"].to_list())


@pytest.mark.parametrize("jt", ["LEFT_JOIN", "RIGHT_JOIN", "SEMI_JOIN", "ANTI_SEMI_JOIN"])
def test_group_by_either_side(jt):
    rng = np.random.default_rng(29)
    build, probe = F.random_tables(rng, 2_000, 30_000, key_range=1_800)
    pf = [("lt", col(0, 3), ("add", col(0, 1), ("int", 2))), ("or", ("is_null", col(0, 2, T.DOUBLE)), ("gt", col(0, 2, T.DOUBLE), ("int", -100)))]
    bf = [] if jt in ("LEFT_JOIN", "RIGHT_JOIN") else [("ne", col(1, 2), ("int", 4))]
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("count", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE)), P.agg_expr("sum", 2, 3, None, P.slot_ref(1, 3, T.DOUBLE)),
            P.agg_expr("min", 2, 4, None, P.slot_ref(0, 3, T.INT32)), P.agg_expr("avg", 2, 5, 6, P.slot_ref(0, 2, T.DOUBLE))]
    slots = P.agg_tuple_slots(aggs, [T.INT64, T.INT64, T.DOUBLE, T.INT32, T.DOUBLE])
    for group in ([P.slot_ref(1, 2, T.INT32)], [P.slot_ref(0, 3, T.INT32)], [P.slot_ref(1, 2, T.INT32), P.slot_ref(0, 3, T.INT32)], []):
        pl = P.Plan(P.packet(P.agg(C.join(jt, bf, pf, C.RESIDUALS[1]), 2, group, aggs)), {**C.TUPLES, 2: slots})
        run_both(pl, build + probe, keys=[f"{g.tuple_id}_{g.slot_id}" for g in group], batches=[build] + ragged(probe, [9_999]))


@pytest.mark.parametrize("jt", ["LEFT_JOIN", "RIGHT_JOIN"])
def test_outer_join_rows_over_a_filtered_inner_side(jt):
    rng = np.random.default_rng(37)
    build, probe = F.random_tables(rng, 1_500, 20_000, key_range=1_800)
    pf = [("gt", col(0, 2, T.DOUBLE), ("int", -60)), ("lt", col(0, 3), ("int", 9))]
    batches = [build] + ragged(probe, [7_777, 3])
    got, _, _ = run_both(P.Plan(C.join(jt, pfilter=pf, residual=C.RESIDUALS[2]), C.TUPLES), build + probe, keys=["1_4", "0_4"], batches=batches)
    assert None in {c.name: c for c in got}["0_4"].to_list()
    order = [P.slot_ref(1, 4, T.INT64), P.slot_ref(0, 4, T.INT64)]
    top = P.limit(P.sort(C.join(jt, pfilter=pf), order, [True, False], tuple_id=0), 50, offset=7)
    run_both(P.Plan(top, C.TUPLES), build + probe, keys=None, batches=batches, check_scanned=False)


def test_same_plan_twice_through_reset_with_other_build_rows():
    """the build child's filter, the multimap and matched[] are rebuilt for the second request's build rows"""
    rng = np.random.default_rng(43)
    pl = C.pairs_plan("ANTI_SEMI_JOIN", [("or", ("is_null", col(1, 1)), ("lt", col(1, 2), ("int", 6)))], [("lt", col(0, 3), ("int", 7))])
    runs = [F.random_tables(rng, 2_000, 25_000, key_range=2_000), F.random_tables(rng, 3_000, 20_000, key_range=2_500, null_frac=0.2)]
    node, st = GpuExecNode(), RuntimeState(device=0)
    node.init(pl)
    node.add_child(ColumnSource([runs[0][0], runs[0][1]]))
    try:
        assert node.open(st) == 0, st.error_msg
        for i, (build, probe) in enumerate(runs):
            if i:
                node.reset(); node.push(build); node.push(probe); node.finish()
            got, eos, rb = [], False, RowBatch()
            while not eos:
                rc, eos = node.get_next(st, rb)
                assert rc == 0
                got = got or list(rb.columns)
            assert_same_rows(got, oracle.execute(pl.serialize(), build + probe).columns, ["1_4"])
    finally:
        node.close(st)


@pytest.mark.parametrize("jt", ["SEMI_JOIN", "ANTI_SEMI_JOIN"])
def test_ten_million_by_one_million_against_torch(jt):
    """1M build rows (filter bflag < 7, a few NULL keys) x 10M probe rows (filter a < b + 20), GROUP BY a build attribute, COUNT(*)"""
    import torch
    nb, np_ = 1_000_000, 10_000_000
    g = torch.Generator().manual_seed(13)
    key = torch.randperm(nb, generator=g).to(torch.int32)
    attr = (key % 97).to(torch.int32)
    bflag = torch.randint(0, 10, (nb,), generator=g, dtype=torch.int32)
    fk = torch.randint(0, nb + nb // 20, (np_,), generator=g, dtype=torch.int32)
    a, b = torch.randint(0, 100, (np_,), generator=g, dtype=torch.int32), torch.randint(0, 100, (np_,), generator=g, dtype=torch.int32)
    dvalid, fvalid = torch.rand(nb, generator=g) > 1e-4, torch.rand(np_, generator=g) > 1e-4
    build = [make_column(1, 1, T.INT32, key.numpy(), dvalid.numpy()), make_column(1, 2, T.INT32, attr.numpy()), make_column(1, 3, T.INT32, bflag.numpy())]
    probe = [make_column(0, 1, T.INT32, fk.numpy(), fvalid.numpy()), make_column(0, 2, T.INT32, a.numpy()), make_column(0, 3, T.INT32, b.numpy())]
    tuples = {1: [(1, T.INT32), (2, T.INT32), (3, T.INT32)], 0: [(1, T.INT32), (2, T.INT32), (3, T.INT32)]}
    aggs = [P.agg_expr("count_star", 2, 1)]
    j = P.join(P.where(P.scan(1), P.lt(P.slot_ref(1, 3, T.INT32), P.int_lit(7))),
               P.where(P.scan(0), P.lt(P.slot_ref(0, 2, T.INT32), P.add(P.slot_ref(0, 3, T.INT32), P.int_lit(20)))),
               [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))], join_type=getattr(P.JoinType, jt))
    pl = P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs), {**tuples, 2: P.agg_tuple_slots(aggs, [T.INT64])})
    got, _ = execute(pl, [build] + ragged(probe, [4_000_000]), device=0)
    hit = torch.zeros(nb, dtype=torch.bool)
    live = fvalid & (a < b + 20) & (fk < nb)
    hit[fk[live].long()] = True
    passes = bflag < 7
    matched = passes & dvalid & hit[key.long()]
    emit = matched if jt == "SEMI_JOIN" else passes & ~matched
    cnt = torch.bincount(attr[emit].long(), minlength=97)
    want = {k: int(cnt[k]) for k in range(97) if cnt[k] > 0}
    by = {c.name: c.to_list() for c in got}
    assert dict(zip(by["1_2"], by["2_1"])) == want

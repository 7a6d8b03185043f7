"""Host only: the plans of tests/row_store_cases.py lower, and the row oracle (and the window oracle) agree with the NumPy reference of
which input rows pass through, on ~2k-row versions of the tables.  The GPU tests (tests/test_gpu_row_store.py) rest on that
reference."""
import numpy as np
import pytest

from baikaldb_b200 import _lib
from baikaldb_b200 import plan as P
from baikaldb_b200.column import make_column
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests import row_store_cases as R
from tests import window_oracle

N = 2_100


def small_scan(rng, types, layout):
    return R.scan_table(rng, types, layout, n=N, cuts=R.SMALL_CUTS)


def small_join(rng, types, layout, **kw):
    return R.join_tables(rng, types, layout, nb=N, np_=900, bcuts=R.SMALL_CUTS, pcuts=[3, 300, 13], **kw)


def plans(types):
    rng = np.random.default_rng(1)
    t = small_scan(rng, types, "seam")
    b, p = small_join(rng, types, "seam")
    fact, dims = R.star_tables(rng, types, nf=3_000)
    out = [R.where_plan(t), R.where_plan(t, 1_000, 5), R.sort_plan(t), R.window_plan(t), R.window_plan(t, (900, 7))]
    out += [R.join_rows_plan(b, p, jt) for jt in R.JOIN_TYPES]
    out += [R.join_agg_plan(b, p, "INNER_JOIN", a) for a in R.arg_chunks(b.payloads())]
    out += [R.join_agg_plan(b, p, "FULL_JOIN", a) for a in R.arg_chunks(b.payloads() + p.payloads())]
    out += [R.star_plan(fact, dims, a) for a in R.arg_chunks(R.star_args(fact, dims))]
    return out + [R.merge_join_case(rng, nb=100, np_=100)[0]]


@pytest.mark.parametrize("group", list(R.GROUPS))
def test_every_plan_lowers(group):
    for pl in plans(R.GROUPS[group]):
        assert _lib.explain(pl.serialize())


def test_merge_over_a_join_carries_a_string_build_column():
    """a 16-byte STRING build column (AVG's {sum, count} blob) reaches the join's aggregate through MERGE_AGG; the oracle's merged
    result is the NumPy one, which the GPU test of the FK -> PK gather compares against"""
    plan, build, probe = R.merge_join_case(np.random.default_rng(3), nb=3_000, np_=5_000)
    text = _lib.explain(plan.serialize())
    assert text.startswith("kind=4") and f"= {R.AT}_3 prim={int(T.STRING)}" in text
    by = {c.name: c for c in oracle.execute(plan.serialize(), build + probe).columns}
    want = R.merge_join_reference(build, probe)
    assert sorted(by[f"0_{R.GRP}"].values.tolist()) == sorted(want)
    for i, g in enumerate(by[f"0_{R.GRP}"].values.tolist()):
        n, total, cnt = want[g]
        blob = by[f"{R.AT}_3"].values[i]
        assert int(by[f"{R.AT}_1"].values[i]) == n
        assert blob[:8].view("<f8")[0] == total and blob[8:].view("<i8")[0] == cnt
        assert by[f"{R.AT}_2"].values[i] == total / cnt


@pytest.mark.parametrize("layout", R.LAYOUTS)
@pytest.mark.parametrize("group", list(R.GROUPS))
def test_oracle_agrees_on_scans(group, layout):
    rng = np.random.default_rng(10 + R.LAYOUTS.index(layout))
    t = small_scan(rng, R.GROUPS[group], layout)
    for pl, ids, ordered in ((R.where_plan(t), R.where_ids(t), False), (R.where_plan(t, 1_000, 5), None, False),
                             (R.sort_plan(t), R.sort_ids(t), True)):
        got = oracle.execute(pl.serialize(), t.cols).columns
        if ids is None:   # a LIMIT over unordered rows: which rows is the engine's choice, not their bytes
            ids = got[0].values
            assert len(ids) == 1_000 and set(ids) <= set(R.where_ids(t))
        R.assert_rows(got, [(t, t.index_of(ids))], ordered, what="oracle")


@pytest.mark.parametrize("layout", R.LAYOUTS)
@pytest.mark.parametrize("group", list(R.GROUPS))
def test_window_oracle_agrees(group, layout):
    rng = np.random.default_rng(20 + R.LAYOUTS.index(layout))
    t = small_scan(rng, R.GROUPS[group], layout)
    for outer in (None, (900, 7)):
        pl = R.window_plan(t, outer)
        ids, rn = R.window_rows(t, outer)
        rows = t.index_of(ids)
        ref = [make_column(c.tuple_id, c.slot_id, c.prim_type, c.values[rows], None if c.valid is None else c.valid[rows]) for c in t.cols]
        assert window_oracle.assert_matches(ref + [make_column(R.WT, 1, T.INT64, rn)], pl, t.cols) == len(ids)


@pytest.mark.parametrize("layout", R.LAYOUTS)
@pytest.mark.parametrize("group", list(R.GROUPS))
def test_oracle_agrees_on_joins(group, layout):
    rng = np.random.default_rng(30 + R.LAYOUTS.index(layout))
    b, p = small_join(rng, R.GROUPS[group], layout, nans=False)
    for jt in R.JOIN_TYPES[:3]:   # (the row oracle has no FULL join: its rows are the union of LEFT's and RIGHT's, checked here)
        got = oracle.execute(R.join_rows_plan(b, p, jt).serialize(), b.cols + p.cols).columns
        pi, bi = R.join_rows(b, p, jt)
        R.assert_rows(got, [(p, pi), (b, bi)], ordered=False, what=f"oracle {jt}")
    for args in R.arg_chunks(b.payloads() + p.payloads()):
        got = oracle.execute(R.join_agg_plan(b, p, "LEFT_JOIN", args).serialize(), b.cols + p.cols).columns
        R.assert_agg(got, R.join_agg_reference(b, p, "LEFT_JOIN", args), f"0_{R.GRP}", args, what="oracle LEFT")
    b, p = small_join(rng, R.GROUPS[group], layout, unique=True, nans=False)
    for args in R.arg_chunks(b.payloads()):
        got = oracle.execute(R.join_agg_plan(b, p, "INNER_JOIN", args).serialize(), b.cols + p.cols).columns
        R.assert_agg(got, R.join_agg_reference(b, p, "INNER_JOIN", args), f"0_{R.GRP}", args, what="oracle FK-PK")


@pytest.mark.parametrize("group", list(R.GROUPS))
def test_oracle_agrees_on_the_star_join(group):
    rng = np.random.default_rng(40)
    fact, dims = R.star_tables(rng, R.GROUPS[group], nf=3_000)
    for args in R.arg_chunks(R.star_args(fact, dims)):
        got = oracle.execute(R.star_plan(fact, dims, args).serialize(), fact.cols + dims[0].cols + dims[1].cols).columns
        R.assert_agg(got, R.star_reference(fact, dims, args), f"0_{R.GRP}", args, what="oracle star")

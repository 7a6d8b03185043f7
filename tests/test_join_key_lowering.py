"""The join-key matrix of tests/test_gpu_join_keys.py on the host alone: every plan it builds lowers with the expected kind and key cast
(bkgpu_plan_explain parses, type-infers and lowers without a device), every key pair the reference compares as strings is refused, and
the oracle's result for each case on a small table equals a plain Python enumeration of the joined rows."""
import numpy as np
import pytest

from baikaldb_b200 import _lib
from baikaldb_b200.column import rows_as_set
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests.join_key_cases import (AT, PAIRS, REFUSED, Dim, agg_plan, cast_of, fused_plan, group_keys, index_mode, make_case, make_dim,
                                  pair_id, reference)
from tests.test_gpu_join_keys import (DUP_TYPES, EXPECTED, NOTHING, dense_keys, dup_dim, made_dense, mode_keys, nothing_case,
                                      rejects_all)


def explain(plan):
    return _lib.explain(plan.serialize())


def assert_two_table(plan, dim: Dim):
    """PK_JOIN_AGG over the dimension's key column and the fact's foreign key, each with its own type (the two-table explain text
    does not print the cast: its key columns' types are what it shows)"""
    text = explain(plan)
    assert text.startswith("kind=4 scan_tuple=0"), text
    assert f"= {dim.tid}_1 prim={int(dim.key_type)}\n" in text and f"= 0_{10 + dim.tid} prim={int(dim.fk_type)}\n" in text, text


def assert_star(plan, dims, conjuncts=()):
    text = explain(plan)
    assert text.startswith("kind=6 scan_tuple=0") and f"star: fact tuple=0 dims={len(dims)}\n" in text, text
    for d in dims:
        want = f"tuple={d.tid} key={d.tid}_1 fk=0_{10 + d.tid} cast={int(cast_of(d.key_type, d.fk_type))} build_conjuncts={int(d.tid in conjuncts)}\n"
        assert want in text, (want, text)


def assert_oracle(case, grouped=True, dim_ok=None, leaf=None):
    """the oracle against a Python enumeration of the joined rows: COUNT(*), SUM(row id), SUM(value) and every dimension aggregate"""
    want = reference(case, grouped, dim_ok)
    got = oracle.execute(agg_plan(case.dims, grouped, leaf).serialize(), case.all_columns()).columns
    rows = rows_as_set(got, group_keys(case.dims) if grouped else [])
    names = [c.name for c in got]
    if not grouped and not want:   # no joined row: one row, COUNT(*) = 0 and every other aggregate NULL
        (row,) = rows.values()
        assert row[names.index(f"{AT}_1")] == 0 and all(row[names.index(f"{AT}_{k}")] is None for k in range(2, 4 + 3 * len(case.dims)) if f"{AT}_{k}" in names)
        return
    assert set(rows) == set(want)
    fns = [(j, f) for j in range(len(case.dims)) for f in (("sum", "min", "max") if len(case.dims) <= 3 else ("sum", "min" if j % 2 else "max"))]
    for k, w in want.items():
        row = rows[k]
        assert [row[names.index(f"{AT}_{s}")] for s in (1, 2, 3)] == [w[0], w[1], w[2]], k
        for s, (j, f) in enumerate(fns, start=4):
            assert row[names.index(f"{AT}_{s}")] == w[3 + 3 * j + ("sum", "min", "max").index(f)], (k, s)


# ---------------------------------------------------------------- a. the key-type matrix
@pytest.mark.parametrize("pair", PAIRS, ids=pair_id)
def test_two_table_key_types_lower_and_run_on_the_oracle(pair):
    rng = np.random.default_rng(10 + PAIRS.index(pair))
    dim = make_dim(rng, 1, *pair, 60)
    assert_two_table(agg_plan([dim]), dim)
    assert_two_table(fused_plan(dim), dim)
    assert_oracle(make_case(rng, [dim], 400))


@pytest.mark.parametrize("i", range(len(PAIRS)), ids=[pair_id(p) for p in PAIRS])
def test_star_key_types_lower_and_run_on_the_oracle(i):
    rng = np.random.default_rng(20 + i)
    pairs = [PAIRS[i], PAIRS[(i + 7) % len(PAIRS)], PAIRS[(i + 12) % len(PAIRS)]]
    dims = [make_dim(rng, d, dk, fk, 20 + 10 * d, null_keys=0.05) for d, (dk, fk) in enumerate(pairs, start=1)]
    assert_star(agg_plan(dims), dims)
    assert_oracle(make_case(rng, dims, 300))
    dense = [make_dim(rng, d, dk, fk, 40, keys=dense_keys(dk, fk, 40)) for d, (dk, fk) in enumerate(pairs, start=1)]
    assert all(index_mode(d) == "dense" for d in dense)
    assert_oracle(make_case(rng, dense, 300))


@pytest.mark.parametrize("pair", REFUSED, ids=pair_id)
def test_key_pairs_compared_as_strings_are_refused(pair):
    """signed with unsigned, DATE with DATETIME or an integer, BOOL with an integer, FLOAT / DOUBLE and STRING keys: never lowered"""
    dk, fk = pair
    one = Dim(1, dk, fk, [])
    star = [Dim(1, T.INT32, T.INT32, []), Dim(2, dk, fk, []), Dim(3, T.INT64, T.INT32, [])]
    for plan in (agg_plan([one]), agg_plan(star), agg_plan(star, grouped=False)):
        with pytest.raises(_lib.BkgpuError) as e:
            explain(plan)
        assert e.value.code == _lib.EUNSUPPORTED, e.value
        assert "STRING" in str(e.value) or "join key type" in str(e.value), e.value


# ---------------------------------------------------------------- b. to e.: the star edges
@pytest.mark.parametrize("kt", [T.INT32, T.INT64], ids=["INT32", "INT64"])
@pytest.mark.parametrize("name", list(EXPECTED))
def test_index_mode_cases_lower_and_select_their_mode(name, kt):
    rng = np.random.default_rng(30)
    dim = make_dim(rng, 1, kt, kt, 1000, keys=mode_keys(rng, name, kt))
    assert index_mode(dim) == EXPECTED[name][kt == T.INT64]
    other = make_dim(rng, 2, T.INT32, T.INT32, 400, keys=[int(x) for x in rng.permutation(400)])
    assert_star(agg_plan([dim, other]), [dim, other])
    assert_two_table(agg_plan([dim]), dim)
    small = Dim(1, kt, kt, dim.keys[:50])
    case = make_case(rng, [small, Dim(2, T.INT32, T.INT32, other.keys[:50])], 200)
    assert_oracle(case)
    assert_oracle(made_dense(case, 1))


@pytest.mark.parametrize("kt", [T.INT32, T.INT64], ids=["INT32", "INT64"])
@pytest.mark.parametrize("what", NOTHING)
def test_dimensions_that_contribute_nothing_lower_and_run_on_the_oracle(what, kt):
    case = nothing_case(np.random.default_rng(40), what, kt, n=300)
    conj = what == "rejected_by_its_conjunct"
    leaf, dim_ok = (rejects_all, lambda d, r: d.tid != 2) if conj else (None, None)
    assert_star(agg_plan(case.dims, leaf=leaf), case.dims, conjuncts=(2,) if conj else ())
    assert_oracle(case, True, dim_ok, leaf)
    if what != "one_row_every_partner":
        assert not reference(case, True, dim_ok)
        assert_oracle(case, False, dim_ok, leaf)


@pytest.mark.parametrize("n_dup", [2, 4])
def test_duplicate_key_stars_lower_and_run_on_the_oracle(n_dup):
    rng = np.random.default_rng(50 + n_dup)
    dims = [dup_dim(rng, d, dk, fk) if d <= n_dup else make_dim(rng, d, dk, fk, 50, keys=dense_keys(dk, fk, 50)) for d, (dk, fk) in enumerate(DUP_TYPES, start=1)]
    assert_star(agg_plan(dims), dims)
    assert_oracle(make_case(rng, dims, 40, miss=0.05, null=0.05))

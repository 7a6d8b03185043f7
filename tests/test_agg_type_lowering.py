"""The aggregate-type matrix of tests/test_gpu_agg_types.py on the host alone: every GROUP BY key and aggregate argument type lowers to
the direct kernel with the reference's output types (bkgpu_plan_explain parses, type-infers and lowers without a device), the oracle
equals the reference of tests/agg_type_cases.py bit for bit on every case, and filter literals at and past a narrow type's range take
the reference's typing."""
import re

import numpy as np
import pytest

from baikaldb_b200 import _lib, plan as P
from baikaldb_b200.plan import PrimitiveType as T
from oracle import oracle
from tests.agg_type_cases import (AVG_FNS, FLOATS, FNS, main_fns, TYPES, Table, agg_plan, assert_matches, column_array, key_table, out_type, reference, tname,
                                  value_table)
from tests.test_gpu_agg_types import LITERAL_CASES, filter_reference, filter_table, literal_plan


def explain(plan):
    return _lib.explain(plan.serialize())


def out_prims(text):
    return [int(x) for x in re.findall(r"agg\[\d+\] kind=\d+ .* out_prim=(\d+)", text)]


def run_oracle(t: Table, fns=FNS, **kw):
    got = oracle.execute(agg_plan(t, fns, **kw).serialize(), t.columns()).columns
    assert_matches(got, reference(t, fns), t.kt if t.grouped else None, what="oracle")


@pytest.mark.parametrize("kt", TYPES, ids=tname)
def test_key_types_lower_to_the_direct_kernel_and_match_on_the_oracle(kt):
    rng = np.random.default_rng(100 + int(kt))
    t = key_table(rng, kt, 1_203, key_nulls=0.05, value_nulls=0.1)
    text = explain(agg_plan(t))
    assert "direct=1" in text, text
    assert out_prims(text) == [out_type(f, T.DOUBLE) for f in FNS], text
    run_oracle(t)
    run_oracle(key_table(rng, kt, 1_001, vt=T.INT64), main_fns(T.INT64))


@pytest.mark.parametrize("vt", TYPES, ids=tname)
def test_argument_types_lower_with_their_output_types_and_match_on_the_oracle(vt):
    """SUM(UINT8) -> UINT64, SUM(INT8) / SUM(BOOL) / SUM(DATE) -> INT64, SUM(FLOAT) -> DOUBLE, MIN / MAX keep the argument's type, AVG
    -> DOUBLE (AggFnCall::type_inferer, agg_fn_call.cpp:87-122)"""
    rng = np.random.default_rng(200 + int(vt))
    t = value_table(rng, vt, 2_003)
    for fns in (main_fns(vt), AVG_FNS):
        for grouped in (True, False):
            text = explain(agg_plan(t, fns, grouped=grouped))
            assert "direct=1" in text, text
            assert out_prims(text) == [out_type(f, vt) for f in fns], text
        run_oracle(t, fns)
        run_oracle(value_table(rng, vt, 1_001, grouped=False), fns)


def test_bool_against_a_literal_is_not_lowered():
    """`bool = 2` (or = TRUE): two BOOL operands are neither integers nor dates nor doubles to FunctionManager::complete_fn
    (fn_manager.cpp:316-409), so the reference compares them as strings, which the lowering refuses"""
    t, _ = filter_table(np.random.default_rng(1), T.BOOL, 10)
    for lit in (2, 1):
        with pytest.raises(_lib.BkgpuError) as e:
            explain(literal_plan(t, T.BOOL, "eq", lit))
        assert e.value.code == _lib.EUNSUPPORTED and "STRING" in str(e.value), e.value


@pytest.mark.parametrize("case", LITERAL_CASES, ids=lambda c: c[0])
def test_filter_literals_at_and_past_a_narrow_range(case):
    """the literal takes the column's type before the comparison (see LITERAL_CASES); the oracle's rows are the ones that model passes"""
    name, ft, op, lit, rule = case
    rng = np.random.default_rng(300 + LITERAL_CASES.index(case))
    t, fcol = filter_table(rng, ft, 1_003)
    plan = literal_plan(t, ft, op, lit)
    assert "direct=1" in explain(plan), explain(plan)
    got = oracle.execute(plan.serialize(), t.columns() + [fcol]).columns
    assert_matches(got, filter_reference(t, fcol, ft, op, lit), t.kt, what="oracle")

"""CPU: select_agg_launch (csrc/agg_select.cpp) sends every plan with hll_add_agg to k_agg_interp with no shared table, whatever the batch
offers the lean and direct kernels: a sketch lives in the global table's register arena.  Driven through tests/cpp/agg_select_check.cpp."""
import pytest

from baikaldb_b200.plan import PrimitiveType as T
from tests import hll_cases as C
from tests.test_agg_select import select  # noqa: F401  (the driver fixture)


@pytest.mark.parametrize("name,plan", [("grouped", C.scan_plan(T.INT32)), ("scalar", C.scan_plan(T.DOUBLE, grouped=False)),
                                       ("beside COUNT / SUM / AVG", C.scan_plan(T.INT64, extra=True)), ("two sketches", C.two_sketch_plan()),
                                       ("MERGE_AGG", C.merge_plan()), ("scalar MERGE_AGG", C.merge_plan(False))])
@pytest.mark.parametrize("args", [{}, {"known_groups": 100}, {"smem_cap_log2": 8}, {"valid": "0_2"}, {"vec_ok": 0}])
def test_hll_plans_take_the_interpreter_without_a_shared_table(select, name, plan, args):  # noqa: F811
    if "valid" in args and "MERGE" in name:
        args = {"valid": "9_1"}
    r = select(plan, **args)
    assert (r["rc"], r["kernel"], r["name"], r["smem"], r["smem_cap_log2"], r["fused_ok"], r["lean"]) == ("0", "INTERP", "k_agg_interp", "0", "0", "0", "0"), r

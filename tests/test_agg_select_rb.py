"""CPU: select_agg_launch (csrc/agg_select.cpp) sends every plan with rb_build_agg to k_agg_interp with no shared table, whatever the
batch offers the lean and direct kernels: a pair key names the group's slot in the global table.  Driven through
tests/cpp/agg_select_check.cpp."""
import pytest

from baikaldb_b200.plan import PrimitiveType as T
from tests import rb_cases as C
from tests.test_agg_select import select  # noqa: F401  (the driver fixture)


@pytest.mark.parametrize("name,plan", [("grouped", C.scan_plan(T.INT32)), ("scalar", C.scan_plan(T.INT64, grouped=False)),
                                       ("beside COUNT / SUM / COUNT", C.scan_plan(T.INT64, extra=True)), ("four bitmaps", C.many_plan(4)),
                                       ("BOOL", C.scan_plan(T.BOOL)), ("UINT64", C.scan_plan(T.UINT64, grouped=False))])
@pytest.mark.parametrize("args", [{}, {"known_groups": 100}, {"smem_cap_log2": 8}, {"valid": "0_2"}, {"vec_ok": 0}, {"force_generic": 1}])
def test_rb_plans_take_the_interpreter_without_a_shared_table(select, name, plan, args):  # noqa: F811
    r = select(plan, **args)
    assert (r["rc"], r["kernel"], r["name"], r["smem"], r["smem_cap_log2"], r["fused_ok"], r["lean"]) == ("0", "INTERP", "k_agg_interp", "0", "0", "0", "0"), r

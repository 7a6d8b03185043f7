"""CPU: the choice of the aggregate kernel for a batch (csrc/agg_select.cpp) and the AggArgs fields it fills, through the driver
tests/cpp/agg_select_check.cpp (plan descriptor + fake device columns, no CUDA calls).  The expected values are those of the code
that made the choice inside launch_agg_batch / launch_agg / launch_direct before it moved behind select_agg_launch."""
import os
import subprocess

import pytest

from baikaldb_b200 import plan as P, queries
from baikaldb_b200.plan import PlanNodeType, PrimitiveType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def select(tmp_path_factory):
    d = tmp_path_factory.mktemp("agg_select")
    exe = str(d / "agg_select_check")
    csrc = os.path.join(ROOT, "csrc")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-Wextra", "-I", csrc, "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include",
                           os.path.join(ROOT, "tests", "cpp", "agg_select_check.cpp"), os.path.join(csrc, "agg_select.cpp"),
                           os.path.join(csrc, "plan.cpp"), os.path.join(csrc, "literal.cpp"), "-o", exe])

    def run(plan, **args):
        path = d / "plan.bin"
        path.write_bytes(plan.serialize())
        out = subprocess.run([exe, str(path)] + [f"{k}={v}" for k, v in args.items()], capture_output=True, text=True, timeout=60)
        assert out.returncode == 0, out.stderr
        return dict(line.split("=", 1) for line in out.stdout.split())
    return run


def min_max_plan():
    """the shape of test_gpu_agg.py::test_lean_kernel_min_max_and_several_aggregates_per_column"""
    d, i64, u64, e = P.slot_ref(0, 3, T.DOUBLE), P.slot_ref(0, 4, T.INT64), P.slot_ref(0, 5, T.UINT64), P.slot_ref(0, 6, T.DOUBLE)
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("min", 1, 2, None, d), P.agg_expr("max", 1, 3, None, d), P.agg_expr("sum", 1, 4, None, d),
            P.agg_expr("max", 1, 5, None, i64), P.agg_expr("sum", 1, 6, None, i64), P.agg_expr("min", 1, 7, None, u64), P.agg_expr("count", 1, 8, None, e),
            P.agg_expr("avg", 1, 9, 10, d)]
    root = P.agg(P.where(P.scan(0), P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(70))), 1, [P.slot_ref(0, 1, T.INT32)], aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE), (4, T.INT64), (5, T.UINT64), (6, T.DOUBLE)],
                         1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE, T.DOUBLE, T.INT64, T.INT64, T.UINT64, T.DOUBLE, T.DOUBLE])})


def int64_key_plan():
    """the shape of test_gpu_agg.py::test_lean_int64_key_and_integer_sums"""
    aggs = [P.agg_expr("count_star", 1, 1), P.agg_expr("sum", 1, 2, None, P.slot_ref(0, 3, T.DOUBLE)),
            P.agg_expr("sum", 1, 3, None, P.slot_ref(0, 4, T.INT64)), P.agg_expr("avg", 1, 4, 5, P.slot_ref(0, 3, T.DOUBLE))]
    root = P.agg(P.where(P.scan(0), P.ge(P.slot_ref(0, 1, T.INT32), P.int_lit(-50)), P.ne(P.slot_ref(0, 1, T.INT32), P.int_lit(7))), 1,
                 [P.slot_ref(0, 2, T.INT64)], aggs)
    return P.Plan(root, {0: [(1, T.INT32), (2, T.INT64), (3, T.DOUBLE), (4, T.INT64)], 1: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.INT64, T.DOUBLE])})


def scalar_sum_plan():
    aggs = [P.agg_expr("sum", 1, 1, None, P.slot_ref(0, 3, T.DOUBLE))]
    root = P.agg(P.where(P.scan(0), P.lt(P.slot_ref(0, 2, T.INT32), P.int_lit(1 << 19))), 1, [], aggs)
    return P.Plan(P.packet(root), {0: [(1, T.INT32), (2, T.INT32), (3, T.DOUBLE), (4, T.DOUBLE)], 1: P.agg_tuple_slots(aggs, [T.DOUBLE])})


def c3_min_max_plan():
    aggs = [P.agg_expr("count_star", 2, 1), P.agg_expr("sum", 2, 2, None, P.slot_ref(0, 2, T.DOUBLE)), P.agg_expr("min", 2, 3, None, P.slot_ref(0, 2, T.DOUBLE))]
    j = P.join(P.scan(1), P.scan(0), [P.eq(P.slot_ref(1, 1, T.INT32), P.slot_ref(0, 1, T.INT32))])
    return P.Plan(P.agg(j, 2, [P.slot_ref(1, 2, T.INT32)], aggs), {0: [(1, T.INT32), (2, T.DOUBLE)], 1: [(1, T.INT32), (2, T.INT32)],
                                                                    2: P.agg_tuple_slots(aggs, [T.INT64, T.DOUBLE, T.DOUBLE])})


def c2_with(above):
    """C2 with a HAVING or a SORT above the aggregate: the plan gets a post fragment"""
    pl = queries.c2_filter_groupby()
    if above == "having":
        root = P.where(pl.root, P.gt(P.slot_ref(1, 1, T.INT64), P.int_lit(3)), node_type=PlanNodeType.HAVING_FILTER_NODE)
    else:
        root = P.limit(P.sort(pl.root, [P.slot_ref(0, 1, T.INT32)], [True], tuple_id=1), 10)
    return P.Plan(root, pl.tuples)


# ---- C1: COUNT(*) WHERE int32 < c ----
@pytest.mark.parametrize("args,kernel,name", [
    ({}, "COUNT_WHERE_TMA", "k_count_where_tma"),
    ({"scalar_tma": 0}, "SCALAR_DIRECT", "k_agg_scalar_direct"),
    ({"valid": "0_1"}, "SCALAR_DIRECT", "k_agg_scalar_direct"),
    ({"offset": "0_1:4"}, "SCALAR_DIRECT", "k_agg_scalar_direct"),
    ({"offset": "0_1:16"}, "COUNT_WHERE_TMA", "k_count_where_tma"),
    ({"vec_ok": 0}, "INTERP", "k_agg_interp"),
])
def test_c1(select, args, kernel, name):
    r = select(queries.c1_count_where(), **args)
    assert (r["rc"], r["kernel"], r["name"], r["smem"], r["fused_ok"]) == ("0", kernel, name, "0", "0")


# ---- C2: GROUP BY one int32 key, SUM + AVG of doubles ----
def test_c2_default_is_fx_with_its_lane_layout(select):
    r = select(queries.c2_filter_groupby())
    assert (r["kernel"], r["name"]) == ("LEAN_FX", "k_agg_group_lean_fx")
    # {rows, -, sumA, -, sumB}: the two double sums share a 16-byte pair; the extension limbs sit behind table and queues
    assert (r["smem_cap_log2"], r["n_smem_lanes"], r["smem_lane"]) == ("11", "4", "0,-1,2,-1,3")
    assert (r["lean_fx"], r["fx_ext_off"], r["smem"]) == ("1", str(174592), str(174592 + 2 * 4 * 2048))
    assert r["fused_ok"] == "1"


@pytest.mark.parametrize("args,kernel", [
    ({"lean_fx": 0}, "LEAN"),
    ({"fx_off": 1}, "LEAN"),
    ({"nrows": 1 << 31}, "LEAN"),
    ({"nrows": (1 << 31) - 1}, "LEAN_FX"),
    ({"fx_off": 1, "known_groups": 1000}, "LEAN"),
    ({"lean_fx": 0, "known_groups": 1000}, "LEAN"),
    ({"no_lean": 1}, "GROUP_DIRECT"),
    ({"force_generic": 1}, "INTERP"),
    ({"vec_ok": 0}, "INTERP"),
])
def test_c2_variants(select, args, kernel):
    r = select(queries.c2_filter_groupby(), **args)
    assert r["kernel"] == kernel
    assert r["lean_fx"] == ("1" if kernel == "LEAN_FX" else "0")
    if kernel.startswith("LEAN"):
        assert (r["name"], r["smem_cap_log2"], r["n_smem_lanes"], r["smem_lane"], r["fused_ok"]) == (
            "k_agg_group_lean_fx" if kernel == "LEAN_FX" else "k_agg_group_lean", "11", "4", "0,-1,2,-1,3", "1")
    else:
        assert r["fused_ok"] == "0"


@pytest.mark.parametrize("valid,args,kernel", [
    ("0_3", {}, "LEAN_NULLS"),
    ("0_3,0_4", {}, "LEAN_NULLS"),
    ("0_2", {}, "LEAN_NULLS"),
    ("0_3", {"no_lean_nulls": 1}, "GROUP_DIRECT"),
    ("0_2", {"no_lean_nulls": 1}, "GROUP_DIRECT"),
    ("0_1", {}, "GROUP_DIRECT"),
])
def test_c2_with_nulls(select, valid, args, kernel):
    r = select(queries.c2_filter_groupby(), valid=valid, **args)
    assert (r["kernel"], r["lean_fx"]) == (kernel, "0")


def test_c2_null_value_columns_get_shared_counters(select):
    r = select(queries.c2_filter_groupby(), valid="0_3,0_4")
    # lanes 1 and 3 count the non-NULL inputs of SUM(0_3) and AVG(0_4): with NULLs they join the shared table behind the sums
    assert (r["n_smem_lanes"], r["smem_lane"]) == ("6", "0,4,2,5,3")


@pytest.mark.parametrize("args,kernel", [({}, "LEAN_MM"), ({"valid": "0_3,0_4"}, "LEAN_MM"), ({"no_lean_mm": 1}, "GROUP_DIRECT")])
def test_min_max_shape(select, args, kernel):
    r = select(min_max_plan(), **args)
    assert (r["kernel"], r["name"] if kernel == "LEAN_MM" else "k_agg_group_lean") == (kernel, "k_agg_group_lean")


def test_int64_key_takes_lean_fx(select):
    r = select(int64_key_plan())
    assert (r["kernel"], r["lean_fx"], r["smem_cap_log2"]) == ("LEAN_FX", "1", "11")


def test_scalar_sum_of_doubles(select):
    r = select(scalar_sum_plan())
    assert (r["kernel"], r["name"], r["smem"]) == ("SCALAR_DIRECT", "k_agg_scalar_direct", "0")


# ---- the shared table's capacity ----
@pytest.mark.parametrize("args,log2,kernel", [
    ({"known_groups": 0}, "11", "LEAN_FX"),
    ({"known_groups": 1000}, "11", "LEAN_FX"),
    ({"known_groups": 2000}, "11", "LEAN_FX"),
    ({"known_groups": 3000}, "0", "GROUP_DIRECT"),
    ({"known_groups": 100000}, "0", "GROUP_DIRECT"),
    ({"smem_cap_log2": 8}, "8", "LEAN_FX"),
    ({"smem_cap_log2": 4, "known_groups": 100000}, "4", "LEAN_FX"),
    ({"smem_cap_log2": 14}, "11", "LEAN_FX"),
    ({"smem_cap_log2": 0}, "0", "GROUP_DIRECT"),
])
def test_shared_table_size(select, args, log2, kernel):
    r = select(queries.c2_filter_groupby(), **args)
    assert (r["smem_cap_log2"], r["kernel"]) == (log2, kernel)


# ---- C3: the FK -> PK probe fused into the lean kernel ----
def test_c3_fused_probe(select):
    r = select(queries.c3_join_groupby(), fused=1)
    assert (r["rc"], r["kernel"], r["name"], r["fused_ok"]) == ("0", "LEAN_FX_JOIN", "k_agg_group_lean_fx", "1")
    assert select(queries.c3_join_groupby(), fused=1, lean_fx=0)["kernel"] == "LEAN_JOIN"


@pytest.mark.parametrize("plan,args", [(queries.c3_join_groupby, {"valid": "0_2"}), (c3_min_max_plan, {}), (queries.c3_join_groupby, {"no_lean": 1})])
def test_c3_fused_probe_refuses(select, plan, args):
    assert select(plan(), fused=1, **args)["rc"] == "1"


def test_c3_general_probe_is_the_interpreter(select):
    assert select(queries.c3_join_groupby())["kernel"] == "INTERP"


# ---- the lean kernel's own result extraction ----
@pytest.mark.parametrize("plan,args,fused", [
    (queries.c2_filter_groupby, {}, "1"),
    (queries.c2_filter_groupby, {"multi_rank": 1}, "0"),
    (lambda: c2_with("having"), {}, "0"),
    (lambda: c2_with("sort"), {}, "0"),
    (queries.c2_filter_groupby, {"force_generic": 1}, "0"),
    (queries.c2_filter_groupby, {"no_lean": 1}, "0"),
])
def test_fused_extraction(select, plan, args, fused):
    assert select(plan(), **args)["fused_ok"] == fused


def test_lean_table_that_does_not_fit_is_an_error(select):
    """the general kernel's layout fits 2^11 slots for 1,000 groups, the lean layout (with the non-NULL counters) fits none"""
    assert select(min_max_plan(), known_groups=1000, valid="0_3,0_4")["rc"] == "-4"
    assert select(min_max_plan(), known_groups=1000)["kernel"] == "LEAN_MM"

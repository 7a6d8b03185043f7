// The C++ side of APPLY plans (host/bkgpu_host.hpp's writer, host/bkgpu_dictionary.hpp's adapter), printed for tests/test_apply_plan.py to
// compare with plan.py / dictionary.py:
//   line 1: an EXISTS plan (AGG -> FILTER -> APPLY(SEMI)) as hex
//   line 2: an APPLY with every flag set (max_one_row, compare_type ALL, is_select_field) as hex
//   line 3: an IN over STRING columns (APPLY condition 1_1 = 0_1) rewritten to dictionary codes, as hex
//   line 4, 5: the code columns of 1_1 and 0_1 (-1 = NULL)
//   g++ -std=c++17 -I include -I host tests/cpp/apply_plan_check.cpp
#include <stdio.h>
#include "bkgpu_dictionary.hpp"
using namespace bkgpu;

static void hex(const std::vector<uint8_t>& b) {
    for (uint8_t x : b) printf("%02x", x);
    printf("\n");
}
static PlanNode node(int type, std::vector<PlanNode> ch = {}) { PlanNode n; n.node_type = type; n.children = std::move(ch); return n; }
static PlanNode scan(int tuple) { PlanNode n = node(BK_SCAN_NODE); n.tuple_id = tuple; return n; }
static Expr eq(Expr a, Expr b) { return Expr::fn(BK_FT_EQ, "eq", {std::move(a), std::move(b)}); }

int main() {
    PlanNode sub = node(BK_WHERE_FILTER_NODE, {scan(0)});
    sub.conjuncts = {eq(Expr::slot_ref(0, 1, BK_INT32), Expr::slot_ref(1, 1, BK_INT32)),
                     Expr::fn(BK_FT_LT, "lt", {Expr::slot_ref(0, 3, BK_INT32), Expr::int_literal(7)})};
    PlanNode apply = node(BK_APPLY_NODE, {scan(1), sub});
    apply.join_type = BK_SEMI_JOIN;
    PlanNode above = node(BK_WHERE_FILTER_NODE, {apply});
    above.conjuncts = {Expr::fn(BK_FT_GT, "gt", {Expr::slot_ref(1, 2, BK_INT32), Expr::int_literal(1)})};
    PlanNode agg = node(BK_AGG_NODE, {above});
    agg.agg_tuple_id = 2;
    agg.group_exprs = {Expr::slot_ref(1, 2, BK_INT32)};
    agg.agg_fn_calls = {Expr::agg("count_star", 2, 1, 1, {})};
    Plan p;
    p.tuples = {{0, {{1, BK_INT32}, {2, BK_DOUBLE}, {3, BK_INT32}, {4, BK_INT64}}}, {1, {{1, BK_INT32}, {2, BK_INT32}, {3, BK_DOUBLE}, {4, BK_INT64}}},
                {2, {{1, BK_INT64}}}};
    p.root = agg;
    hex(p.serialize());

    Plan flags = p;
    PlanNode& a = flags.root.children[0].children[0];
    a.join_type = BK_LEFT_JOIN; a.max_one_row = true; a.compare_type = BK_CMP_ALL; a.is_select_field = true;
    a.conjuncts = {eq(Expr::slot_ref(1, 4, BK_INT64), Expr::slot_ref(0, 4, BK_INT64))};
    hex(flags.serialize());

    // IN (SELECT s FROM t0 WHERE ...) over STRING columns: the condition's two columns share one dictionary
    PlanNode in_apply = node(BK_APPLY_NODE, {scan(1), scan(0)});
    in_apply.join_type = BK_SEMI_JOIN;
    in_apply.conjuncts = {eq(Expr::slot_ref(1, 1, BK_STRING), Expr::slot_ref(0, 1, BK_STRING))};
    PlanNode sagg = node(BK_AGG_NODE, {in_apply});
    sagg.agg_tuple_id = 2;
    sagg.group_exprs = {Expr::slot_ref(1, 2, BK_INT32)};
    sagg.agg_fn_calls = {Expr::agg("count_star", 2, 1, 1, {})};
    Plan sp;
    sp.tuples = {{0, {{1, BK_STRING}}}, {1, {{1, BK_STRING}, {2, BK_INT32}}}, {2, {{1, BK_INT64}}}};
    sp.root = sagg;
    std::vector<StringColumn> cols = {{1, 1, {std::string("pear"), std::string("apple"), std::nullopt, std::string("fig")}},
                                      {0, 1, {std::string("apple"), std::string("kiwi"), std::string("fig"), std::nullopt, std::string("fig")}}};
    EncodedStrings enc = encode_strings(sp, cols);
    hex(enc.plan.serialize());
    for (auto& c : enc.columns) {
        for (int64_t r = 0; r < c.length; r++) {
            const bool valid = c.validity.empty() || ((c.validity[(size_t)(r >> 3)] >> (r & 7)) & 1);
            printf("%s%d", r ? " " : "", valid ? c.at<int32_t>(r) : -1);
        }
        printf("\n");
    }
    return 0;
}

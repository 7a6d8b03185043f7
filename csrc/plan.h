// plan.h — host side: parse the plan word stream (include/bkgpu_plan.h), run the reference's type
// inference, and lower the operator subtree to device programs.  Pure C++, no CUDA calls, so
// bkgpu_plan_explain() works on a machine without a GPU.
#pragma once
#include <stdint.h>
#include <memory>
#include <string>
#include <vector>
#include "dev_types.h"
#include "../include/bkgpu_plan.h"

namespace bk {

struct HExpr {
    int node_type = 0, col_type = 0;
    std::vector<HExpr> ch;
    int tuple_id = 0, slot_id = 0;
    int fn_op = 0;
    std::string name;
    std::vector<int> arg_types;
    int return_type = 0;
    // literal: value image in `lit_prim`
    bool lit_null = false;
    uint64_t lit_bits = 0;
    int lit_prim = 0;
    std::string lit_str;              // STRING literal text (lit_prim == BK_STRING) until type inference folds it into an image
    int final_slot = 0, inter_slot = 0;
    bool distinct = false;            // AGG_EXPR count_distinct / sum_distinct / avg_distinct: name holds the base function
    bool is_constant = false;
};

// WINDOW_NODE frame bound (pb::FrameBound): type BK_BT_*, unbounded flag, optional INT_LITERAL offset
struct HFrameBound { int type = 0; bool unbounded = false; bool has_expr = false; HExpr expr; };

struct HNode {
    int node_type = 0;
    int64_t limit = -1;
    std::vector<HNode> ch;
    int tuple_id = -1;
    std::vector<HExpr> conjuncts;            // filter / join conditions
    int agg_tuple_id = -1;
    std::vector<HExpr> group_exprs, agg_fns; // agg
    std::vector<HExpr> order_exprs;          // sort
    std::vector<int> is_asc, is_null_first;
    int join_type = 0;
    int64_t offset = 0;
    // apply (pb::ApplyNode): join_type and the conditions in conjuncts
    bool max_one_row = false, is_select_field = false;
    int compare_type = 0;
    // window (pb::WindowNode): func_exprs in agg_fns, partition exprs in group_exprs, order exprs + is_asc in order_exprs / is_asc
    bool has_frame = false;
    int frame_type = 0;
    HFrameBound frame_start, frame_end;
};

struct HTuple { int tuple_id; std::vector<std::pair<int, int>> slots; /* (slot_id, prim) */ };

struct ColRef { int tuple_id, slot_id, prim; };

struct OutCol {
    int tuple_id, slot_id, prim;
    int kind;       // 0 = plain value column, 1 = AVG intermediate blob (two device images: sum, count), 2 = HLL sketch (RAW, 16400 bytes;
                    //   one device image: the sketch reference, whose registers the host copies from the arena), 3 = rb_build_agg's BITMAP
                    //   (one device image: the group's slot; the bytes come from the device build, rb.cu)
};

enum PlanKind { PK_AGG = 1, PK_FILTER = 2, PK_SORT = 3, PK_JOIN_AGG = 4, PK_JOIN = 5, PK_STAR_AGG = 6, PK_WINDOW = 7 };

struct SortKey { int out_reg; int prim; bool asc, null_first; };

// one dimension of a star join (PK_STAR_AGG): a table INNER-joined to the fact tuple on one key
struct StarDim {
    int tuple_id = -1;
    int key_col = -1, fk_col = -1;     // indices into Compiled::cols: the dimension's key, the fact tuple's foreign key
    int cast_prim = 0;                 // type both keys are compared in (strip_out_equal_slots' cast, joiner.cpp:166-217)
    int n_filter = 0;                  // conjuncts that read this dimension alone: evaluated once over its rows at build time
    Program filter{};                  // output 0 = their conjunction (column indices into Compiled::cols)
};

// window functions (WindowFnCall::init's name table, window_fn_call.cpp:20-38)
enum WinFnKind { WF_COUNT_STAR = 0, WF_COUNT, WF_SUM, WF_AVG, WF_MIN, WF_MAX, WF_ROW_NUMBER, WF_RANK, WF_DENSE_RANK, WF_PERCENT_RANK,
                 WF_CUME_DIST, WF_NTILE, WF_LEAD, WF_LAG, WF_FIRST_VALUE, WF_LAST_VALUE, WF_NTH_VALUE };
// how an aggregate / value function reads its frame [start, end) on the device
enum WinMethod { WM_NONE = 0,   // ranking, LEAD / LAG: no frame
                 WM_FWD,        // the frame starts at the partition start: a forward scan segmented by partition, read at end - 1
                 WM_BWD,        // the frame ends at the partition end: a backward scan segmented by partition, read at start
                 WM_PEER,       // RANGE CURRENT ROW .. CURRENT ROW: a forward scan segmented by peer group, read at the group's last row
                 WM_DIRECT };   // bounded ROWS frame (<= 4096 rows): each row loops over its frame
struct WinBound { int type = BK_BT_PRECEDING; bool unbounded = true; int64_t num = 0; };
struct WinFn {
    int kind = 0, tuple_id = 0, slot_id = 0;
    int out_prim = 0;                  // result type (WindowFnCall::type_inferer)
    int arg = -1, def = -1;            // indices into WinStage::exprs: the value argument, LEAD / LAG's default
    int arg_prim = 0;                  // type of the argument's image as evaluated (after the cast to the result type)
    int64_t n = 0;                     // NTILE buckets, LEAD / LAG offset, NTH_VALUE position
    int method = WM_NONE;
};
// one WINDOW -> SORT pair.  Every expression is its own one-output device program over the scan columns.
struct WinStage {
    bool new_sort = true;              // false: the SORT's keys equal the previous stage's (a stable re-sort is the identity)
    std::vector<Program> exprs;
    std::vector<int> expr_prim;
    std::vector<SortKey> sort_keys;    // out_reg = index into exprs; partition keys first
    int n_part = 0;                    // the first n_part sort keys are the partition expressions, the rest the order expressions
    bool has_frame = false;
    int frame_type = 0;
    WinBound start, end;
    std::vector<WinFn> fns;
};

// An IN list lowered to OP_IN_SET: the hashed set of its entries (in_set.h), built once per IN expression and shared by every
// program lowered from it (a join's jfast lowers the same conjuncts again).  bkgpu_open uploads all of a plan's sets in one allocation.
struct InSet {
    int vclass = 0;
    bool has_null = false;             // the list held a NULL literal: a miss is NULL
    uint32_t n_distinct = 0;
    std::vector<uint64_t> image;       // the device image: header + slots
};
struct InSets {
    std::vector<InSet> sets;           // index = OP_IN_SET's b
    std::vector<std::pair<const HExpr*, int>> of_expr;   // (IN expression, set index)
};

struct Compiled {
    int kind = 0;
    std::vector<HTuple> tuples;
    // main (probe-side / only) scan
    int scan_tuple = -1;
    std::vector<ColRef> cols;          // columns the device program references (index = DevCol index)
    std::vector<int> col_side;         // per column: 0 = probe / only scan tuple, 1 = build side of a join; star join: 0 = fact, 1 + d = dims[d]
    Program prog;                      // outputs: [predicate][keys...][agg args...] / sort keys
    // aggregate
    AggPlan ap;
    bool is_merge = false, emit_default = false;
    int n_rb = 0;                      // AG_RB aggregates in ap (at most MAX_RB): their keys go to the pair buffer (AggArgs::rb_keys)
    bool has_direct = false;
    DirectPlan direct;
    std::vector<int> direct_cols;      // indices into `cols`, in [terms][key][values] order
    std::vector<int> arg_cols_mask;    // per aggregate: bitmask of cols its argument reads (nullability per batch)
    std::vector<bool> arg_can_null;    // per aggregate: NULL possible even when all its columns are valid
    std::vector<OutCol> out_cols;
    int64_t agg_limit = -1;
    // filter-only / sort: rows of the scan tuple are returned
    int64_t limit = -1, offset = 0;
    std::vector<SortKey> sort_keys;
    // hash join (build side = outer child, probe side = inner child; join_node.cpp:920-1022)
    int build_tuple = -1;
    int build_key_col = -1;            // index into cols (side 1)
    int probe_key_col = -1;            // index into cols
    int join_type = 0;
    int join_key_prim = 0;
    // LEFT / SEMI / ANTI_SEMI over filtered children: each child's own filter, apart from the join conditions (a build row that fails it must
    // not exist, not even in the tail).  Output 0 = the conjunction of that child's n_*_filter conjuncts (column indices into cols).
    int n_build_filter = 0, n_probe_filter = 0;
    Program build_filter{}, probe_filter{};
    // an APPLY (correlated subquery) lowered as the SEMI / ANTI_SEMI join above: its join type (0 = no APPLY), the conjuncts moved from the
    // subquery's filters into the join conditions, the conjuncts of the filter above it folded into the outer child's filter (explain only)
    int apply_join_type = 0, apply_moved = 0, apply_folded = 0;
    // FK -> PK fast path: the same aggregate lowered over the virtual joined tuple (build-side columns are gathered
    // to probe-row alignment first); usable while every probe row has exactly one match
    std::shared_ptr<Compiled> jfast;
    std::vector<int> jfast_of_main;    // for every column of jfast->cols: index of the same column in this->cols
    // star join (PK_STAR_AGG): scan_tuple is the fact tuple; the aggregate runs as `jfast` over fact and dimension columns gathered side by side
    std::vector<StarDim> dims;
    // operators ABOVE the aggregate ([LIMIT ->] [SORT ->] [HAVING ->] AGG, exec_node.cpp:347-394): a second, small fragment of kind
    // PK_SORT / PK_FILTER whose "scan tuple" is the aggregate's output row (its columns = this->out_cols, in order)
    std::shared_ptr<Compiled> post;
    // window (PK_WINDOW): the stages bottom-up; the output rows are the scan tuple's slots (out_cols) followed by one column per window
    // function, in the topmost stage's sort order.  `post` (kind PK_SORT), when present, is the query's ORDER BY over those rows.
    std::vector<WinStage> win;
    // the plan's IN sets, shared with its post and jfast fragments
    std::shared_ptr<InSets> in_sets;
    std::string explain;
};

// returns 0 or a negative BKGPU_E* code; `err` receives the message
int compile_plan(const uint8_t* desc, size_t len, Compiled& out, std::string& err);
// every program of the plan (main, post, jfast, join children's and star dimensions' filters, window stages' expressions): OP_IN_SET's constant := addr[set]
void patch_in_sets(Compiled& c, const std::vector<uint64_t>& addr);

// host-side ExprValue::cast_to on canonical images (x86 semantics == the reference's build)
uint64_t host_cast_prim(uint64_t v, int from, int to);
// literal.cpp: the text of a literal as a DATETIME / TIMESTAMP / DATE / TIME image (ExprValue::cast_to from STRING)
uint64_t parse_literal(const char* text, size_t length, int to_prim);
int host_prim_class(int prim);
int prim_storage(int prim);       // SType of the column buffer carrying `prim`
int storage_bytes(int stype);

}  // namespace bk
